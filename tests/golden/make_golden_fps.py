#!/usr/bin/env python
"""Writes tests/golden/fps.npz: the reference farthest-point sampling's indices (oracle/_ref/libfps_ref.so, the unmodified
lib/csrc/fps source built by oracle/build_fps_ref.py with its setup.py flags) for the seeded clouds of
tests/fps_cases.cases(), in both modes.  Only the seeds and the indices are stored; the tests rebuild the points.  In the
random mode the reference draws its own start (rand() % pn after srand(time(0))); its idxs[0] is that start and is
stored as `start`, and sn == 0 cases store start 0.

    python tests/golden/make_golden_fps.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import fps_cases  # noqa: E402


def main():
    lib = fps_cases.ref_lib()
    if lib is None:
        raise SystemExit(f"{fps_cases.REF_LIB} is missing: run oracle/build_fps_ref.py first")
    rows, idxs = [], []
    for kind, pn, sn, seed in fps_cases.cases():
        pts = fps_cases.cloud(kind, pn, seed)
        for init_center in (1, 0):
            r = fps_cases.ref_fps(lib, pts, sn, init_center)
            start = int(r[0]) if (sn and not init_center) else 0
            rows.append((fps_cases.KINDS.index(kind), pn, sn, seed, init_center, start))
            idxs.append(r)
    rows = np.array(rows, np.int64)
    offset = np.concatenate([[0], np.cumsum([len(r) for r in idxs])]).astype(np.int64)
    np.savez_compressed(fps_cases.GOLDEN, kind=rows[:, 0].astype(np.int8), pn=rows[:, 1].astype(np.int32),
                        sn=rows[:, 2].astype(np.int32), seed=rows[:, 3].astype(np.int32),
                        init_center=rows[:, 4].astype(np.int8), start=rows[:, 5].astype(np.int32), offset=offset,
                        idxs=np.concatenate(idxs).astype(np.int32))
    print(f"wrote {fps_cases.GOLDEN}: {len(rows)} cases, {int(offset[-1])} indices")


if __name__ == "__main__":
    main()
