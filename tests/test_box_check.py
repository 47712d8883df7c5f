"""CPU: pass 1's per-box classification (DESIGN.md section 4.2) checked empirically.  tools/box_check.c re-states
cone_record, hyp_frame and box_class of csrc/vote.cu next to the reference predicate and searches adversarial boxes of
hypotheses for a pixel the box decides while the reference disagrees for some hypothesis of it (exit code 1)."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def box_check(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("box") / "box_check")
    cc = os.environ.get("CC", "gcc")
    flags = ["-O2", "-ffp-contract=off"]
    with open("/proc/cpuinfo") as fh:
        if " fma " in fh.read():
            flags.append("-mfma")
    subprocess.check_call([cc] + flags + [os.path.join(ROOT, "tools", "box_check.c"), "-lm", "-o", exe])
    return exe


@pytest.mark.parametrize("thresh", ["0.5", "0.9", "0.99", "0.999"])
def test_no_decided_pixel_disagrees(box_check, thresh):
    r = subprocess.run([box_check, "1000000", thresh], stdout=subprocess.PIPE, text=True, timeout=120)
    assert r.returncode == 0, r.stdout
    m = re.search(r"decided=(\d+) tested=(\d+) mismatches=0 worst \|m\|/delta_H=([0-9.]+)", r.stdout)
    assert m and int(m.group(1)) > 100000 and float(m.group(3)) >= 1.0, r.stdout
