"""CPU: pass 1's per-box classification (pass1_box_twin, the model of box_class in csrc/vote.cu) against the oracle's exact
verdicts.  A pixel the model calls a certain inlier (outlier) of a box must be an inlier (outlier) of every hypothesis
the oracle tests inside the box: the box's corners, its centre and random points, as float32 tile-frame values.  Boxes are
drawn to be hard: a point, one ulp wide, straddling a pixel's cone edge, around the pixel itself, and far away."""
import numpy as np
import pytest

import pvnet_oracle as po
import pass1_box_twin as twin

F = np.float32


def _boxes(rng, xy, dirs, kappa):
    """adversarial boxes (x0, x1, y0, y1) in image coordinates around the pixels of a tile (the first four are bad vectors)"""
    out = []
    for _ in range(40):
        i = rng.integers(4, len(xy))                                              # a pixel with a real vector
        c, v = xy[i].astype(np.float64), dirs[i].astype(np.float64)
        v = v / np.hypot(*v)
        r = rng.uniform(0.5, 300)
        th = np.arctan(kappa) * rng.choice([-1, 1]) * rng.uniform(0.98, 1.02)   # on the cone edge
        e = c + r * np.array([np.cos(th) * v[0] - np.sin(th) * v[1], np.sin(th) * v[0] + np.cos(th) * v[1]])
        w = rng.choice([0.0, 1e-6, 1e-3, 0.5, 5.0])
        out.append((e[0], e[0] + w, e[1], e[1] + w))
        ex, ey = F(e[0]), F(e[1])                                                 # one ulp wide
        out.append((ex, np.nextafter(ex, F(np.inf)), ey, np.nextafter(ey, F(np.inf))))
        out.append((c[0] - 1e-4, c[0] + 1e-4, c[1] - 1e-4, c[1] + 1e-4))           # around the pixel itself
        d = rng.uniform(-20, 20, 2)
        out.append((c[0] + d[0], c[0] + d[0] + abs(d[1]) * 0.1, c[1] + d[1], c[1] + d[1] + 0.3))
    return out


@pytest.mark.parametrize("t", [0.5, 0.9, 0.99, 0.999])
def test_classification_agrees_with_the_oracle(t):
    rng = np.random.default_rng(int(t * 1000))
    kappa, band, floor = twin.cone_params(t)
    ang = rng.uniform(0, 2 * np.pi, 512)
    xy = np.stack([rng.integers(0, 64, 512), rng.integers(0, 16, 512)], 1).astype(F)
    dirs = np.stack([np.cos(ang), np.sin(ang)], 1).astype(F)
    dirs[:4] = [(0, 0), (np.nan, 1), (np.inf, 0), (1e30, -1e30)]                  # never vote / outside the analysis
    rec, ox, oy, cmax = twin.tile_records(xy, dirs, kappa)
    decided = 0
    for x0, x1, y0, y1 in _boxes(rng, xy, dirs, float(kappa)):
        pts = [(x0, y0), (x1, y0), (x0, y1), (x1, y1), ((x0 + x1) / 2, (y0 + y1) / 2)]
        pts += list(zip(rng.uniform(x0, x1, 3), rng.uniform(y0, y1, 3)))
        hyp = np.array(pts, F)
        xc, yc, ok = twin.hyp_frame(hyp, ox, oy)
        cls = twin.classify(rec, xc, yc, ok, cmax, band, floor)
        inl = po.voting_for_hypothesis(dirs[:, None, :], xy, hyp[:, None, :],
                                       np.zeros((len(hyp), 1, len(xy)), np.uint8), t)[:, 0, :]   # [hyp, pixel]
        assert (inl[:, cls == 1] == 1).all(), "a certain inlier is an outlier of some hypothesis of its box"
        assert (inl[:, cls == -1] == 0).all(), "a certain outlier is an inlier of some hypothesis of its box"
        assert (cls[:4] == [-1, -1, 0, 0]).all()          # zero and NaN vectors never vote; inf and huge ones: undecided
        decided += np.count_nonzero(cls)
    assert decided > 0


def test_unbounded_hypothesis_decides_nothing():
    kappa, band, floor = twin.cone_params(0.99)
    xy = np.array([[0, 0], [5, 5]], F)
    dirs = np.array([[1, 0], [0, 1]], F)
    rec, ox, oy, cmax = twin.tile_records(xy, dirs, kappa)
    xc, yc, ok = twin.hyp_frame(np.array([[10, 0], [np.inf, 0]], F), ox, oy)
    assert (twin.classify(rec, xc, yc, ok, cmax, band, floor) == 0).all()


def test_cfg2_boxes_predict_fewer_instructions():
    """the go/no-go of the box path: on two cfg-2 images one box of pass 1's 128 hypotheses predicts at least 1.5x fewer
    issued instructions in pass 1 than scoring every test"""
    tot, today = twin.workload_report("cfg2", (1236,), B=2, sizes=(128,))
    assert today / tot[128][2] >= 1.5
