"""CPU tests of the CenterNet heatmap loss (clean_pvnet_b200.ct_loss, csrc/ct_loss.cu): the numpy restatement of the
datasets' heatmap against the stored fixture and, where the clean-pvnet checkout exists, against the reference functions
themselves; ct_radius against gaussian_radius; the fp64 exp margins that make the device target bit-equal; the C ABI's
argument validation (before any CUDA call, so no device is needed); and the zero-edit drop-in on a miniature clean-pvnet
tree, from a dataset's sample through the collator to the trainer factory."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from ct_target_cases import case_images, pack, restate_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ct_target.npz")
REFERENCE = os.environ.get("PVNET_REFERENCE", "/root/reference")
HAS_REFERENCE = os.path.isfile(os.path.join(REFERENCE, "lib", "utils", "data_utils.py"))


def _reference():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        import make_golden_ct_target as g
    finally:
        sys.path.pop(0)
    return g, g.reference_data_utils(REFERENCE)


def test_restatement_equals_fixture():
    z = np.load(GOLDEN)
    for c, (B, C, H, W, images) in enumerate(case_images()):
        ind, rad, cls, c01, wh = pack(images, W, lambda h, w: 0)
        assert np.array_equal(z[f"ct_ind{c}"], ind) and np.array_equal(z[f"ct_cls{c}"], cls)
        assert np.array_equal(z[f"ct_01{c}"], c01) and np.array_equal(z[f"wh{c}"], wh, equal_nan=True)
        got = restate_batch(z[f"ct_ind{c}"], z[f"ct_radius{c}"], cls, c01, C, H, W)
        assert got.dtype == np.float32 and got.shape == (B, C, H, W)
        assert np.array_equal(got.view(np.uint32), z[f"ct_hm{c}"].view(np.uint32)), c


def test_fixture_covers_the_edge_cases():
    z = np.load(GOLDEN)
    ind, rad, c01, hm = z["ct_ind0"], z["ct_radius0"], z["ct_010"], z["ct_hm0"]
    H, W = hm.shape[2:]
    cy, cx = np.divmod(ind, W)
    on = c01 == 1
    assert (rad[on] == 0).sum() >= 3                                          # r = 0
    for sel in (cx == 0, cx == W - 1, cy == 0, cy == H - 1, (cx == 0) & (cy == 0), (cx == W - 1) & (cy == H - 1)):
        assert (sel & on).any()                                               # borders and corners
    assert not on[3].any() and not hm[3].any()                                # an image without objects
    img1 = [(int(i), int(c)) for i, c, v in zip(ind[1], z["ct_cls0"][1], c01[1]) if v == 1]
    assert len({i for i, _ in img1}) < len(img1)                              # several classes at one centre
    assert len([c for _, c in img1 if c == 0]) >= 2                           # same-class overlapping windows
    wh = z["wh0"][2]
    h = wh[:, 1][np.isfinite(wh[:, 1])]
    assert (np.ceil(h) != np.ceil(h.astype(np.float32))).any()                # float32 would change the radius rule
    assert np.unique(z["ct_cls1"][z["ct_011"] == 1]).size >= 5
    assert hm.max() == 1 and z["ct_hm1"].shape[1:] == (30, 104, 128) and z["ct_hm2"].shape[1:] == (30, 136, 184)


def test_half_pixel_centres_round_half_to_even():
    from ct_target_cases import centre
    assert centre((2, 2, 7, 9)) == (4, 6) and centre((4, 3, 11, 12)) == (8, 8) and centre((13, 2.5, 18, 7.5)) == (16, 5)


@pytest.mark.skipif(not HAS_REFERENCE, reason="no clean-pvnet checkout")
def test_restatement_equals_live_draw_umich_gaussian():
    g, du = _reference()
    radius = g.reference_radius(du)
    for c, (B, C, H, W, images) in enumerate(case_images(seed=99)):
        ind, rad, cls, c01, _ = pack(images, W, radius)
        want = g.reference_ct_hm(du, ind, rad, cls, c01, C, H, W)
        assert np.array_equal(restate_batch(ind, rad, cls, c01, C, H, W).view(np.uint32), want.view(np.uint32))


# ---- radius -----------------------------------------------------------------------------------------------------------

def test_ct_radius_equals_the_fixture(pvb):
    z = np.load(GOLDEN)
    h, w = np.meshgrid(np.arange(1, 257, dtype=np.float64), np.arange(1, 257, dtype=np.float64), indexing="ij")
    assert np.array_equal(pvb.ct_radius(np.stack([w, h], -1)), z["radius_table"])
    assert np.array_equal(pvb.ct_radius(z["edge_wh"]), z["edge_radius"])
    for c in range(3):
        wh, rad, c01 = z[f"wh{c}"], z[f"ct_radius{c}"], z[f"ct_01{c}"]
        box = (c01 == 1) & np.isfinite(wh[..., 0])
        assert np.array_equal(pvb.ct_radius(wh[box]), rad[box])
    # the float32 batch wh would give another radius for some of these
    assert not np.array_equal(pvb.ct_radius(z["edge_wh"].astype(np.float32)), z["edge_radius"])
    assert pvb.ct_radius(np.zeros((0, 2))).shape == (0,) and pvb.ct_radius(np.zeros((2, 3, 2))).shape == (2, 3)


@pytest.mark.skipif(not HAS_REFERENCE, reason="no clean-pvnet checkout")
def test_ct_radius_equals_live_gaussian_radius(pvb):
    g, du = _reference()
    radius = g.reference_radius(du)
    rng = np.random.default_rng(5)
    wh = np.concatenate([rng.uniform(0, 300, (2000, 2)), np.floor(rng.uniform(1, 300, (500, 2))) + 1e-7])
    want = np.array([radius(h, w) for w, h in wh], np.int32)
    assert np.array_equal(pvb.ct_radius(wh), want)


def test_exp_margins_make_any_two_ulp_exp_exact():
    """For every r <= 128 and every (dx, dy) in the window, g = exp(-e/2) lies more than 2 fp64 ulps from an fp32
    rounding midpoint and more than 4 ulps from the 2^-52 cut, so an exp accurate to 2 ulps (the device's is within 1)
    gives the reference's float32 target.  g is symmetric in (dx, dy), so one octant is enough."""
    cut = np.finfo(np.float64).eps
    n = 0
    for r in range(129):
        s = (2 * r + 1) / 6
        s2 = s * s
        d = np.arange(r + 1, dtype=np.float64)
        a = d * d / s2
        e = a[:, None] + a[None, :]
        g = np.exp(-e / 2)[np.triu_indices(r + 1)]
        n += g.size
        lo, hi = g, g
        for _ in range(2):
            lo, hi = np.nextafter(lo, 0), np.nextafter(hi, 2)
        keep = g >= cut
        assert np.array_equal(lo[keep].astype(np.float32), hi[keep].astype(np.float32)), r
        lo4, hi4 = g, g
        for _ in range(4):
            lo4, hi4 = np.nextafter(lo4, 0), np.nextafter(hi4, 2)
        assert np.array_equal(lo4 >= cut, hi4 >= cut), r
    assert n == sum((r + 1) * (r + 2) // 2 for r in range(129))


# ---- C ABI ------------------------------------------------------------------------------------------------------------

def _buf():
    buf = ctypes.create_string_buffer(1 << 20)
    return buf, ctypes.addressof(buf)


def test_ct_target_validation(pvb):
    L = pvb._lib
    lib = L.load()
    INV, OK = L.PVB_ERR_INVALID, L.PVB_OK
    _keep, p = _buf()
    t = lib.pvb_ct_target

    def f(ind=p, rad=p, cls=p, c01=p, out=p, B=2, M=5, C=30, H=8, W=12):
        return t(ind, rad, cls, c01, out, B, M, C, H, W, None)

    for k in ("B", "M", "C", "H", "W"):
        assert f(**{k: -1}) == INV
        assert b"negative size" in lib.pvb_last_error()
    assert f(M=1025) == INV and b"M must be at most 1024" in lib.pvb_last_error()
    assert f(B=65536) == INV and f(C=65536) == INV
    assert f(H=65536, W=32768) == INV and b"too large" in lib.pvb_last_error()
    for k in ("ind", "rad", "cls", "c01", "out"):
        assert f(**{k: None}) == INV, k
        assert b"NULL tensor" in lib.pvb_last_error()
    # nothing to draw or nothing to read: no-ops, whatever the pointers
    assert f(ind=None, rad=None, cls=None, c01=None, out=None, B=0) == OK
    assert f(out=None, H=0) == OK
    assert f(ind=None, rad=None, cls=None, c01=None, M=0, B=2, C=0) == OK


def test_ct_loss_workspace_sizing(pvb):
    ws = pvb._lib.load().pvb_ct_loss_workspace_bytes

    def want(B, C, H, W):
        n = B * C * ((W + 31) // 32) * ((H + 15) // 16)       # one partial per (32x16 tile, class, image)
        up = lambda x: (x + 255) // 256 * 256                  # noqa: E731
        return 256 + 2 * up(8 * n) + up(4 * n)
    for shape in ((32, 30, 104, 128), (4, 30, 136, 184), (1, 1, 1, 1), (3, 7, 17, 33)):
        assert ws(*shape) == want(*shape), shape
    assert ws(0, 30, 104, 128) == 256 and ws(-1, 4, 4, 4) == 0 and ws(1, -1, 4, 4) == 0


def test_ct_loss_validation(pvb):
    L = pvb._lib
    lib = L.load()
    INV, WS = L.PVB_ERR_INVALID, L.PVB_ERR_WORKSPACE
    _keep, p = _buf()
    ls = (ctypes.c_int64 * 4)(30 * 96, 96, 12, 1)
    fwd, bwd = lib.pvb_ct_loss_forward, lib.pvb_ct_loss_backward
    need = lib.pvb_ct_loss_workspace_bytes(2, 30, 8, 12)
    p256 = (p + 255) // 256 * 256

    def f(x=p, lstr=ls, ind=p, rad=p, cls=p, c01=p, loss=p, B=2, M=5, C=30, H=8, W=12, ws=p256, nb=need):
        return fwd(x, lstr, ind, rad, cls, c01, loss, B, M, C, H, W, ws, nb, None)

    def b(x=p, lstr=ls, ind=p, rad=p, cls=p, c01=p, g=p, grad=p, B=2, M=5, C=30, H=8, W=12, ws=p256, nb=need):
        return bwd(x, lstr, ind, rad, cls, c01, g, grad, B, M, C, H, W, ws, nb, None)

    for call in (f, b):
        assert call(B=-1) == INV and call(M=-1) == INV and call(C=-1) == INV and call(H=-1) == INV
        assert call(M=1025) == INV and call(B=65536) == INV and call(H=65536, W=32768) == INV
        assert call(lstr=None) == INV and b"stride array" in lib.pvb_last_error()
        assert call(lstr=(ctypes.c_int64 * 4)(30 * 96, 96, -12, 1)) == INV
        assert b"negative stride" in lib.pvb_last_error()
        for name in ("x", "ind", "rad", "cls", "c01"):
            assert call(**{name: None}) == INV, name
            assert b"NULL tensor" in lib.pvb_last_error()
        assert call(ws=None) == WS
        assert call(nb=need - 1) == WS and b"workspace" in lib.pvb_last_error()
        assert call(ws=p256 + 8) == WS and b"aligned" in lib.pvb_last_error()
    assert f(loss=None) == INV
    assert b(g=None) == INV and b(grad=None) == INV
    assert b(x=None, ind=None, rad=None, cls=None, c01=None, g=None, grad=None, B=0, ws=None, nb=0) == L.PVB_OK


def test_python_surface_rejects_bad_inputs(pvb):
    import torch
    objs = [torch.zeros(2, 3, dtype=dt) for dt in (torch.int64, torch.int32, torch.int64, torch.float32)]
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        pvb.ct_focal_loss(torch.zeros(2, 30, 8, 8), *objs)
    with pytest.raises(RuntimeError, match="CUDA device"):
        pvb.ct_target_batch(*objs, 30, 8, 8)
    with pytest.raises(RuntimeError, match="ct_radius"):
        pvb.CtNetworkWrapper(torch.nn.Identity())({'inp': torch.zeros(1), 'ct_hm': torch.zeros(1, 30, 8, 8)})
    with pytest.raises(ValueError):
        pvb.ct_radius(np.zeros((3, 3)))


# ---- drop-in ----------------------------------------------------------------------------------------------------------

def _run(code, cwd):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=cwd, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    return r.stdout


# A miniature clean-pvnet tree: the dataset draws ct_hm per object as lib/datasets/tless/ct.py does (through the numpy
# restatement and a recorded radius rule), the original 'ct' collator must never run, make_collator reads the dict at
# call time, and the trainer factory loads the trainer file by path (make_trainer.py:6-10).
TREE = {
    "lib/__init__.py": "",
    "lib/config/__init__.py": "cfg = 'real lib.config'\n",
    "lib/utils/__init__.py": "",
    "lib/utils/pvnet/pvnet_data_utils.py": "def compute_vertex(mask, kpt_2d):\n    raise RuntimeError('dense compute_vertex')\n",
    "lib/datasets/__init__.py": "",
    "lib/datasets/collate_batch.py": textwrap.dedent("""\
        from torch.utils.data.dataloader import default_collate


        def ct_collator(batch):
            raise RuntimeError('the dense ct collator ran')


        _collators = {'ct': ct_collator}


        def make_collator(cfg):
            if cfg.task in _collators:
                return _collators[cfg.task]
            return default_collate
        """),
    "lib/datasets/tless/__init__.py": "",
    "lib/datasets/tless/ct.py": textwrap.dedent("""\
        import math
        import numpy as np
        import torch.utils.data as data
        from ct_target_cases import centre, restate_ct_hm

        RADII = []


        class Dataset(data.Dataset):
            def __init__(self, images, C, H, W, radius):
                self.images, self.C, self.H, self.W, self.radius = images, C, H, W, radius

            def __getitem__(self, index):
                ct_hm = np.zeros([self.C, self.H, self.W], dtype=np.float32)
                wh, ct_cls, ct_ind = [], [], []
                for box, cls_id in self.images[index]:
                    x_min, y_min, x_max, y_max = box
                    ct = centre(box)
                    h, w = y_max - y_min, x_max - x_min
                    radius = self.radius(h, w)
                    RADII.append(radius)
                    ct_hm[cls_id] = np.maximum(ct_hm[cls_id], restate_ct_hm([ct[1] * self.W + ct[0]], [radius], [0],
                                                                            [1], 1, self.H, self.W)[0])
                    wh.append([w, h])
                    ct_cls.append(cls_id)
                    ct_ind.append(ct[1] * self.W + ct[0])
                ret = {'inp': np.zeros((3, 4 * self.H, 4 * self.W), np.float32), 'ct_hm': ct_hm, 'wh': wh,
                       'ct_cls': ct_cls, 'ct_ind': ct_ind}
                ret.update({'meta': {'center': np.zeros(2), 'scale': np.ones(2), 'ct_num': len(ct_ind)}})
                return ret

            def __len__(self):
                return len(self.images)
        """),
    "lib/train/__init__.py": "from .trainers import make_trainer\n",
    "lib/train/trainers/__init__.py": "from .make_trainer import make_trainer\n",
    "lib/train/trainers/make_trainer.py": textwrap.dedent("""\
        import importlib.machinery
        import os


        class Trainer(object):
            def __init__(self, network):
                self.network = network


        def _wrapper_factory(cfg, network):
            module = '.'.join(['lib.train.trainers', cfg.task])
            path = os.path.join('lib/train/trainers', cfg.task+'.py')
            network_wrapper = importlib.machinery.SourceFileLoader(module, path).load_module().NetworkWrapper(network)
            return network_wrapper


        def make_trainer(cfg, network):
            network = _wrapper_factory(cfg, network)
            return Trainer(network)
        """),
    "lib/train/trainers/pvnet.py": "raise RuntimeError('reference pvnet trainer loaded')\n",
    "lib/train/trainers/ct.py": "raise RuntimeError('reference ct trainer loaded')\n",
    "lib/train/trainers/snake.py": "class NetworkWrapper(object):\n    tag = 'snake'\n\n    def __init__(self, net):\n        self.net = net\n",
}


def _checkout(tmp_path):
    for rel, text in TREE.items():
        f = tmp_path / rel
        f.parent.mkdir(parents=True, exist_ok=True)
        f.write_text(text)
    return str(tmp_path)


def test_dropin_on_a_miniature_checkout(tmp_path):
    tree = _checkout(tmp_path)
    code = f"""
        import sys
        sys.path.insert(0, {tree!r})
        import numpy as np
        import torch
        import clean_pvnet_b200
        from ct_target_cases import case_images, restate_batch
        clean_pvnet_b200.install_ct_loss_as_reference()

        # the collator: no ct_hm, the dataset's radii, and a heatmap rebuilt from the batch equal to the stacked one
        from lib.datasets.collate_batch import make_collator
        from lib.datasets.tless.ct import Dataset, RADII
        B, C, H, W, images = case_images()[0]
        images = images[1:]                                 # the images of boxes, the last one empty
        ds = Dataset(images, C, H, W, lambda h, w: clean_pvnet_b200.ct_radius([w, h]).item())
        class Cfg: task = 'ct'
        samples = [ds[i] for i in range(len(ds))]
        batch = make_collator(Cfg)(samples)
        assert 'ct_hm' not in batch and 'img' not in batch
        assert set(batch) == {{'inp', 'meta', 'wh', 'ct_cls', 'ct_ind', 'ct_01', 'ct_radius'}}
        c01 = batch['ct_01']
        assert c01.dtype == torch.float32 and batch['ct_radius'].dtype == torch.int32
        assert batch['ct_ind'].dtype == torch.int64 and batch['ct_cls'].dtype == torch.int64
        assert batch['wh'].dtype == torch.float32 and list(batch['wh'].shape) == [3, c01.shape[1], 2]
        assert batch['ct_radius'][c01 == 1].tolist() == RADII
        dense = np.stack([s['ct_hm'] for s in samples])
        rebuilt = restate_batch(*(batch[k].numpy() for k in ('ct_ind', 'ct_radius', 'ct_cls', 'ct_01')), C, H, W)
        assert np.array_equal(rebuilt.view(np.uint32), dense.view(np.uint32))
        for s in samples:
            s['img'] = np.zeros((2, 2), np.uint8)
        assert list(make_collator(Cfg)(samples)['img'].shape) == [3, 2, 2]

        # the trainer: ct and pvnet get the fused wrappers in either install order, other tasks the original factory
        from lib.train import make_trainer
        net = torch.nn.Identity()
        def check():
            Cfg.task = 'ct'
            assert type(make_trainer(Cfg, net).network) is clean_pvnet_b200.CtNetworkWrapper
            Cfg.task = 'snake'
            assert make_trainer(Cfg, net).network.tag == 'snake'
        check()
        clean_pvnet_b200.install_vote_loss_as_reference()
        check()
        Cfg.task = 'pvnet'
        assert type(make_trainer(Cfg, net).network) is clean_pvnet_b200.NetworkWrapper
        factory = sys.modules['lib.train.trainers.make_trainer']._wrapper_factory
        clean_pvnet_b200.install_ct_loss_as_reference()               # idempotent, whatever came in between
        clean_pvnet_b200.install_vote_loss_as_reference()
        assert sys.modules['lib.train.trainers.make_trainer']._wrapper_factory is factory
        check()

        import lib, lib.config
        assert lib.__file__.startswith({tree!r}) and not getattr(lib, '__pvb_stand_in__', False)
        assert lib.config.cfg == 'real lib.config'
        print('ok')
    """
    assert "ok" in _run(code, cwd=tree)


def test_dropin_vote_loss_first(tmp_path):
    tree = _checkout(tmp_path)
    code = f"""
        import sys
        sys.path.insert(0, {tree!r})
        import torch
        import clean_pvnet_b200
        clean_pvnet_b200.install_vote_loss_as_reference()
        clean_pvnet_b200.install_ct_loss_as_reference()
        factory = sys.modules['lib.train.trainers.make_trainer']._wrapper_factory
        clean_pvnet_b200.install_vote_loss_as_reference()
        clean_pvnet_b200.install_ct_loss_as_reference()
        assert sys.modules['lib.train.trainers.make_trainer']._wrapper_factory is factory
        from lib.train import make_trainer
        class Cfg: task = 'pvnet'
        net = torch.nn.Identity()
        assert type(make_trainer(Cfg, net).network) is clean_pvnet_b200.NetworkWrapper
        Cfg.task = 'ct'
        assert type(make_trainer(Cfg, net).network) is clean_pvnet_b200.CtNetworkWrapper
        Cfg.task = 'snake'
        assert make_trainer(Cfg, net).network.tag == 'snake'
        print('ok')
    """
    assert "ok" in _run(code, cwd=tree)


@pytest.mark.skipif(not HAS_REFERENCE, reason="no clean-pvnet checkout")
def test_collator_equals_the_reference_collator_but_for_ct_hm():
    """On samples that carry 'img' (the reference collator needs it), every key the reference's ct_collator builds,
    except ct_hm, equals the twin's."""
    import importlib.util
    import torch
    from clean_pvnet_b200.ct_loss import ct_collator
    spec = importlib.util.spec_from_file_location("reference_collate_batch",
                                                  os.path.join(REFERENCE, "lib", "datasets", "collate_batch.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    rng = np.random.default_rng(3)
    samples = []
    for n in (3, 0, 5):
        wh = rng.uniform(1, 40, (n, 2)).tolist()
        samples.append({'inp': np.zeros((3, 8, 8), np.float32), 'img': np.zeros((8, 8, 3), np.uint8),
                        'ct_hm': np.zeros((30, 2, 2), np.float32), 'wh': wh,
                        'ct_cls': rng.integers(0, 30, n).tolist(), 'ct_ind': rng.integers(0, 4, n).tolist(),
                        'meta': {'center': np.zeros(2), 'scale': np.ones(2), 'ct_num': n}})
    want = ref.ct_collator(samples)
    got = ct_collator(samples)
    assert set(want) - set(got) == {'ct_hm'} and set(got) - set(want) == {'ct_radius'}
    for k in ('inp', 'img', 'wh', 'ct_cls', 'ct_ind', 'ct_01'):
        assert want[k].dtype == got[k].dtype and torch.equal(want[k], got[k]), k
    assert torch.equal(want['meta']['ct_num'], got['meta']['ct_num'])
