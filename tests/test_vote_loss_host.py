"""CPU tests of the vote loss (clean_pvnet_b200.vote_loss, csrc/loss.cu): the numpy restatement of compute_vertex against
the stored fixture and, where the clean-pvnet checkout exists, against the reference function itself; the C ABI's
argument validation (before any CUDA call, so no device is needed); and the zero-edit drop-in on a miniature clean-pvnet
tree, from a dataset's compute_vertex call through default_collate to the trainer factory."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from vote_target_cases import case_inputs, restate_vertex

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "vote_target.npz")
REFERENCE = os.environ.get("PVNET_REFERENCE", "/root/reference")


def test_restatement_equals_fixture():
    z = np.load(GOLDEN)
    for c, (mask, kpt) in enumerate(case_inputs()):
        assert np.array_equal(z[f"mask{c}"], mask) and np.array_equal(z[f"kpt{c}"], kpt)
        got = np.stack([restate_vertex(m, k) for m, k in zip(mask, kpt)])
        assert got.dtype == np.float32
        assert np.array_equal(got.view(np.uint32), z[f"vertex{c}"].view(np.uint32)), c


def test_fixture_covers_the_edge_cases():
    z = np.load(GOLDEN)
    ks, values, on_pixel, near_pixel, far = set(), set(), 0, 0, 0
    for c in range(3):
        mask, kpt, v = z[f"mask{c}"], z[f"kpt{c}"], z[f"vertex{c}"]
        ks.add(kpt.shape[1])
        values |= set(np.unique(mask).tolist())
        for i in range(mask.shape[0]):
            for j, (x, y) in enumerate(kpt[i]):
                far += abs(x) >= 1e6
                if x == int(x) and y == int(y) and 0 <= x < mask.shape[2] and 0 <= y < mask.shape[1]:
                    on_pixel += 1
                    assert v[i, 2 * j, int(y), int(x)] == 0 and v[i, 2 * j + 1, int(y), int(x)] == 0
                d = np.hypot(x - np.round(x), y - np.round(y))
                near_pixel += 0 < d < 1e-3
    assert ks == {1, 9, 17} and values == {0, 1, 2, 255}
    assert on_pixel and near_pixel and far and (np.concatenate([z[f"kpt{c}"].ravel() for c in range(3)]) < 0).any()


def test_restatement_equals_live_compute_vertex():
    if not os.path.isfile(os.path.join(REFERENCE, "lib", "utils", "pvnet", "pvnet_data_utils.py")):
        pytest.skip("no clean-pvnet checkout")
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        from make_golden_vote_target import reference_compute_vertex
    finally:
        sys.path.pop(0)
    compute_vertex = reference_compute_vertex(REFERENCE)
    rng = np.random.default_rng(7)
    for mask, kpt in case_inputs(seed=99):
        for m, k in zip(mask, kpt):
            want = compute_vertex(m, k).transpose(2, 0, 1)
            assert np.array_equal(restate_vertex(m, k).view(np.uint32), want.view(np.uint32))
            k32 = k.astype(np.float32)                      # float32 keypoints are promoted exactly
            assert np.array_equal(restate_vertex(m, k32).view(np.uint32),
                                  compute_vertex(m, k32).transpose(2, 0, 1).view(np.uint32))
    m = (rng.random((48, 64)) < 0.3).astype(np.uint8)
    k = rng.uniform(-10, 70, (9, 2))
    assert np.array_equal(restate_vertex(m, k).view(np.uint32), compute_vertex(m, k).transpose(2, 0, 1).view(np.uint32))


# ---- C ABI ------------------------------------------------------------------------------------------------------------

def _buf():
    buf = ctypes.create_string_buffer(1 << 20)
    return buf, ctypes.addressof(buf)


def test_vote_target_validation(pvb):
    L = pvb._lib
    lib = L.load()
    INV, OK, U8 = L.PVB_ERR_INVALID, L.PVB_OK, L.PVB_MASK_U8
    _keep, p = _buf()
    s = (ctypes.c_int64 * 3)(48, 8, 1)
    vt = lib.pvb_vote_target
    # mask, mask_dtype, mask_stride, kpt_2d, vertex, B, H, W, K, stream
    for B, H, W in ((-1, 6, 8), (1, -6, 8), (1, 6, -8)):
        assert vt(p, U8, s, p, p, B, H, W, 9, None) == INV
        assert b"negative size" in lib.pvb_last_error()
    for K in (0, -1, 1025):
        assert vt(p, U8, s, p, p, 1, 6, 8, K, None) == INV
        assert b"K must be" in lib.pvb_last_error()
    assert vt(p, U8, s, p, p, 65536, 6, 8, 9, None) == INV
    assert vt(p, U8, s, p, p, 1, 65536, 32768, 9, None) == INV
    assert b"too large" in lib.pvb_last_error()
    for bad in (L.PVB_MASK_F32, L.PVB_MASK_F64, 7, -1):
        assert vt(p, bad, s, p, p, 1, 6, 8, 9, None) == INV
        assert b"dtype" in lib.pvb_last_error()
    assert vt(p, U8, None, p, p, 1, 6, 8, 9, None) == INV
    assert b"stride array" in lib.pvb_last_error()
    assert vt(p, U8, (ctypes.c_int64 * 3)(48, -8, 1), p, p, 1, 6, 8, 9, None) == INV
    assert b"negative stride" in lib.pvb_last_error()
    for i in (0, 3, 4):
        args = [p, U8, s, p, p]
        args[i] = None
        assert vt(*args, 1, 6, 8, 9, None) == INV, i
        assert b"NULL tensor" in lib.pvb_last_error()
    # an empty batch or image is a no-op, whatever the tensor pointers
    assert vt(None, U8, s, None, None, 0, 6, 8, 9, None) == OK
    assert vt(None, U8, s, None, None, 2, 0, 8, 9, None) == OK


def test_vote_loss_workspace_sizing(pvb):
    ws = pvb._lib.load().pvb_vote_loss_workspace_bytes
    # the fp32 weight sum in the first 256 bytes, then one fp64 and one int64 partial per 256-pixel CTA, 256-byte aligned
    assert ws(32, 480, 640) == 256 + 2 * 32 * 1200 * 8
    assert ws(1, 1, 1) == 256 + 256 + 256
    assert ws(3, 479, 641) == 256 + 2 * ((3 * 1200 * 8 + 255) // 256 * 256)
    assert ws(0, 480, 640) == 256 and ws(-1, 4, 4) == 0


def test_vote_loss_validation(pvb):
    L = pvb._lib
    lib = L.load()
    INV, WS, U8 = L.PVB_ERR_INVALID, L.PVB_ERR_WORKSPACE, L.PVB_MASK_U8
    _keep, p = _buf()
    ms = (ctypes.c_int64 * 3)(48, 8, 1)
    ps = (ctypes.c_int64 * 4)(864, 48, 8, 1)
    fwd, bwd = lib.pvb_vote_loss_forward, lib.pvb_vote_loss_backward
    need = lib.pvb_vote_loss_workspace_bytes(2, 6, 8)
    p256 = (p + 255) // 256 * 256

    def f(pred=p, pstr=ps, mask=p, dt=U8, mstr=ms, kpt=p, loss=p, B=2, H=6, W=8, K=9, ws=p256, nb=need):
        return fwd(pred, pstr, mask, dt, mstr, kpt, loss, B, H, W, K, ws, nb, None)

    def b(pred=p, pstr=ps, mask=p, dt=U8, mstr=ms, kpt=p, g=p, grad=p, B=2, H=6, W=8, K=9, ws=p256, nb=need):
        return bwd(pred, pstr, mask, dt, mstr, kpt, g, grad, B, H, W, K, ws, nb, None)

    for call in (f, b):
        assert call(B=-1) == INV and call(H=-1) == INV and call(W=-1) == INV
        assert call(K=0) == INV and call(K=1025) == INV
        assert b"K must be" in lib.pvb_last_error()
        assert call(dt=L.PVB_MASK_F32) == INV and call(dt=7) == INV
        assert call(mstr=None) == INV and call(pstr=None) == INV
        assert b"stride array" in lib.pvb_last_error()
        assert call(pstr=(ctypes.c_int64 * 4)(864, 48, -8, 1)) == INV
        assert b"negative stride" in lib.pvb_last_error()
        for name in ("pred", "mask", "kpt"):
            assert call(**{name: None}) == INV, name
            assert b"NULL tensor" in lib.pvb_last_error()
        assert call(ws=None) == WS
        assert call(nb=need - 1) == WS
        assert b"workspace" in lib.pvb_last_error()
        assert call(ws=p256 + 8) == WS
        assert b"aligned" in lib.pvb_last_error()
    assert f(loss=None) == INV
    assert b(g=None) == INV and b(grad=None) == INV
    # the backward pass of an empty batch is a no-op
    assert b(pred=None, mask=None, kpt=None, g=None, grad=None, B=0, ws=None, nb=0) == L.PVB_OK


def test_python_surface_rejects_bad_inputs(pvb):
    from clean_pvnet_b200.vote_loss import keypoints_from_compact
    cpu_mask = torch.zeros(2, 6, 8, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        pvb.vote_target_batch(cpu_mask, np.zeros((2, 9, 2)))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        pvb.vote_loss(torch.zeros(2, 18, 6, 8), cpu_mask, np.zeros((2, 9, 2)))
    with pytest.raises(RuntimeError, match="compact keypoint form"):
        keypoints_from_compact(torch.zeros(2, 18, 6, 8))                 # a dense field: the dataset was not patched
    with pytest.raises(RuntimeError, match="compact keypoint form"):
        keypoints_from_compact(torch.zeros(2, 2, 1, 9, dtype=torch.float32))
    kpt = torch.arange(36, dtype=torch.float64).reshape(2, 9, 2)
    from clean_pvnet_b200.vote_loss import compact_vertex
    compact = torch.from_numpy(np.stack([compact_vertex(None, k).transpose(2, 0, 1) for k in kpt.numpy()]))
    assert compact.dtype == torch.float64 and list(compact.shape) == [2, 2, 1, 9]
    assert torch.equal(keypoints_from_compact(compact), kpt)


def test_network_wrapper_keeps_the_pose_test_branch(pvb):
    w = pvb.NetworkWrapper(torch.nn.Identity())
    inp = torch.ones(1, 3, 4, 4)
    out, loss, scalar_stats, image_stats = w({'inp': inp, 'meta': {'pose_test': True}})
    assert out is inp and loss.item() == 0 and scalar_stats == {} and image_stats == {}
    assert isinstance(w.seg_crit, torch.nn.CrossEntropyLoss)


# ---- drop-in ----------------------------------------------------------------------------------------------------------

def _run(code, cwd):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=cwd, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    return r.stdout


# A miniature clean-pvnet tree: the dense compute_vertex must never run, the trainer factory loads the trainer file by
# path (make_trainer.py:6-10; `imp.load_source` is SourceFileLoader.load_module on Pythons without `imp`), and the
# reference pvnet trainer must never be loaded.
TREE = {
    "lib/__init__.py": "",
    "lib/config/__init__.py": "cfg = 'real lib.config'\n",
    "lib/utils/__init__.py": "",
    "lib/utils/pvnet/pvnet_data_utils.py": "def compute_vertex(mask, kpt_2d):\n    raise RuntimeError('dense compute_vertex')\n",
    "lib/datasets/__init__.py": "",
    "lib/datasets/linemod/__init__.py": "",
    "lib/datasets/linemod/pvnet.py": textwrap.dedent("""\
        import numpy as np
        import torch.utils.data as data
        from lib.utils.pvnet import pvnet_data_utils


        class Dataset(data.Dataset):
            def __init__(self, masks, kpts):
                self.masks, self.kpts = masks, kpts

            def __getitem__(self, index):
                mask, kpt_2d = self.masks[index], self.kpts[index]
                inp = np.zeros((3,) + mask.shape, np.float32)
                vertex = pvnet_data_utils.compute_vertex(mask, kpt_2d).transpose(2, 0, 1)
                return {'inp': inp, 'mask': mask.astype(np.uint8), 'vertex': vertex, 'img_id': index, 'meta': {}}

            def __len__(self):
                return len(self.masks)
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
    "lib/train/trainers/ct.py": "class NetworkWrapper(object):\n    tag = 'ct'\n\n    def __init__(self, net):\n        self.net = net\n",
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
        from torch.utils.data.dataloader import default_collate
        import clean_pvnet_b200
        from clean_pvnet_b200.vote_loss import keypoints_from_compact
        clean_pvnet_b200.install_vote_loss_as_reference()

        # datasets: the unmodified __getitem__ now emits the compact form, and default_collate keeps it
        from lib.datasets.linemod.pvnet import Dataset
        rng = np.random.default_rng(0)
        masks = [(rng.random((6, 8)) < 0.5).astype(np.uint8) for _ in range(3)]
        kpts = [rng.uniform(-3, 9, (9, 2)) for _ in range(2)] + [rng.uniform(-3, 9, (9, 2)).astype(np.float32)]
        ds = Dataset(masks, kpts)
        item = ds[0]
        assert item['vertex'].dtype == np.float64 and item['vertex'].shape == (2, 1, 9)
        batch = default_collate([ds[i] for i in range(3)])
        v = batch['vertex']
        assert v.dtype == torch.float64 and list(v.shape) == [3, 2, 1, 9]
        want = torch.from_numpy(np.stack([k.astype(np.float64) for k in kpts]))
        assert torch.equal(keypoints_from_compact(v), want)
        assert batch['mask'].dtype == torch.uint8 and list(batch['mask'].shape) == [3, 6, 8]

        # trainer: pvnet gets the fused wrapper, every other task the original factory
        from lib.train import make_trainer
        class Cfg: task = 'pvnet'
        net = torch.nn.Identity()
        assert type(make_trainer(Cfg, net).network) is clean_pvnet_b200.NetworkWrapper
        Cfg.task = 'ct'
        assert make_trainer(Cfg, net).network.tag == 'ct'
        clean_pvnet_b200.install_vote_loss_as_reference()             # idempotent
        assert make_trainer(Cfg, net).network.tag == 'ct'
        Cfg.task = 'pvnet'
        assert type(make_trainer(Cfg, net).network) is clean_pvnet_b200.NetworkWrapper

        import lib, lib.config
        assert lib.__file__.startswith({tree!r}) and not getattr(lib, '__pvb_stand_in__', False)
        assert lib.config.cfg == 'real lib.config'
        print('ok')
    """
    assert "ok" in _run(code, cwd=tree)
