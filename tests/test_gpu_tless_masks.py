"""GPU tests of T-LESS's instance masks (DESIGN.md 8k): the compose kernel against the reference's own handle_test_data
code (tests/golden/tless_masks.npz), instance_masks_batch against the numpy restatement (tests/tless_mask_cases.py)
applied to render_depth_batch of each instance, determinism, batch independence, stream / sync behaviour and the
OpenGL drop-in on a miniature checkout."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from tless_mask_cases import compose_restated
from test_tless_masks_host import ROOT, golden_cases, write_tless_checkout
from vsd_cases import K_SMALL, box, icosphere, torus

pytestmark = pytest.mark.gpu

MESHES = [box(), icosphere(3), torus(nu=48, nv=24)]
W, H = 100, 75                                          # not a multiple of 32 either way
OBJ = [3, 17, 30]


def cpu(t):
    return t.cpu().numpy()


def scene(B, per_image, seed):
    """B images with `per_image` (a count or a list) instances each, crowded into the view so they overlap."""
    rng = np.random.default_rng(seed)
    counts = per_image if isinstance(per_image, (list, tuple)) else [per_image] * B
    image_index = np.repeat(np.arange(B), counts)
    n = len(image_index)
    mesh_index = rng.integers(0, len(MESHES), n)
    obj_ids = np.array([OBJ[m] for m in mesh_index])
    poses = np.zeros((n, 3, 4))
    for i in range(n):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        w, x, y, z = q
        poses[i, :, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                           [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                           [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]
        poses[i, :, 3] = (rng.uniform(-80, 80), rng.uniform(-60, 60), rng.uniform(350, 700))
    Ks = np.repeat(K_SMALL[None], B, 0).copy()
    Ks[:, 0, 0] *= rng.uniform(0.5, 0.6, B)
    Ks[:, 1, 1] *= rng.uniform(0.5, 0.6, B)
    Ks[:, 0, 2] = rng.uniform(45, 55, B)
    Ks[:, 1, 2] = rng.uniform(33, 42, B)
    return mesh_index, obj_ids, image_index, poses, Ks


def expected(mesh_index, obj_ids, image_index, poses, K, B):
    """The restatement on render_depth_batch of each instance (at clip planes 10 / 10000)."""
    import clean_pvnet_b200 as pvb
    n = len(image_index)
    depth = np.zeros((n, H, W), np.float32)
    for i in range(n):
        Ki = K if K.ndim == 2 else K[image_index[i]]
        p, f = MESHES[mesh_index[i]]
        depth[i] = cpu(pvb.render_depth_batch(p, f, poses[i:i + 1], Ki, (W, H), near=10, far=10000))[0]
    label = np.zeros((B, H, W), np.int16)
    a, pn, bb = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros((n, 4), np.int64)
    for b in range(B):
        idx = np.flatnonzero(image_index == b)
        if len(idx):
            label[b], a[idx], pn[idx], bb[idx] = compose_restated(depth[idx], obj_ids[idx])
    return label, a, pn, bb


def assert_equal(got, want):
    label, a, p, bb = got
    assert label.dtype == torch.int16 and a.dtype == torch.int64 and p.dtype == torch.int64 and bb.dtype == torch.int32
    assert np.array_equal(cpu(label), want[0])
    assert np.array_equal(cpu(a), want[1]) and np.array_equal(cpu(p), want[2]) and np.array_equal(cpu(bb), want[3])


def test_compose_equals_the_reference_bit_for_bit(pvb):
    cs = golden_cases()
    for c in cs:
        m = c["depth"].shape[0]
        out = pvb.instance_masks_from_depth(torch.from_numpy(c["depth"]).cuda(), np.arange(m), c["obj_ids"],
                                           np.zeros(m, np.int64))
        assert_equal(out, (c["label"][None], c["a_pixel_num"], c["pixel_num"], c["bbox"]))
    # every case of one size in one call, with the slots in reverse order
    same = [c for c in cs if c["depth"].shape[1:] == (37, 53)]
    depth = np.concatenate([c["depth"] for c in same])[::-1].copy()
    n = len(depth)
    img = np.concatenate([np.full(c["depth"].shape[0], b) for b, c in enumerate(same)])
    label, a, p, bb = pvb.instance_masks_from_depth(torch.from_numpy(depth).cuda(), n - 1 - np.arange(n),
                                                    np.concatenate([c["obj_ids"] for c in same]), img)
    assert np.array_equal(cpu(label), np.stack([c["label"] for c in same]))
    assert np.array_equal(cpu(a), np.concatenate([c["a_pixel_num"] for c in same]))
    assert np.array_equal(cpu(p), np.concatenate([c["pixel_num"] for c in same]))
    assert np.array_equal(cpu(bb), np.concatenate([c["bbox"] for c in same]))


@pytest.mark.parametrize("k_per_image", [False, True])
@pytest.mark.parametrize("windows", ["one", "several"])
def test_batch_equals_the_restatement_on_rendered_depth(pvb, k_per_image, windows):
    B = 7
    mi, obj, img, poses, Ks = scene(B, [1, 5, 3, 0, 8, 2, 4], seed=11 + k_per_image)
    K = Ks if k_per_image else Ks[0]
    want = expected(mi, obj, img, poses, K, B if k_per_image else int(img[-1]) + 1)
    budget = 1 << 30 if windows == "one" else 6 * H * W * 4        # windows of at most 6 instances (or one image)
    meshes = [(torch.from_numpy(p).cuda(), torch.from_numpy(f).cuda()) for p, f in MESHES]
    got = pvb.instance_masks_batch(meshes, mi, obj, img, torch.from_numpy(poses).cuda(), torch.from_numpy(K).cuda(),
                                   (W, H), max_render_bytes=budget)
    assert_equal(got, want)
    assert cpu(got[2]).sum() > 0 and (cpu(got[2]) < cpu(got[1])).any()   # something is occluded
    assert not cpu(got[0][3]).any()                                      # the image without instances


def test_deterministic_and_independent_of_the_batch(pvb):
    B = 6
    mi, obj, img, poses, Ks = scene(B, 20, seed=5)
    args = dict(meshes=MESHES, mesh_index=mi, obj_ids=obj, image_index=img, size=(W, H))
    full = pvb.instance_masks_batch(poses=poses, K=Ks, **args)
    again = pvb.instance_masks_batch(poses=poses, K=Ks, **args)
    for x, y in zip(full, again):
        assert torch.equal(x, y)
    for b in (0, 4):
        sel = img == b
        one = pvb.instance_masks_batch(MESHES, mi[sel], obj[sel], np.zeros(sel.sum(), np.int64), poses[sel], Ks[b],
                                       (W, H))
        assert torch.equal(one[0][0], full[0][b])
        for x, y in zip(one[1:], full[1:]):
            assert torch.equal(x, y[torch.from_numpy(np.flatnonzero(sel)).cuda()])


def test_no_sync_and_side_stream(pvb):
    B = 4
    mi, obj, img, poses, Ks = scene(B, 3, seed=9)
    dev = torch.device("cuda")
    meshes = [(torch.from_numpy(p).to(dev), torch.from_numpy(f).to(dev)) for p, f in MESHES]
    pz, K = torch.from_numpy(poses).to(dev), torch.from_numpy(Ks).to(dev)
    ref = pvb.instance_masks_batch(meshes, mi, obj, img, pz, K, (W, H))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = pvb.instance_masks_batch(meshes, mi, obj, img, pz, K, (W, H), max_render_bytes=3 * H * W * 4)
        dep = pvb.instance_masks_from_depth(torch.zeros((2, H, W), device=dev), [0, 1], [1, 2], [0, 1])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for x, y in zip(out, ref):
        assert torch.equal(x, y)
    assert not dep[0].any() and not dep[1].any()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        side = pvb.instance_masks_batch(meshes, mi, obj, img, pz, K, (W, H))
    torch.cuda.current_stream().wait_stream(s)
    for x, y in zip(side, ref):
        assert torch.equal(x, y)


def test_reference_loop_over_the_dropin_equals_the_batch(tmp_path):
    """The miniature checkout's opengl_renderer.render (the reference's call of its backend at clip planes 10 / 10000
    and its division by 1000) over install_tless_renderer_as_reference(), composed as update_mask composes, and its
    np.sum(depth != 0), equal instance_masks_batch; models are dicts as load_ply returns them."""
    tree = write_tless_checkout(tmp_path)
    code = f"""
        import sys
        sys.path.insert(0, {tree!r})
        sys.path.insert(0, {os.path.join(ROOT, 'tests')!r})
        import numpy as np
        import clean_pvnet_b200 as pvb
        pvb.install_tless_renderer_as_reference()
        from lib.datasets.tless import opengl_renderer, handle_test_data
        from test_gpu_tless_masks import MESHES, W, H, scene
        from tless_mask_cases import LABEL_BG
        B = 3
        mi, obj, img, poses, Ks = scene(B, [4, 1, 6], seed=21)
        models = {{o: {{'pts': p.astype(np.float64), 'faces': f.astype(np.float64)}} for o, (p, f) in zip((3, 17, 30), MESHES)}}
        pose_m = poses.copy()
        pose_m[:, :, 3] *= 0.001                                     # gt.yml's cam_t_m2c * 0.001
        pose_mm = pose_m.copy()
        pose_mm[:, :, 3] = pose_m[:, :, 3] * 1000.                   # as opengl_renderer.render scales it back
        got = [t.cpu().numpy() for t in pvb.instance_masks_batch(MESHES, mi, obj, img, pose_mm, Ks, (W, H))]
        for b in range(B):
            idx = np.flatnonzero(img == b)
            mask_map = np.full((H, W), LABEL_BG, np.int16)
            depth_map = 10 * np.ones((H, W), np.float32)
            for instance_id, i in enumerate(idx):
                depth = opengl_renderer.render(models[obj[i]], pose_m[i], Ks[b], W, H)
                assert depth.dtype == np.float32
                take = (depth != 0) & (depth < depth_map)
                mask_map[take] = obj[i] * 1000 + instance_id
                depth_map[take] = depth[take]
                assert np.sum(depth != 0) == got[1][i]
            assert np.array_equal(mask_map, got[0][b]), b
        print('ok')
    """
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=tree, env=dict(os.environ, PYTHONPATH=ROOT),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout
