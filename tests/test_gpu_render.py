"""GPU tests of T-LESS's VSD layer (DESIGN.md 8f): the depth rasterizer against the fp64 ray-casting oracle
(oracle/render_oracle.c), its watertightness and determinism, the VSD kernel against the numpy restatement of the
reference (tests/vsd_cases.py, itself pinned to the reference's vsd_utils by tests/golden/vsd.npz), the batched T-LESS
tail pnp_batch -> vsd_batch -> flags, the OpenGL drop-in, and stream / sync behaviour."""
import numpy as np
import pytest
import torch

import render_oracle
from vsd_cases import (CLOSED, K_SMALL, K_TLESS, MESHES, THRESHOLD, box, poses, vsd_metric_restated, vsd_restated)

pytestmark = pytest.mark.gpu

SIZES = {"720x540": ((720, 540), K_TLESS), "128x128": ((128, 128), K_SMALL)}
# pixels the comparison with the oracle leaves out: within EDGE_PX of a projected edge of a triangle that could take the
# pixel, where the two nearest hits are within GAP_MM, or where a hit is within GAP_MM of a clip plane.  Their count is
# bounded by EXCLUDED_MAX of the covered pixels plus BAND_FACTOR times the area of the EDGE_PX-wide band around every
# projected edge (2 * EDGE_PX * total edge length, in pixels): a mesh with many triangles per pixel puts more pixel
# centres near an edge, and the factor covers the band's ends and both triangles of a shared edge.
EDGE_PX, GAP_MM, REL_TOL, EXCLUDED_MAX, BAND_FACTOR = 1e-3, 1e-3, 1e-5, 0.02, 4
_mesh_cache = {}


@pytest.fixture(scope="module", autouse=True)
def _oracle():
    render_oracle.build()


def mesh(name):
    if name not in _mesh_cache:
        _mesh_cache[name] = MESHES[name]()
    return _mesh_cache[name]


def per_pose_k(K, n, seed):
    rng = np.random.default_rng(seed)
    Ks = np.repeat(K[None], n, 0).copy()
    Ks[:, 0, 0] *= rng.uniform(0.9, 1.1, n)
    Ks[:, 1, 1] *= rng.uniform(0.9, 1.1, n)
    Ks[:, 0, 2] += rng.uniform(-5, 5, n)
    Ks[:, 1, 2] += rng.uniform(-5, 5, n)
    Ks[:, 0, 1] = rng.uniform(-2, 2, n)                       # a skew, which _compute_calib_proj honours
    return Ks


def edge_band_px(v, f, pose, K):
    """2 * EDGE_PX * the summed projected length of the edges of the triangles in front of the camera."""
    P = v.astype(np.float64) @ pose[:, :3].T + pose[:, 3]
    front = np.all(P[f][:, :, 2] > 0, axis=1)
    q = P @ K.T
    uv = q[:, :2] / np.where(q[:, 2:] > 0, q[:, 2:], 1.0)
    t = uv[f[front]]
    length = sum(np.linalg.norm(t[:, j] - t[:, (j + 1) % 3], axis=1).sum() for j in range(3))
    return 2 * EDGE_PX * length


def compare_with_oracle(dev_depth, v, f, pose, K, size, label):
    o = render_oracle.render_depth(v, f, pose, K, size)
    z, d = o["z"], dev_depth.astype(np.float64)
    ok = (o["edge"] > EDGE_PX) & (o["gap"] > GAP_MM) & (o["clip"] > GAP_MM)
    covered = (z > 0) | (d > 0)
    excluded = int((covered & ~ok).sum())
    assert np.array_equal((d > 0)[ok], (z > 0)[ok]), f"{label}: hit / background disagree at {int(((d > 0) != (z > 0))[ok].sum())} px"
    hit = ok & (z > 0)
    rel = float((np.abs(d[hit] - z[hit]) / z[hit]).max()) if hit.any() else 0.0
    bound = EXCLUDED_MAX * int(covered.sum()) + BAND_FACTOR * edge_band_px(v, f, pose, K)
    print(f"[render] {label}: {int(hit.sum())} px compared, max rel {rel:.2e}, {excluded} of {int(covered.sum())} "
          f"covered px excluded (bound {bound:.0f})")
    assert rel <= REL_TOL
    assert excluded <= bound
    return z


@pytest.mark.parametrize("per_k", [False, True], ids=["sharedK", "poseK"])
@pytest.mark.parametrize("n", [1, 16, 256])
@pytest.mark.parametrize("size", list(SIZES))
@pytest.mark.parametrize("name", list(MESHES))
def test_depth_matches_the_oracle(pvb, name, size, n, per_k):
    v, f = mesh(name)
    wh, K = SIZES[size]
    P = poses(n, seed=n * 7 + len(name))
    Ks = per_pose_k(K, n, seed=n) if per_k else K
    depth = pvb.render_depth_batch(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(P).cuda(),
                                   torch.from_numpy(np.asarray(Ks)).cuda(), wh)
    assert depth.shape == (n, wh[1], wh[0]) and depth.dtype == torch.float32
    d = depth.cpu().numpy()
    for i in sorted({0, n - 1}):
        compare_with_oracle(d[i], v, f, P[i], Ks[i] if per_k else K, wh, f"{name} {size} n={n} pose {i}")


@pytest.mark.parametrize("name", CLOSED)
def test_closed_meshes_are_watertight_at_random_poses(pvb, name):
    """Every pixel the oracle covers, away from the silhouette (where entry and exit hits differ by > GAP_MM), is covered."""
    v, f = mesh(name)
    P = poses(200, seed=99)
    d = pvb.render_depth_batch(v, f, P, K_TLESS, (720, 540)).cpu().numpy()
    holes = 0
    for i in range(200):
        o = render_oracle.render_depth(v, f, P[i], K_TLESS, (720, 540))
        holes += int(((o["z"] > 0) & (o["gap"] > GAP_MM) & (d[i] == 0)).sum())
    assert holes == 0


def test_edges_and_vertices_exactly_on_pixel_centres_leave_no_crack(pvb):
    """A plane at Z = 1024 seen with fx = fy = 1024 and cx = cy = 0.5: grid vertex (X, Y) projects exactly to the pixel
    centre (X + 0.5, Y + 0.5), so every vertical, horizontal and diagonal edge passes exactly through pixel centres and
    every vertex sits on one.  Both diagonal directions and both windings are used; no pixel may read 0."""
    K = np.array([[1024.0, 0, 0.5], [0, 1024.0, 0.5], [0, 0, 1]])
    xs = np.arange(-2, 70, 4.0)
    V = np.array([[x, y, 0.0] for y in xs for x in xs], np.float32)
    m = len(xs)
    F = []
    for j in range(m - 1):
        for i in range(m - 1):
            a, b, c, d = j * m + i, j * m + i + 1, (j + 1) * m + i + 1, (j + 1) * m + i
            F += [[a, b, c], [a, d, c]] if (i + j) % 2 else [[a, b, d], [b, c, d]]
    pose = np.hstack([np.eye(3), [[0], [0], [1024.0]]])[None]
    d = pvb.render_depth_batch(V, np.array(F, np.int32), pose, K, (64, 64), near=100, far=10000).cpu().numpy()[0]
    assert np.all(d == 1024.0)


def test_outputs_are_deterministic_and_batch_independent(pvb):
    v, f = mesh("torus")
    P = poses(256, seed=5)
    a = pvb.render_depth_batch(v, f, P, K_TLESS, (720, 540))
    b = pvb.render_depth_batch(v, f, P, K_TLESS, (720, 540))
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    for i in (0, 77, 255):
        alone = pvb.render_depth_batch(v, f, P[i:i + 1], K_TLESS, (720, 540))
        assert torch.equal(alone[0].view(torch.int32), a[i].view(torch.int32))


def test_clipping_near_far_and_behind_the_camera(pvb):
    v, f = box(300.0, 300.0, 300.0)
    P = np.stack([np.hstack([np.eye(3), [[0], [0], [z]]]) for z in (-2000.0, 150.0, 12000.0)])
    d = pvb.render_depth_batch(v, f, P, K_TLESS, (720, 540)).cpu().numpy()
    assert not d[0].any() and not d[2].any()                   # behind the camera; beyond far
    compare_with_oracle(d[1], v, f, P[1], K_TLESS, (720, 540), "box around the near plane")
    assert d[1].any()


def _scene(pvb, name, B, ng_per, ne_per, seed, size=(720, 540), K=K_TLESS):
    """B test images, each the render of ng_per ground-truth poses plus noise and an occluding band, and ne_per estimates
    per image near its ground truths (some far off).  Returns device tensors and the (est, gt, image) rows of every pair."""
    v, f = mesh(name)
    rng = np.random.default_rng(seed)
    pg = poses(B * ng_per, seed=seed)
    pe = np.repeat(pg, ne_per // ng_per, 0)[:B * ne_per].copy()
    pe[:, :, 3] += rng.normal(0, 6, (len(pe), 3)) * rng.choice([0.3, 1, 4], (len(pe), 1))
    gt_depth = pvb.render_depth_batch(v, f, pg, K, size).cpu().numpy()
    tests = []
    for b in range(B):
        d = gt_depth[b * ng_per:(b + 1) * ng_per]
        d = np.where(d > 0, d, np.inf).min(0)
        d = np.where(np.isfinite(d), d, 1200.0).astype(np.float32)
        d = np.round((d + rng.normal(0, 2, d.shape)) * 10) / 10                # a uint16 depth image * 0.1
        d[:, 300:330] = 500.0                                                  # an occluder
        d[rng.random(d.shape) < 0.05] = 0                                      # missing depth
        tests.append(d.astype(np.float32))
    rows = [(e, g, b) for b in range(B) for e in range(b * ne_per, (b + 1) * ne_per)
            for g in range(b * ng_per, (b + 1) * ng_per)]
    return v, f, pe, pg, np.stack(tests), np.array(rows, np.int32)


@pytest.mark.parametrize("npairs", [16, 256])
def test_vsd_equals_the_restatement_bit_for_bit(pvb, npairs):
    B, ng_per = (2, 2) if npairs == 16 else (4, 4)
    ne_per = npairs // B // ng_per
    v, f, pe, pg, dt, rows = _scene(pvb, "icosphere", B, ng_per, ne_per, seed=npairs)
    e = pvb.vsd_batch(v, f, torch.from_numpy(pe).cuda(), torch.from_numpy(pg).cuda(), K_TLESS,
                      torch.from_numpy(dt).cuda(), torch.from_numpy(rows).cuda()).cpu().numpy()
    de = pvb.render_depth_batch(v, f, pe, K_TLESS, (720, 540)).cpu().numpy()
    dg = pvb.render_depth_batch(v, f, pg, K_TLESS, (720, 540)).cpu().numpy()
    want = np.array([vsd_restated(de[i], dg[j], dt[b], K_TLESS) for i, j, b in rows])
    assert len(e) == npairs and np.array_equal(e, want), np.abs(e - want).max()
    assert (want < THRESHOLD).any() and (want >= THRESHOLD).any()
    # the T-LESS flags on the oracle's depth, wherever no row of the image is within 0.01 of the threshold
    zo = {}
    for i in set(rows[:, 0]):
        zo[("e", i)] = render_oracle.render_depth(v, f, pe[i], K_TLESS, (720, 540))["z"].astype(np.float32)
    for j in set(rows[:, 1]):
        zo[("g", j)] = render_oracle.render_depth(v, f, pg[j], K_TLESS, (720, 540))["z"].astype(np.float32)
    eo = np.array([vsd_restated(zo[("e", i)], zo[("g", j)], dt[b], K_TLESS) for i, j, b in rows])
    decided = 0
    for b in range(B):
        r = rows[:, 2] == b
        if np.all(np.abs(eo[r] - THRESHOLD) > 0.01):
            assert (e[r] < THRESHOLD).any() == (eo[r] < THRESHOLD).any()
            decided += 1
    print(f"[vsd] {npairs} rows: max |e_device_depth - e_oracle_depth| = {np.abs(e - eo).max():.4f}; "
          f"{decided} of {B} image flags compared")


def test_vsd_windows_and_per_image_K(pvb):
    """Rendering in windows (a small max_render_bytes) and a K per image give the same e as one window."""
    v, f, pe, pg, dt, rows = _scene(pvb, "torus", 2, 2, 4, seed=3, size=(128, 128), K=K_SMALL)
    Ks = np.stack([K_SMALL, K_SMALL * np.array([[1.02, 0, 1], [0, 1.01, 1], [0, 0, 1]])])
    args = (v, f, torch.from_numpy(pe).cuda(), torch.from_numpy(pg).cuda(), torch.from_numpy(Ks).cuda(),
            torch.from_numpy(dt).cuda(), torch.from_numpy(rows).cuda())
    one = pvb.vsd_batch(*args)
    win = pvb.vsd_batch(*args, max_render_bytes=3 * 128 * 128 * 4)
    assert torch.equal(one, win)
    de = [pvb.render_depth_batch(v, f, pe[i:i + 1], Ks[b], (128, 128)).cpu().numpy()[0] for i, _, b in rows]
    dg = [pvb.render_depth_batch(v, f, pg[j:j + 1], Ks[b], (128, 128)).cpu().numpy()[0] for _, j, b in rows]
    want = np.array([vsd_restated(de[k], dg[k], dt[b], Ks[b]) for k, (_, _, b) in enumerate(rows)])
    assert np.array_equal(one.cpu().numpy(), want)
    bad = torch.from_numpy(np.array([[0, 0, 0], [99, 0, 0], [0, 0, 7]], np.int32)).cuda()
    e = pvb.vsd_batch(v, f, args[2], args[3], args[4], args[5], bad).cpu().numpy()
    assert np.isfinite(e[0]) and np.isnan(e[1]) and np.isnan(e[2])


def test_tless_tail_pnp_to_vsd_flags(pvb):
    """pnp_batch -> vsd_batch -> any-of per image, against a per-image loop of the restated Evaluator.vsd_metric."""
    v, f, _, pg, dt, _ = _scene(pvb, "torus", 3, 1, 1, seed=11)
    rng = np.random.default_rng(11)
    kpt_3d = np.concatenate([v[rng.choice(len(v), 8, replace=False)], v.mean(0, keepdims=True)]).astype(np.float64)
    n_est = 2
    pose_true = np.repeat(pg, n_est, 0)
    uv = []
    for p in pose_true:
        x = kpt_3d @ p[:, :3].T + p[:, 3]
        q = x @ K_TLESS.T
        uv.append(q[:, :2] / q[:, 2:] + rng.normal(0, rng.choice([0.2, 8.0]), (len(kpt_3d), 2)))
    pe = pvb.pnp_batch(kpt_3d, torch.from_numpy(np.array(uv)).cuda(), K_TLESS)
    rows = torch.from_numpy(np.array([(i, i // n_est, i // n_est) for i in range(len(pe))], np.int32)).cuda()
    e = pvb.vsd_batch(v, f, pe, torch.from_numpy(pg).cuda(), K_TLESS, torch.from_numpy(dt).cuda(), rows)
    flags = torch.zeros(3, dtype=torch.int64, device="cuda").scatter_reduce_(0, rows[:, 2].long(),
                                                                              (e < THRESHOLD).long(), "amax")
    pe_h = pe.cpu().numpy()
    depth_of = lambda p: pvb.render_depth_batch(v, f, p[None], K_TLESS, (720, 540)).cpu().numpy()[0]   # noqa: E731
    want = [vsd_metric_restated(depth_of, pe_h[b * n_est:(b + 1) * n_est], pg[b:b + 1], K_TLESS, dt[b]) for b in range(3)]
    assert flags.cpu().tolist() == want


def test_dropin_depth_render_equals_the_batch(pvb):
    v, f = mesh("icosphere")
    P = poses(3, seed=4)
    r = pvb.render.DepthRender({"pts": v, "faces": f}, (720, 540))
    got = r.render((720, 540), 100, 10000, K_TLESS, P[1][:, :3], P[1][:, 3:])
    assert got.dtype == np.float32 and got.shape == (540, 720)
    assert np.array_equal(got, pvb.render_depth_batch(v, f, P, K_TLESS, (720, 540)).cpu().numpy()[1])
    assert np.array_equal(pvb.render.render({"pts": v, "faces": f}, (720, 540), K_TLESS, P[1][:, :3], P[1][:, 3:],
                                            clip_near=100, clip_far=10000, mode="depth"), got)


def test_no_host_sync_and_side_stream(pvb):
    v, f, pe, pg, dt, rows = _scene(pvb, "box", 2, 1, 2, seed=8)
    args = [torch.from_numpy(a).cuda() for a in (v, f, pe, pg, K_TLESS, dt, rows)]
    ref = pvb.vsd_batch(*args)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        e = pvb.vsd_batch(*args)
        d = pvb.render_depth_batch(args[0], args[1], args[3], args[4], (720, 540))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        e2 = pvb.vsd_batch(*args)
        d2 = pvb.render_depth_batch(args[0], args[1], args[3], args[4], (720, 540))
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(e, ref) and torch.equal(e2, ref) and torch.equal(d, d2)
