"""GPU: the point-average grid (b2v_grid.cu) and the frame preparation (b2v_prep.cu) at their edges, bit for bit.

Grid: against `oracle.numpy_grid` on scenes whose float32 sums are exact in any order (tests/_grid_prep_scenes.py), so
counts, sums, means and every query output must be equal, not close.  Shadow filter: against
`oracle.numpy_shadow_filter`.  remap: against live `cv2.remap`, including NaN map entries (the zero border, as OpenCV's
cvRound sends NaN out of range).  tests/test_grid_prep_oracles_cpu.py pins both oracles to the reference's own outputs
and checks that each scene reaches its case."""

import ctypes as C
import os

import numpy as np
import pytest

import oracle
from pyslam_b200 import B200TsdfVolume, BoundingBox3D, CameraFrustrum, VoxelBlockGrid, filter_shadow_points, remap
from pyslam_b200 import synthetic as S
from tests import _grid_prep_scenes as E
from tests._util import GOLDEN, sort_dump

pytestmark = pytest.mark.gpu
f32 = np.float32


def _rows(p, c):
    a = np.concatenate([p, c], 1)
    return a[np.lexsort(a.T[::-1])]


def _same_voxels(got, ref):
    assert got.points.dtype == np.float32 and len(got.points) == len(ref[0])
    assert np.array_equal(_rows(got.points, got.colors), _rows(*ref))


def _same_dump(grid, G, sums=True):
    d = sort_dump(grid.dump_blocks())
    r = G.dump()
    assert np.array_equal(d["keys"], r["keys"])
    assert np.array_equal(d["count"], r["count"])
    if sums:
        assert np.array_equal(d["pos_sum"], r["pos_sum"]) and np.array_equal(d["col_sum"], r["col_sum"])
    return d


# ---- integrate / get_voxels / remove_low_count_voxels / clear -------------------------------------------------------

def test_exact_scene_counts_sums_and_means_equal_the_oracle():
    grid = VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=1 << 12)
    G = oracle.numpy_grid(E.VS_EXACT)
    for _, p, c in E.exact_batches():
        grid.integrate(p, c)
        G.integrate(p, c)
    _same_dump(grid, G)
    top = int(G.count.max())
    for m in (1, 2, 3, top, top + 1):
        _same_voxels(grid.get_voxels(min_count=m), G.get_voxels(m))
    assert len(grid.get_voxels(min_count=top).points) == 1 and len(grid.get_voxels(min_count=top + 1).points) == 0
    assert grid.size() == int((G.count > 0).sum())
    grid.remove_low_count_voxels(3)
    G.remove_low_count_voxels(3)
    _same_dump(grid, G)
    for m in (1, 3, 4):
        _same_voxels(grid.get_voxels(min_count=m), G.get_voxels(m))
    # a reset voxel starts again from zero; clear forgets every block
    _, p, c = E.exact_batches(seed=5)[3]
    grid.integrate(p, c)
    G.integrate(p, c)
    _same_dump(grid, G)
    _same_voxels(grid.get_voxels(1), G.get_voxels(1))
    grid.clear()
    G.clear()
    assert grid.empty() and grid.size() == 0
    _, p, c = E.exact_batches(seed=6)[3]
    grid.integrate(p, c)
    G.integrate(p, c)
    _same_dump(grid, G)
    _same_voxels(grid.get_voxels(2), G.get_voxels(2))


def test_colour_kinds_uint8_float_and_none():
    """uint8 colours (float32(c) * float32(1/255), non-dyadic) on voxels with at most two points, dyadic float
    colours on the exact scene, and no colours (zero colour sums)."""
    rng = np.random.default_rng(3)
    p = E.edge_points_ref_voxel()
    c8 = rng.integers(0, 256, p.shape, dtype=np.uint8)
    for cols in (c8, None):
        grid = VoxelBlockGrid(E.VS_REF, 8, capacity_blocks=1 << 13)
        G = oracle.numpy_grid(E.VS_REF)
        grid.integrate(p, cols)
        G.integrate(p, cols)
        _same_dump(grid, G)
        _same_voxels(grid.get_voxels(1), G.get_voxels(1))
        _same_voxels(grid.get_voxels(2), G.get_voxels(2))
    _, p, c = E.exact_batches()[3]
    grid = VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=1 << 12)
    G = oracle.numpy_grid(E.VS_EXACT)
    grid.integrate(p)
    G.integrate(p)
    d = _same_dump(grid, G)
    assert not d["col_sum"].any()


def test_voxel_edges_at_the_reference_voxel_size_and_far_keys():
    """0.015 m: points within two float32 ulps of voxel edges, where the float32 product x * inv_vs decides the key;
    keys around +-2^20 at 2^-6 m."""
    for vs, p in ((E.VS_REF, E.edge_points_ref_voxel()), (E.VS_EXACT, E.far_points())):
        grid = VoxelBlockGrid(vs, 8, capacity_blocks=1 << 14)
        G = oracle.numpy_grid(vs)
        cols = np.random.default_rng(1).random(p.shape).astype(f32)
        grid.integrate(p, cols)
        G.integrate(p, cols)
        _same_dump(grid, G)
        _same_voxels(grid.get_voxels(1), G.get_voxels(1))


def test_float64_points_take_the_double_precision_key():
    """float64 points are keyed with floor(x * float64(inv_vs)) and accumulate float32(x); narrowing first would key
    other voxels (test_grid_prep_oracles_cpu checks that the scene differs)."""
    p = E.float64_points()
    for pts in (p, p.astype(f32)):
        grid = VoxelBlockGrid(0.005, 8, capacity_blocks=1 << 15)
        G = oracle.numpy_grid(0.005)
        grid.integrate(pts)
        G.integrate(pts)
        _same_dump(grid, G)
        _same_voxels(grid.get_voxels(1), G.get_voxels(1))


def test_pool_capacity_boundary():
    """Exactly capacity_blocks distinct blocks fit; one more raises "block pool full"."""
    cap = 64
    k = np.stack(np.meshgrid(np.arange(4) - 2, np.arange(4) - 2, np.arange(4) - 2, indexing="ij"), -1).reshape(-1, 3)
    pts = ((k * 8 + 3.5) * E.VS_EXACT).astype(f32)
    grid = VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=cap)
    grid.integrate(pts)
    assert grid.num_blocks() == cap
    G = oracle.numpy_grid(E.VS_EXACT)
    G.integrate(pts)
    _same_dump(grid, G)
    with pytest.raises(RuntimeError, match="block pool full"):
        grid.integrate(np.array([[5 * 8 * E.VS_EXACT, 0, 0]], f32))


# ---- box and frustum queries, carve ---------------------------------------------------------------------------------

@pytest.mark.parametrize("box", range(len(E.BOXES)))
def test_box_query_faces_and_key_bounds(box):
    bb = E.BOXES[box]
    pts = E.box_probe_points(bb)
    cols = E.dyadic_colors(np.random.default_rng(box), len(pts))
    grid = VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=256)
    G = oracle.numpy_grid(E.VS_EXACT)
    grid.integrate(pts, cols)
    G.integrate(pts, cols)
    got = grid.get_voxels_in_bb(BoundingBox3D(*bb), min_count=1)
    _same_voxels(got, G.get_voxels_in_bb(bb))
    assert len(grid.get_voxels_in_bb(BoundingBox3D(*bb), min_count=2).points) == 0


@pytest.mark.parametrize("pose", [0, 1])
def test_frustum_query_bounds(pose):
    T = E.cam_poses()[pose]
    pts = E.frustum_probe_points(T)
    pts = np.concatenate([pts, pts[:20]])          # twenty voxels with count 2 (means unchanged)
    cols = E.dyadic_colors(np.random.default_rng(pose), len(pts))
    grid = VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=256)
    G = oracle.numpy_grid(E.VS_EXACT)
    grid.integrate(pts, cols)
    G.integrate(pts, cols)
    fr = CameraFrustrum(*E.CAM_K, E.CAM_W, E.CAM_H, T, depth_max=E.DEPTH_MAX, depth_min=E.DEPTH_MIN)
    for m in (1, 2):
        got = grid.get_voxels_in_camera_frustrum(fr, min_count=m)
        _same_voxels(got, G.get_voxels_in_frustum(E.CAM_K, E.CAM_W, E.CAM_H, T, E.DEPTH_MAX, E.DEPTH_MIN, m))


@pytest.mark.parametrize("pose", [0, 1])
def test_carve_special_depths_threshold_and_truncation(pose):
    T = E.cam_poses()[pose]
    pts, img = E.carve_scene(T)
    grid = VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=256)
    G = oracle.numpy_grid(E.VS_EXACT)
    grid.integrate(pts)
    G.integrate(pts)
    fr = CameraFrustrum(*E.CAM_K, E.CAM_W, E.CAM_H, T, depth_max=E.DEPTH_MAX, depth_min=E.DEPTH_MIN)
    grid.carve(fr, img, depth_threshold=E.CARVE_THR)
    gone = G.carve(E.CAM_K, E.CAM_W, E.CAM_H, T, img, E.CARVE_THR, E.DEPTH_MAX, E.DEPTH_MIN)
    assert len(gone) >= 10
    _same_dump(grid, G)
    _same_voxels(grid.get_voxels(1), G.get_voxels(1))


# ---- fused RGBD front end -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("flt", [False, True])
def test_integrate_rgbd_exact_scene(flt):
    """integrate_rgbd == numpy_shadow_filter (optionally) + the back-projection in rgbd_point's order + numpy_grid."""
    grid = VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=1 << 12)
    G = oracle.numpy_grid(E.VS_EXACT)
    for d, c, Twc in E.rgbd_frames():
        grid.integrate_rgbd(d, c, E.RGBD_K, Twc, filter_shadow_points=flt)
        dd = oracle.numpy_shadow_filter(d, 2, 2, -1.0)[0] if flt else d
        G.integrate(*E.rgbd_points(dd, c, E.RGBD_K, Twc))
    _same_dump(grid, G)
    _same_voxels(grid.get_voxels(1), G.get_voxels(1))


# ---- shadow filter --------------------------------------------------------------------------------------------------

def _shadow_device(d, dx, dy, fill):
    import torch
    from pyslam_b200 import _lib
    t = torch.from_numpy(np.ascontiguousarray(d)).cuda()
    out = torch.empty_like(t)
    rc = _lib.load().b2v_filter_shadow_points(C.c_void_p(t.data_ptr()), d.shape[0], d.shape[1], dx, dy, float(fill),
                                              C.c_void_p(out.data_ptr()), 0)
    assert rc == _lib.B2V_OK
    return out.cpu().numpy()


@pytest.mark.parametrize("name", list(E.shadow_scenes()))
def test_shadow_filter_edges(name):
    d, dx, dy = E.shadow_scenes()[name]
    ref, _ = oracle.numpy_shadow_filter(d, dx, dy, -1.0)
    got = filter_shadow_points(d, delta_x=dx, delta_y=dy, fill_value=-1)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    got = _shadow_device(d, dx, dy, -1.0)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))


# ---- remap against live OpenCV --------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", E.REMAP_KINDS)
@pytest.mark.parametrize("size", E.REMAP_SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_remap_equals_live_opencv(kind, size):
    cv2 = pytest.importorskip("cv2")
    H, W = size
    rng = np.random.default_rng(H * 1000 + W)
    mx, my = E.remap_maps(kind, H, W, seed=W)
    bgr = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    ref = cv2.remap(bgr, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    assert np.array_equal(remap(bgr, mx, my, "linear"), ref)
    assert np.array_equal(remap(bgr, mx, my, "linear", swap_rb=True), cv2.cvtColor(ref, cv2.COLOR_BGR2RGB))
    depth = rng.uniform(0.1, 5.0, (H, W)).astype(f32)
    got = remap(depth, mx, my, "nearest")
    ref_d = cv2.remap(depth, mx, my, cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    assert np.array_equal(got.view(np.uint32), ref_d.view(np.uint32))
    labels = rng.integers(-2 ** 31, 2 ** 31 - 1, (H, W), dtype=np.int64).astype(np.int32)
    ref_l = cv2.remap(labels, mx, my, cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    assert np.array_equal(remap(labels, mx, my, "nearest"), ref_l)


@pytest.mark.parametrize("raw16", [False, True])
def test_volume_rectification_raw_u16_and_device_inputs(raw16):
    """set_rectification with raw uint16 depth (widened before the remap) or with device (torch CUDA) frames equals the
    volume fed frames pre-rectified with cv2.remap, frame by frame and in fused batches."""
    cv2 = pytest.importorskip("cv2")
    import torch
    g = np.load(os.path.join(GOLDEN, "remap_T0.npz"))
    cfg = S.CONFIGS["T0"]
    K = (float(g["new_K"][0, 0]), float(g["new_K"][1, 1]), float(g["new_K"][0, 2]), float(g["new_K"][1, 2]))
    mx, my = g["map1"], g["map2"]
    n = 5
    frames = [S.render_frame(cfg, i) for i in range(n)]
    scale = f32(0.001)
    raw_u16 = np.stack([np.round(f[0] * 1000).astype(np.uint16) for f in frames])
    raw_d = raw_u16.astype(f32) * scale if raw16 else np.stack([f[0] for f in frames])
    raw_bgr = np.stack([np.ascontiguousarray(f[1][..., ::-1]) for f in frames])
    Ts = np.stack([f[2] for f in frames])
    rect_d = np.stack([cv2.remap(d, mx, my, cv2.INTER_NEAREST) for d in raw_d])
    rect_rgb = np.stack([cv2.cvtColor(cv2.remap(c, mx, my, cv2.INTER_LINEAR), cv2.COLOR_BGR2RGB) for c in raw_bgr])

    def run(batch, rectify):
        vol = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 13)
        if not rectify:
            d, c, kw = rect_d, rect_rgb, {}
        else:
            vol.set_rectification(mx, my, swap_rb=True)
            if raw16:
                d, c, kw = raw_u16, raw_bgr, dict(depth_scale=float(scale))
            else:
                d, c, kw = torch.from_numpy(raw_d).cuda(), torch.from_numpy(raw_bgr).cuda(), {}
        if batch:
            vol.integrate_batch(d, c, K, Ts, **kw)
        else:
            for i in range(n):
                vol.integrate(d[i].contiguous() if torch.is_tensor(d) else d[i],
                              c[i].contiguous() if torch.is_tensor(c) else c[i], K, Ts[i], **kw)
        vol.synchronize()
        out = sort_dump(vol.dump_blocks())
        vol.close()
        return out

    ref = run(False, False)
    assert len(ref["keys"]) > 50
    for batch in (False, True):
        got = run(batch, True)
        assert np.array_equal(got["keys"], ref["keys"]) and np.array_equal(got["vox"], ref["vox"]), batch
