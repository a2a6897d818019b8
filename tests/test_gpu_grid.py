"""GPU: the point-average grid (duck type B) against the UNMODIFIED compiled reference
`volumetric::VoxelBlockGrid` — via the committed golden vectors (tests/golden/refgrid_T0.npz,
produced by oracle/_ref here) and, when oracle/_ref travelled to this box, live.

Bars: block keys, BlockKeyHash, per-voxel counts BIT-EXACT; position / colour sums within
rel 1e-5 * sqrt(count) (float atomics reorder the reference's input-order sums, SURVEY.md §8c);
voxels with count <= 2 are bit-exact (two-term float sums commute)."""

import os

import numpy as np
import pytest

import oracle
from pyslam_b200 import VoxelBlockGrid
from tests._util import GOLDEN, sort_dump

pytestmark = pytest.mark.gpu


def _sum_close(a, b, count):
    tol = 1e-5 * np.sqrt(np.maximum(count, 1))[..., None] * np.maximum(np.abs(b), 1e-3)
    return np.all(np.abs(a - b) <= tol)


def _feed(grid, g):
    start = 0
    for n in g["frame_counts"]:
        grid.integrate(g["points"][start:start + n], g["colors"][start:start + n])
        start += int(n)


def test_golden_reference_vectors():
    g = np.load(os.path.join(GOLDEN, "refgrid_T0.npz"))
    grid = VoxelBlockGrid(float(g["voxel_size"]), 8, capacity_blocks=4096)
    _feed(grid, g)
    d = sort_dump(grid.dump_blocks())
    assert np.array_equal(d["keys"], g["keys"])
    assert np.array_equal(d["hashes"], g["hashes"])
    assert np.array_equal(d["count"], g["count"])
    assert _sum_close(d["pos_sum"], g["pos_sum"], g["count"])
    assert _sum_close(d["col_sum"], g["col_sum"], g["count"])
    few = g["count"] <= 2
    assert np.array_equal(d["pos_sum"][few], g["pos_sum"][few])
    assert np.array_equal(d["col_sum"][few], g["col_sum"][few])
    assert grid.num_blocks() == len(g["keys"])
    assert grid.size() == int((g["count"] > 0).sum()) == grid.get_total_voxel_count()
    assert grid.get_block_size() == 8 and not grid.empty()
    # get_voxels(min_count=2): compare as a set keyed by position order
    out = grid.get_voxels(min_count=2)
    order = np.lexsort((out.points[:, 2], out.points[:, 1], out.points[:, 0]))
    assert out.points.shape == g["voxels_min2_points"].shape
    assert np.allclose(out.points[order], g["voxels_min2_points"], rtol=2e-5, atol=1e-6)
    assert np.allclose(out.colors[order], g["voxels_min2_colors"], rtol=2e-5, atol=1e-6)


@pytest.mark.skipif(not oracle.have_ref(), reason="compiled reference (oracle/_ref) not on this box")
def test_live_against_compiled_reference_with_removal():
    rng = np.random.default_rng(5)
    vs = 0.015  # reference default voxel size (config_parameters.py:311)
    ref = oracle.RefGrid(vs, 8)
    grid = VoxelBlockGrid(vs, 8, capacity_blocks=1 << 14)
    for _ in range(3):
        n = 20000
        # a noisy sphere shell crossing the origin so negative keys are exercised
        dirs = rng.normal(size=(n, 3))
        dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
        pts = (dirs * (0.6 + 0.004 * rng.normal(size=(n, 1))) + [0.1, -0.2, 0.05]).astype(np.float32)
        cols = rng.random((n, 3)).astype(np.float32)
        ref.integrate(pts, cols)
        grid.integrate(pts, cols)
    a, b = sort_dump(grid.dump_blocks()), sort_dump(ref.dump_blocks())
    assert np.array_equal(a["keys"], b["keys"]) and np.array_equal(a["hashes"], b["hashes"])
    assert np.array_equal(a["count"], b["count"])
    assert _sum_close(a["pos_sum"], b["pos_sum"], b["count"])
    assert _sum_close(a["col_sum"], b["col_sum"], b["count"])
    ref.remove_low_count_voxels(3)
    grid.remove_low_count_voxels(3)
    a, b = sort_dump(grid.dump_blocks()), sort_dump(ref.dump_blocks())
    assert np.array_equal(a["count"], b["count"])
    assert grid.size() == int((b["count"] > 0).sum())
    rp, rc = ref.get_voxels(min_count=1)
    out = grid.get_voxels(min_count=1)
    assert len(out.points) == len(rp)
    o1 = np.lexsort((out.points[:, 2], out.points[:, 1], out.points[:, 0]))
    o2 = np.lexsort((rp[:, 2], rp[:, 1], rp[:, 0]))
    assert np.allclose(out.points[o1], rp[o2], rtol=2e-5, atol=1e-6)


def test_argument_checks_and_clear():
    grid = VoxelBlockGrid(0.05, 8, capacity_blocks=256)
    assert grid.empty() and grid.size() == 0
    grid.integrate(np.zeros((0, 3), np.float32))                       # empty input is a no-op
    with pytest.raises(RuntimeError):
        grid.integrate(np.zeros((4, 2), np.float32))                   # shape[1] must be 3
    with pytest.raises(RuntimeError):
        grid.integrate(np.zeros((4, 3), np.float32), np.zeros((3, 3), np.float32))
    with pytest.raises(RuntimeError):
        grid.integrate(np.zeros((4, 3), np.int32))
    pts = np.array([[0.01, 0.02, 0.03], [0.01, 0.02, 0.03], [-0.01, 0.5, 1.2]], np.float32)
    grid.integrate(pts, np.array([[255, 0, 0], [255, 0, 0], [0, 255, 0]], np.uint8))
    assert grid.num_blocks() == 2 and grid.size() == 2
    out = grid.get_voxels(min_count=2)
    assert len(out.points) == 1 and np.allclose(out.points[0], pts[0])
    assert np.allclose(out.colors[0], [1.0, 0.0, 0.0], atol=1e-6)
    grid.clear()
    assert grid.empty() and grid.size() == 0 and len(grid.get_points()) == 0
    with pytest.raises(RuntimeError):
        VoxelBlockGrid(0.05, 4)


def test_uint8_colors_scaled_on_device_like_voxel_data():
    """uint8 colours go to the device as bytes and are scaled there by the float32 constant 1/255
    (voxel_data.h:79-97): the result must be bit-identical to feeding float32(c) * float32(1/255)."""
    rng = np.random.default_rng(5)
    pts = rng.uniform(-1.0, 1.0, (20000, 3))
    cols = rng.integers(0, 256, (20000, 3), dtype=np.uint8)
    a = VoxelBlockGrid(0.05, 8, capacity_blocks=8192)
    b = VoxelBlockGrid(0.05, 8, capacity_blocks=8192)
    for dt in (np.float32, np.float64):
        a.clear(); b.clear()
        a.integrate(pts.astype(dt), cols)
        b.integrate(pts.astype(dt), cols.astype(np.float32) * (np.float32(1.0) / np.float32(255.0)))
        va, vb = a.get_voxels(), b.get_voxels()
        oa = np.lexsort((va.points[:, 2], va.points[:, 1], va.points[:, 0]))
        ob = np.lexsort((vb.points[:, 2], vb.points[:, 1], vb.points[:, 0]))
        assert len(oa) == len(ob) > 1000
        # float atomics: the per-voxel summation order differs between two runs, not the addends
        assert np.allclose(va.points[oa], vb.points[ob], rtol=0, atol=2e-6)
        assert np.allclose(va.colors[oa], vb.colors[ob], rtol=0, atol=2e-6)


def _sorted_pts(p):
    return p[np.lexsort((p[:, 2], p[:, 1], p[:, 0]))]


def test_spatial_queries_and_carve_match_reference_golden():
    """get_voxels_in_camera_frustrum / get_voxels_in_bb / carve against the UNMODIFIED reference's
    outputs (tests/golden/refgrid_T0.npz) on a real scene, where float atomics may move a voxel mean by an ulp: the
    selected sets are compared with a small allowance, positions to 2e-5.  test_gpu_grid_prep_edges.py pins the
    queries and the carve exactly, on scenes whose sums are exact in any order."""
    from pyslam_b200 import BoundingBox3D, CameraFrustrum
    g = np.load(os.path.join(GOLDEN, "refgrid_T0.npz"))
    grid = VoxelBlockGrid(float(g["voxel_size"]), 8, capacity_blocks=4096)
    _feed(grid, g)
    K = g["query_K"]
    H, W = g["query_depth"].shape
    fr = CameraFrustrum(K[0], K[1], K[2], K[3], W, H, g["query_Tcw"], depth_max=3.0, depth_min=0.05)
    out = grid.get_voxels_in_camera_frustrum(fr, min_count=1)
    ref = g["frustum_points"]
    assert abs(len(out.points) - len(ref)) <= max(2, 0.002 * len(ref)) and len(ref) > 1000
    if len(out.points) == len(ref):
        assert np.allclose(_sorted_pts(out.points), ref, rtol=2e-5, atol=1e-6)
    bb = grid.get_voxels_in_bb(BoundingBox3D(*g["query_bbox"]), min_count=1)
    refb = g["bbox_points"]
    assert abs(len(bb.points) - len(refb)) <= max(2, 0.002 * len(refb)) and len(refb) > 100
    if len(bb.points) == len(refb):
        assert np.allclose(_sorted_pts(bb.points), refb, rtol=2e-5, atol=1e-6)
    grid.carve(fr, g["query_depth"], depth_threshold=0.05)
    d = sort_dump(grid.dump_blocks())
    ref_c = g["carved_count"]
    assert (g["count"] > 0).sum() - (ref_c > 0).sum() > 100          # the carve removed something
    mism = int(((d["count"] > 0) != (ref_c > 0)).sum())
    assert mism <= max(2, 0.002 * int((ref_c > 0).sum())), mism
    # a wrongly sized depth image is a soft failure (voxel_grid_carving.h:51-58): nothing changes
    grid.carve(fr, g["query_depth"][:10], depth_threshold=0.05)
    assert np.array_equal(sort_dump(grid.dump_blocks())["count"], d["count"])


def test_fused_rgbd_front_end_equals_reference_pipeline():
    """integrate_rgbd(depth, color, K, Twc) == the reference front-end (depth2pointcloud + Twc transform
    in float64 -> float32) followed by the reference grid: keys / hashes / counts bit-exact vs the golden
    dump of the compiled reference, sums within the atomic-order tolerance."""
    from pyslam_b200 import synthetic as S
    g = np.load(os.path.join(GOLDEN, "refgrid_T0.npz"))
    t = np.load(os.path.join(GOLDEN, "tsdf_T0.npz"))
    grid = VoxelBlockGrid(float(g["voxel_size"]), 8, capacity_blocks=4096)
    for i in range(len(g["frame_counts"])):
        grid.integrate_rgbd(t["depth"][i], t["color"][i], t["K"], S.inv_T(t["Tcw"][i]),
                            max_depth=float(t["depth_trunc"]))
    d = sort_dump(grid.dump_blocks())
    assert np.array_equal(d["keys"], g["keys"]) and np.array_equal(d["hashes"], g["hashes"])
    assert np.array_equal(d["count"], g["count"])
    assert _sum_close(d["pos_sum"], g["pos_sum"], g["count"])
    assert _sum_close(d["col_sum"], g["col_sum"], g["count"])
    one = g["count"] == 1
    assert np.array_equal(d["pos_sum"][one], g["pos_sum"][one])   # single-sample voxels: the point itself
    assert np.array_equal(d["col_sum"][one], g["col_sum"][one])


def test_front_end_rows_match_the_reference_python_functions():
    """tests/golden/frontend_T0.npz holds outputs of the reference's OWN `filter_shadow_points` and
    `depth2pointcloud` (pyslam/utilities/depth.py, imported unmodified by make_golden_frontend.py) and of the
    compiled reference grid fed those points.  The GPU shadow filter must reproduce the filtered depth image
    exactly; the fused RGBD path must reproduce block keys / hashes / counts exactly, sums to tolerance."""
    from pyslam_b200 import filter_shadow_points
    from pyslam_b200 import synthetic as S
    g = np.load(os.path.join(GOLDEN, "frontend_T0.npz"))
    n = g["depth"].shape[0]
    for i in range(n):
        out = filter_shadow_points(g["depth"][i])
        assert np.array_equal(out, g[f"filtered_{i}"]), i
        assert (out != g["depth"][i]).sum() > 100
    for tag, flt in (("nf", False), ("f", True)):
        grid = VoxelBlockGrid(float(g["voxel_size"]), 8, capacity_blocks=4096)
        for i in range(n):
            grid.integrate_rgbd(g["depth"][i], g["color"][i], g["K"], S.inv_T(g["Tcw"][i]),
                                max_depth=float(g["max_depth"]), filter_shadow_points=flt)
        d = sort_dump(grid.dump_blocks())
        assert np.array_equal(d["keys"], g[f"{tag}_keys"]) and np.array_equal(d["hashes"], g[f"{tag}_hashes"])
        mism = int((d["count"] != g[f"{tag}_count"]).sum())
        # the reference multiplies with BLAS (inv_pose @ points.T): a point may land one ulp away and cross a
        # voxel boundary; allow a handful of such voxels out of ~12 000
        assert mism <= 6, mism
        same = d["count"] == g[f"{tag}_count"]
        assert _sum_close(d["pos_sum"][same], g[f"{tag}_pos_sum"][same], g[f"{tag}_count"][same])
        assert _sum_close(d["col_sum"][same], g[f"{tag}_col_sum"][same], g[f"{tag}_count"][same])


@pytest.mark.skipif(not oracle.have_ref(), reason="compiled reference (oracle/_ref) not built")
def test_float64_points_take_the_double_precision_key_like_the_reference():
    """integrate(points float64): the reference's float64 overload keys voxels with floor(x * (double)inv_vs) and
    accumulates float32(x) (volumetric_grid_module.h:737-749, voxel_data.h:53-57).  Points are placed within float32
    rounding of voxel boundaries, where narrowing first would pick the neighbouring voxel."""
    rng = np.random.default_rng(7)
    vs = 0.005
    k = rng.integers(-400, 400, size=(20000, 3)).astype(np.float64)
    pts = k * (1.0 / (np.float32(1.0) / np.float32(vs)).astype(np.float64)) + rng.choice([-1e-9, 1e-9, 3e-10], size=(20000, 3))
    cols = rng.random((20000, 3)).astype(np.float32)
    g = VoxelBlockGrid(vs, 8, capacity_blocks=1 << 15)
    r = oracle.RefGrid(vs, 8)
    g.integrate(pts, cols)
    r.integrate(pts, cols)
    a, b = sort_dump(g.dump_blocks()), sort_dump(r.dump_blocks())
    assert np.array_equal(a["keys"], b["keys"]) and np.array_equal(a["count"], b["count"])
    narrow = VoxelBlockGrid(vs, 8, capacity_blocks=1 << 15)
    narrow.integrate(pts.astype(np.float32), cols)
    assert not np.array_equal(sort_dump(narrow.dump_blocks())["count"], b["count"])   # the case is not vacuous
    one = b["count"] == 1
    assert np.array_equal(a["pos_sum"][one], b["pos_sum"][one])
    assert np.allclose(a["pos_sum"], b["pos_sum"], rtol=1e-5, atol=1e-5)
