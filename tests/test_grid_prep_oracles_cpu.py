"""CPU: the numpy oracles of the point-average grid and the shadow filter reproduce the reference's own outputs bit for
bit, and every edge scene of tests/test_gpu_grid_prep_edges.py reaches the case it is built for (a scene that stops
reaching its edge fails here instead of passing vacuously on the GPU)."""

import os

import numpy as np
import pytest

import oracle
from tests import _grid_prep_scenes as E
from tests._util import GOLDEN

f32 = np.float32


def _rows(p, c=None):
    a = p if c is None else np.concatenate([p, c], 1)
    return a[np.lexsort(a.T[::-1])]


# ---- the oracles against the goldens --------------------------------------------------------------------------------

def test_numpy_grid_reproduces_the_reference_golden():
    """refgrid_T0.npz holds the compiled reference grid's own outputs: the restatement must equal all of them."""
    g = np.load(os.path.join(GOLDEN, "refgrid_T0.npz"))
    G = oracle.numpy_grid(float(g["voxel_size"]))
    start = 0
    for n in g["frame_counts"]:
        G.integrate(g["points"][start:start + n], g["colors"][start:start + n])
        start += int(n)
    d = G.dump()
    for k in ("keys", "count", "pos_sum", "col_sum"):
        assert np.array_equal(d[k], g[k]), k
    p, c = G.get_voxels(2)
    o = np.lexsort((p[:, 2], p[:, 1], p[:, 0]))
    assert np.array_equal(p[o], g["voxels_min2_points"]) and np.array_equal(c[o], g["voxels_min2_colors"])
    bp, _ = G.get_voxels_in_bb(g["query_bbox"])
    assert len(bp) == 2458 and np.array_equal(_rows(bp), g["bbox_points"])
    H, W = g["query_depth"].shape
    fp, _ = G.get_voxels_in_frustum(g["query_K"], W, H, g["query_Tcw"], depth_max=3.0, depth_min=0.05)
    assert len(fp) == 5455 and np.array_equal(_rows(fp), g["frustum_points"])
    gone = G.carve(g["query_K"], W, H, g["query_Tcw"], g["query_depth"], 0.05, depth_max=3.0, depth_min=0.05)
    assert len(gone) == 5354 and np.array_equal(G.dump()["count"], g["carved_count"])


def test_numpy_shadow_filter_reproduces_the_reference_function():
    """frontend_T0.npz holds the reference's own filter_shadow_points outputs for three frames."""
    g = np.load(os.path.join(GOLDEN, "frontend_T0.npz"))
    for i in range(3):
        out, thr = oracle.numpy_shadow_filter(g["depth"][i])
        assert out.dtype == np.float32 and thr.dtype == np.float32
        assert np.array_equal(out.view(np.uint32), g[f"filtered_{i}"].view(np.uint32)), i


def test_numpy_grid_float64_key_rule():
    """float64 points: floor(x * float64(inv_vs)), sums of float32(x); the float32 overload keys the narrowed value."""
    p = E.float64_points()
    G64, G32 = oracle.numpy_grid(0.005), oracle.numpy_grid(0.005)
    G64.integrate(p)
    G32.integrate(p.astype(f32))
    assert not np.array_equal(G64.keys, G32.keys)
    k = np.floor(p * np.float64(f32(1) / f32(0.005))).astype(np.int64)
    assert np.array_equal(G64.keys, np.unique(k, axis=0))
    _, idx, cnt = np.unique(k, axis=0, return_index=True, return_counts=True)
    assert np.array_equal(G64.pos[cnt == 1], p[idx[cnt == 1]].astype(f32))   # the sum holds float32(x)


# ---- census: each scene reaches its case ----------------------------------------------------------------------------

def test_exact_scenes_reach_their_cases():
    batches = dict((n, p) for n, p, _ in E.exact_batches())
    inv = f32(64)
    vk = {n: np.floor(p * inv).astype(np.int64) for n, p in batches.items()}
    assert len(np.unique(vk["warp_one_block"][:32] // 8, axis=0)) == 1
    assert len(np.unique(vk["warp_one_block"][:32], axis=0)) > 8
    blk = vk["alternating"] // 8
    assert len(np.unique(blk, axis=0)) == 2 and np.all(np.any(blk[0::2] != blk[1::2], axis=1))
    assert np.all(blk[0::2] == blk[0]) and np.all(blk[1::2] == blk[1])
    assert len(np.unique(vk["full_block"], axis=0)) == 512 and np.all(vk["full_block"] // 8 == -1)
    allk = np.concatenate(list(vk.values()))
    assert (allk < 0).any() and (allk > 0).any() and np.any((allk < 0).any(1) & (allk > 0).any(1))
    counts = E.voxel_counts(allk)
    assert counts.max() == 300 and (counts == 1).any() and (counts == 2).any() and counts.max() <= 2 ** 9
    assert np.all(np.abs(np.concatenate(list(batches.values()))) < 8)
    for p in batches.values():                                   # few significant bits: exact float32 sums
        assert np.all(p / E.Q == np.round(p / E.Q))


def test_far_and_rounding_scenes_reach_their_cases():
    far = E.far_points()
    k = np.floor(far * f32(64)).astype(np.int64)
    assert np.abs(k).min() > 2 ** 20 - 64 and (k < 0).any() and (k > 0).any()
    assert E.voxel_counts(k).max() <= 2
    ref = E.edge_points_ref_voxel()
    assert E.product_rounding_crossings(ref, E.VS_REF) > 50        # float32 product rounding crosses a voxel edge
    assert ((ref != 0) & (np.abs(ref) < np.finfo(f32).tiny)).any()  # sub-normal coordinates next to the edge at 0
    kr = np.floor(ref * (f32(1) / f32(E.VS_REF))).astype(np.int64)
    assert E.voxel_counts(kr).max() == 2
    p64 = E.float64_points()
    inv = f32(1) / f32(0.005)
    k64 = np.floor(p64 * np.float64(inv))
    k32 = np.floor(p64.astype(f32) * inv)
    assert (k64 != k32).sum() > 100                                # narrowing first would change the key
    assert E.voxel_counts(k64.astype(np.int64)).max() <= 2


@pytest.mark.parametrize("box", range(len(E.BOXES)))
def test_box_scenes_reach_their_faces(box):
    bb = E.BOXES[box]
    pts = E.box_probe_points(bb)
    k = np.floor(pts * f32(64)).astype(np.int64)
    assert len(np.unique(k, axis=0)) == len(k)                    # one point per voxel: the mean is the point
    c = E.box_census(pts, bb)
    assert min(c["on_min_face"]) > 0 and min(c["on_max_face"]) > 0 and c["outside_keys"] >= 6
    if box == 0:
        assert all(c["min_key_not_block_edge"])
    else:
        assert all(c["min_key_negative_block_edge"])
    G = oracle.numpy_grid(E.VS_EXACT)
    G.integrate(pts)
    p, _ = G.get_voxels_in_bb(bb)
    q = p.astype(np.float64)
    assert ((q == bb[:3]).any(0)).all() and ((q == bb[3:]).any(0)).all()    # faces are inclusive
    assert 0 < len(p) < len(pts)
    lo = np.floor(bb[:3] * 64)
    kin = np.floor(p * f32(64))
    if box == 0:   # selected voxels below the first block edge above the min key (-16 < k < -8 on x)
        assert np.any((kin[:, 0] >= lo[0]) & (kin[:, 0] < np.ceil(lo[0] / 8) * 8))


@pytest.mark.parametrize("pose", [0, 1])
def test_frustum_scene_reaches_its_bounds(pose):
    T = E.cam_poses()[pose]
    pts = E.frustum_probe_points(T)
    k = np.floor(pts * f32(64)).astype(np.int64)
    assert len(np.unique(k, axis=0)) == len(k)
    c = E.frustum_census(pts, T)
    assert c["u0_in"] and c["uW"] and c["vH"] and c["dmin_in"] and c["dmax_in"] and c["behind"] >= 2
    assert 40 <= c["inside"] < len(pts)


@pytest.mark.parametrize("pose", [0, 1])
def test_carve_scene_reaches_its_branches(pose):
    T = E.cam_poses()[pose]
    pts, img = E.carve_scene(T)
    k = np.floor(pts * f32(64)).astype(np.int64)
    assert len(np.unique(k, axis=0)) == len(k)
    c = E.carve_census(pts, img, T)
    assert c["at_threshold"] >= 1 and c["ulp_nearer"] >= 1
    assert c["nan"] == 1 and c["posinf"] == 1 and c["neginf"] == 1 and c["special"] >= 5
    assert c["truncation_matters"] >= 1 and c["last_column"] >= 1 and c["carved"] >= 10
    G = oracle.numpy_grid(E.VS_EXACT)
    G.integrate(pts)
    gone = G.carve(E.CAM_K, E.CAM_W, E.CAM_H, T, img, E.CARVE_THR, E.DEPTH_MAX, E.DEPTH_MIN)
    assert 10 <= len(gone) < len(pts)


def test_rgbd_scene_is_exact_and_the_filter_bites():
    for d, c, Twc in E.rgbd_frames():
        p, col = E.rgbd_points(d, c, E.RGBD_K, Twc)
        assert np.all(p / E.Q == np.round(p / E.Q)) and np.all(np.abs(p) < 8)
        assert set(np.unique(col)) <= {0.0, 1.0}
        filtered, _ = oracle.numpy_shadow_filter(d, 2, 2, -1.0)
        assert (filtered == -1).sum() > 20


def test_shadow_scenes_reach_their_cases():
    S = E.shadow_scenes()
    n = {k: len(E.positive_deltas(d, dx, dy)) for k, (d, dx, dy) in S.items()}
    assert n["count0_constant"] == 0 and n["count1"] == 1 and n["count2"] == 2
    assert n["odd_count"] % 2 == 1 and n["even_count"] % 2 == 0
    assert len(np.unique(E.positive_deltas(*S["all_equal"]))) == 1
    v = E.positive_deltas(*S["even_middles_differ"])
    lo, hi = v[(len(v) - 1) // 2], v[len(v) // 2]
    thr, thr_upper = oracle.numpy_shadow_filter(*S["even_middles_differ"])[1], f32(3) * (f32(1.4826) * hi)
    assert len(v) % 2 == 0 and lo < hi and ((v > thr) & (v <= thr_upper)).sum() == 1
    t = E.positive_deltas(*S["ties"])
    assert (t == t[(len(t) - 1) // 2]).sum() > len(t) // 4
    for name, shift in (("pass2", 21), ("pass3", 10)):
        v = E.positive_deltas(*S[name]).view(np.uint32)
        top = v >> shift
        mid = top[(len(v) - 1) // 2]
        assert (top == mid).sum() >= len(v) - 8 and len(np.unique(v)) > 10, name
        if name == "pass2":
            assert len(np.unique(v >> 10)) > 3
    sub = E.positive_deltas(*S["subnormal"])
    assert (sub < np.finfo(f32).tiny).sum() > len(sub) // 2
    assert np.isinf(E.positive_deltas(*S["posinf"])).any()
    mi = E.positive_deltas(*S["median_inf"])
    assert np.isinf(mi[(len(mi) - 1) // 2])
    assert np.isnan(S["nan"][0]).any() and (np.signbit(S["negzero"][0]) & (S["negzero"][0] == 0)).any()
    d, dx, dy = S["dx_W-1_dy_H-1"]
    assert dx == d.shape[1] - 1 and dy == d.shape[0] - 1
    assert S["vga"][0].shape == (480, 640) and S["tiny_3x3_d1"][0].shape == (3, 3)
    for name in ("count0_constant", "count1", "count2", "all_equal"):
        out, _ = oracle.numpy_shadow_filter(S[name][0], S[name][1], S[name][2])
        assert np.array_equal(out, S[name][0]), name
    for name in ("odd_count", "even_count", "ties", "pass2", "pass3", "posinf", "nan", "vga", "d3"):
        out, _ = oracle.numpy_shadow_filter(*S[name])
        assert (out == -1).sum() > 0, name


def test_remap_maps_reach_their_families():
    H, W = 61, 83
    mx, my = E.remap_maps("ties64", H, W)
    assert np.all((mx * 32) % 1 == 0.5)
    mx, my = E.remap_maps("half", H, W)
    assert np.all(mx % 1 == 0.5)
    mx, my = E.remap_maps("border", H, W)
    assert ((mx < 0) & (mx > -1)).any() and ((mx > W - 1) & (mx < W)).any()
    mx, my = E.remap_maps("huge", H, W)
    assert (np.abs(mx) >= 4e4).any() and (np.abs(mx) > 3e38).any() and (np.abs(my) >= 4e4).any()
    mx, my = E.remap_maps("inf", H, W)
    assert np.isposinf(mx).any() and np.isneginf(mx).any()
    for kind, nx, ny in (("nan_x", True, False), ("nan_y", False, True), ("nan_both", True, True)):
        mx, my = E.remap_maps(kind, H, W)
        assert np.isnan(mx).any() == nx and np.isnan(my).any() == ny
        if kind == "nan_both":
            assert (np.isnan(mx) & np.isnan(my)).any()
