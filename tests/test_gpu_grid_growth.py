"""Point-average and semantic grids that grow with the map (`max_capacity_blocks`).

A growable grid starts with storage for `capacity_blocks` blocks.  The integrate call that hands out a pool index past
the storage maps more and replays its accumulation (point grid) or its keys -> sort -> runs (semantic grids) over the
blocks that just got storage, before it returns.  Every case here starts small enough to overflow at least twice and
compares, bit for bit after sorting by key, with a fixed grid created at the ceiling (and with the numpy oracle where
named).  Point-grid scenes keep every float32 sum exact in any order (tests/_grid_prep_scenes.py), so float atomics
cannot make two grids differ."""

import os

import numpy as np
import pytest

import oracle
from pyslam_b200 import (BoundingBox3D, CameraFrustrum, VoxelBlockGrid, VoxelBlockSemanticGrid,
                         VoxelBlockSemanticProbabilisticGrid, remap_instance_ids)
from pyslam_b200 import synthetic as S
from tests import _grid_prep_scenes as E
from tests import plugin_standins as P
from tests._util import GOLDEN, sort_dump
from tests.test_gpu_semantic import _compare_dumps

pytestmark = pytest.mark.gpu
f32 = np.float32
Q = E.Q


def _rows(p, c):
    a = np.concatenate([p, c], 1)
    return a[np.lexsort(a.T[::-1])]


def _same_voxels(a, b):
    assert len(a.points) == len(b.points)
    assert np.array_equal(_rows(a.points, a.colors), _rows(b.points, b.colors))


def _same_point_grids(a, b, G=None):
    da, db = sort_dump(a.dump_blocks()), sort_dump(b.dump_blocks())
    for k in ("keys", "count", "pos_sum", "col_sum"):
        assert np.array_equal(da[k], db[k]), k
    if G is not None:
        r = G.dump()
        for k in ("keys", "count", "pos_sum", "col_sum"):
            assert np.array_equal(da[k], r[k]), k
    for m in (1, 2):
        _same_voxels(a.get_voxels(m), b.get_voxels(m))
        if G is not None:
            ref = G.get_voxels(m)
            got = a.get_voxels(m)
            assert np.array_equal(_rows(got.points, got.colors), _rows(*ref))
    return da


def _many_blocks(seed, n_blocks, per_block=24, lo=-40, hi=40):
    """Dyadic points (multiples of 2^-12, |x| < 8) in `n_blocks` distinct blocks of 2^-6 m voxels, a few voxels of each
    block hit several times; dyadic float colours.  Every float32 sum is exact in any order.  Block-major order, so
    that consecutive slices of the points bring new blocks."""
    rng = np.random.default_rng(seed)
    keys = np.unique(rng.integers(lo, hi, (3 * n_blocks, 3)), axis=0)
    keys = keys[rng.permutation(len(keys))[:n_blocks]]
    vox = rng.integers(0, 8, (n_blocks, per_block // 3, 3))
    vox = np.repeat(vox, 3, axis=1)                              # each voxel three times
    frac = rng.integers(0, 64, vox.shape)                        # position inside the voxel, 2^-12 steps
    p = ((keys[:, None, :] * 8 + vox) * 64 + frac) * Q
    p = p.reshape(-1, 3).astype(f32)
    return p, E.dyadic_colors(rng, len(p))


def _point_grids(vs, start, ceiling):
    return (VoxelBlockGrid(vs, 8, capacity_blocks=start, max_capacity_blocks=ceiling),
            VoxelBlockGrid(vs, 8, capacity_blocks=ceiling))


# ---- 1. point-average grid: growth inside one call and across calls -------------------------------------------------

def test_point_grid_overflow_inside_one_call_and_across_calls():
    p, c = _many_blocks(0, 3000)
    # one call that creates far more than 4x the storage
    g, f = _point_grids(E.VS_EXACT, 16, 1 << 13)
    G = oracle.numpy_grid(E.VS_EXACT)
    for grid in (g, f):
        grid.integrate(p, c)
    G.integrate(p, c)
    assert g.num_blocks() == 3000 and g.capacity()[1] >= 1 and g.capacity()[0] >= 3000
    _same_point_grids(g, f, G)
    # many calls, storage overflowing again and again; blocks of earlier calls keep accumulating
    g, f = _point_grids(E.VS_EXACT, 16, 1 << 13)
    G = oracle.numpy_grid(E.VS_EXACT)
    q, d = _many_blocks(1, 3000, lo=-30, hi=30)
    for part in np.array_split(np.arange(len(q)), 12):
        for grid in (g, f):
            grid.integrate(q[part], d[part])
        G.integrate(q[part], d[part])
    assert g.capacity()[1] >= 3
    for grid in (g, f, G):
        grid.integrate(q[::-1].copy(), d[::-1].copy())
    _same_point_grids(g, f, G)


def test_point_grid_float64_points_and_colour_kinds():
    """float64 points (keys from the float64 coordinates, at most two points per voxel) and uint8 / float / absent
    colours, each from 8 blocks of storage."""
    p = E.float64_points()
    g, f = _point_grids(0.005, 8, 1 << 15)
    G = oracle.numpy_grid(0.005)
    for part in np.array_split(np.arange(len(p)), 3):
        for grid in (g, f):
            grid.integrate(p[part])
        G.integrate(p[part])
    assert g.capacity()[1] >= 2
    _same_point_grids(g, f, G)
    q, fc = _many_blocks(2, 1500)
    # uint8 colours 0 or 255: every non-zero addend of a voxel is the same float32(255) * (1 / 255.0f), so its sums
    # do not depend on the order of the adds either
    u8 = (np.random.default_rng(5).integers(0, 2, q.shape) * 255).astype(np.uint8)
    for cols in (u8, fc, None):
        g, f = _point_grids(E.VS_EXACT, 8, 4096)
        G = oracle.numpy_grid(E.VS_EXACT)
        for part in np.array_split(np.arange(len(q)), 2):
            cc = None if cols is None else cols[part]
            for grid in (g, f):
                grid.integrate(q[part], cc)
            G.integrate(q[part], cc)
        assert g.capacity()[1] >= 2
        d = _same_point_grids(g, f, G)
        assert cols is not None or not d["col_sum"].any()


def _rgbd_frames(seed=9, n=3, H=96, W=128):
    """Frames whose back-projected points are exact: depths in 2^-6 steps, fx = fy = 64, integer principal point,
    identity rotation and dyadic translation, colours 0 or 255.  Many blocks per frame, a depth step for the shadow
    filter."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        d = (64 + rng.integers(0, 96, (H, W))).astype(np.float64) / 64
        d[20:60, 30 + 4 * i:80 + 4 * i] = (200 + rng.integers(0, 3, (40, 50))) / 64
        d[0, :7] = 0.0
        c = (rng.integers(0, 2, (H, W, 3)) * 255).astype(np.uint8)
        Twc = np.eye(4)
        Twc[:3, 3] = [0.25 * i, -0.125, 0.0625 * i]
        out.append((d.astype(f32), c, Twc))
    return out, (64.0, 64.0, W / 2, H / 2)


@pytest.mark.parametrize("flt", [False, True])
def test_point_grid_integrate_rgbd(flt):
    frames, K = _rgbd_frames()
    g, f = _point_grids(E.VS_EXACT, 8, 1 << 15)
    G = oracle.numpy_grid(E.VS_EXACT)
    for d, c, Twc in frames:
        for grid in (g, f):
            grid.integrate_rgbd(d, c, K, Twc, filter_shadow_points=flt)
        dd = oracle.numpy_shadow_filter(d, 2, 2, -1.0)[0] if flt else d
        G.integrate(*E.rgbd_points(dd, c, K, Twc))
    assert g.capacity()[1] >= 2
    _same_point_grids(g, f, G)


def test_point_grid_device_inputs_through_the_c_abi():
    """torch tensors on the device: the replay reads the caller's device buffers (points / colours, RGBD frames)."""
    torch = pytest.importorskip("torch")
    p, c = _many_blocks(3, 2500)
    frames, K = _rgbd_frames(seed=4, n=2)
    g, f = _point_grids(E.VS_EXACT, 8, 1 << 15)
    tp, tc = torch.from_numpy(p).cuda(), torch.from_numpy(c).cuda()
    K4 = np.array(K, np.float64)
    torch.cuda.synchronize()
    for grid in (g, f):
        for part in np.array_split(np.arange(len(p)), 2):
            s, e = int(part[0]), int(part[-1]) + 1
            grid._check(grid._L.b2v_grid_integrate_ex(grid._h, tp[s:e].data_ptr(), 0, tc[s:e].data_ptr(), 0, e - s),
                        "integrate_ex")
            grid._check(grid._L.b2v_grid_synchronize(grid._h), "sync")
        for d, col, Twc in frames:
            td, tcol = torch.from_numpy(d).cuda(), torch.from_numpy(col).cuda()
            T = np.ascontiguousarray(Twc, np.float64).reshape(16)
            torch.cuda.synchronize()
            grid._check(grid._L.b2v_grid_integrate_rgbd(grid._h, td.data_ptr(), tcol.data_ptr(), d.shape[0], d.shape[1],
                                                        K4.ctypes.data, T.ctypes.data, 3.0e38, 0.0, 0), "rgbd")
            grid._check(grid._L.b2v_grid_synchronize(grid._h), "sync")
    assert g.capacity()[1] >= 2
    _same_point_grids(g, f)


# ---- 2. point-average grid after growth: queries, carve, remove_low_count_voxels --------------------------------------

def _filler():
    """Dyadic points in many blocks at x >= 4 m: outside every box and frustum of the query scenes."""
    p, c = _many_blocks(6, 1200, lo=-20, hi=20)
    p[:, 0] = np.abs(p[:, 0]) + 4.0
    return p, c


def _integrate_in_parts(grids, p, c=None, parts=3):
    """The same points in `parts` calls into every grid (and oracle): the storage overflows in several calls."""
    for idx in np.array_split(np.arange(len(p)), parts):
        for grid in grids:
            grid.integrate(p[idx], None if c is None else c[idx])


@pytest.mark.parametrize("box", range(len(E.BOXES)))
def test_point_grid_box_query_after_growth(box):
    bb = E.BOXES[box]
    fp, fc = _filler()
    pts = E.box_probe_points(bb)
    cols = E.dyadic_colors(np.random.default_rng(box), len(pts))
    g, f = _point_grids(E.VS_EXACT, 4, 4096)
    G = oracle.numpy_grid(E.VS_EXACT)
    _integrate_in_parts((g, f, G), fp, fc)
    for grid in (g, f, G):
        grid.integrate(pts, cols)
    assert g.capacity()[1] >= 2
    _same_voxels(g.get_voxels_in_bb(BoundingBox3D(*bb), min_count=1), f.get_voxels_in_bb(BoundingBox3D(*bb), 1))
    got = g.get_voxels_in_bb(BoundingBox3D(*bb), min_count=1)
    assert np.array_equal(_rows(got.points, got.colors), _rows(*G.get_voxels_in_bb(bb)))


@pytest.mark.parametrize("pose", [0, 1])
def test_point_grid_frustum_carve_and_low_count_after_growth(pose):
    T = E.cam_poses()[pose]
    fp, fc = _filler()
    fr = CameraFrustrum(*E.CAM_K, E.CAM_W, E.CAM_H, T, depth_max=E.DEPTH_MAX, depth_min=E.DEPTH_MIN)
    probe = E.frustum_probe_points(T)
    probe = np.concatenate([probe, probe[:20]])
    pcols = E.dyadic_colors(np.random.default_rng(pose), len(probe))
    cpts, img = E.carve_scene(T)
    g, f = _point_grids(E.VS_EXACT, 4, 4096)
    _integrate_in_parts((g, f), fp, fc)
    for grid in (g, f):
        grid.integrate(probe, pcols)
    assert g.capacity()[1] >= 2
    for m in (1, 2):
        _same_voxels(g.get_voxels_in_camera_frustrum(fr, min_count=m), f.get_voxels_in_camera_frustrum(fr, min_count=m))
    g, f = _point_grids(E.VS_EXACT, 4, 4096)
    G = oracle.numpy_grid(E.VS_EXACT)
    _integrate_in_parts((g, f, G), fp, fc)
    for grid in (g, f):
        grid.integrate(cpts)
        grid.carve(fr, img, depth_threshold=E.CARVE_THR)
    G.integrate(cpts)
    assert len(G.carve(E.CAM_K, E.CAM_W, E.CAM_H, T, img, E.CARVE_THR, E.DEPTH_MAX, E.DEPTH_MIN)) >= 10
    _same_point_grids(g, f, G)
    for grid in (g, f):
        grid.integrate(fp[:300], fc[:300])
        grid.remove_low_count_voxels(4)
    G.integrate(fp[:300], fc[:300])
    G.remove_low_count_voxels(4)
    _same_point_grids(g, f, G)


# ---- 3. semantic grids -------------------------------------------------------------------------------------------------

SEM = {"vote": VoxelBlockSemanticGrid, "prob": VoxelBlockSemanticProbabilisticGrid}
DUMP_KEYS = ("keys", "hashes", "count", "pos_sum", "col_sum", "object_id", "class_id", "confidence", "aux", "lab_obj",
             "lab_cls", "lab_logp")


def _same_sem(a, b):
    da, db = sort_dump(a.dump_blocks(8)), sort_dump(b.dump_blocks(8))
    for k in DUMP_KEYS:
        assert np.array_equal(da[k], db[k], equal_nan=True), k
    assert a.label_overflows() == b.label_overflows()
    assert a.num_blocks() == b.num_blocks()
    return da


def _same_readout(a, b):
    assert len(a.points) == len(b.points)
    ka = np.lexsort(a.points.T[::-1])
    kb = np.lexsort(b.points.T[::-1])
    for k in ("points", "colors", "class_ids", "object_ids", "confidences"):
        assert np.array_equal(np.asarray(getattr(a, k))[ka], np.asarray(getattr(b, k))[kb]), k


def _t0_grids(tag, start=8, ceiling=1024):
    g = np.load(os.path.join(GOLDEN, "semantic_T0.npz"))
    grids = (SEM[tag](float(g["voxel_size"]), 8, capacity_blocks=start, max_capacity_blocks=ceiling),
             SEM[tag](float(g["voxel_size"]), 8, capacity_blocks=ceiling))
    for grid in grids:
        grid.set_depth_threshold(float(g[f"{tag}_depth_threshold"]))
        grid.set_depth_decay_rate(float(g[f"{tag}_depth_decay_rate"]))
        for i in range(int(g["n_frames"])):
            grid.integrate(g[f"{tag}_points_{i}"], g[f"{tag}_colors_{i}"], g[f"{tag}_cls_{i}"], g[f"{tag}_inst_{i}"],
                           g[f"{tag}_depths_{i}"])
    return g, grids


@pytest.mark.parametrize("tag", ["vote", "prob"])
def test_semantic_golden_stream_from_far_below_its_block_count(tag):
    """The golden stream's 50 blocks fit in the first granule of every array, so it overflows once; the other
    semantic scenes overflow at least twice."""
    g, (grown, fixed) = _t0_grids(tag, start=4)
    ref = {k: g[f"{tag}_{k}"] for k in DUMP_KEYS}
    assert len(ref["keys"]) >= 10 * 4 and grown.capacity()[1] >= 1
    _same_sem(grown, fixed)
    _compare_dumps(sort_dump(grown.dump_blocks(8)), ref, tag)


def _c3_frames(n=2):
    cfg = S.CONFIGS["C3"]
    out = []
    for i in range(n):
        d, c, Tcw = S.render_frame(cfg, 40 * i)
        cls = S.render_class_ids(cfg, 40 * i)
        obj = np.where(cls % 3 == 0, -1, cls * 7 + (np.arange(cls.shape[1])[None, :] // 400)).astype(np.int32)
        out.append((d, c, S.inv_T(Tcw), cls, obj))
    return cfg, out


@pytest.mark.parametrize("tag", ["vote", "prob"])
def test_semantic_c3_integrate_rgbd_with_labels(tag):
    cfg, frames = _c3_frames()
    for flt, use_depths in ((False, True), (True, False)):
        grown = SEM[tag](0.015, 8, capacity_blocks=16, max_capacity_blocks=1 << 15)
        fixed = SEM[tag](0.015, 8, capacity_blocks=1 << 15)
        for grid in (grown, fixed):
            grid.set_depth_threshold(1.5)
            for d, c, Twc, cls, obj in frames:
                grid.integrate_rgbd(d, c, cfg.K, Twc, cls, obj, max_depth=cfg.depth_trunc, use_depths=use_depths,
                                    filter_shadow_points=flt)
        assert grown.capacity()[1] >= 2 and grown.num_blocks() > 500
        _same_sem(grown, fixed)


@pytest.mark.parametrize("tag", ["vote", "prob"])
def test_semantic_edits_segments_association_and_read_outs_after_growth(tag):
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    vs, K = float(g["voxel_size"]), g["K"]
    grown = SEM[tag](vs, 8, capacity_blocks=8, max_capacity_blocks=1024)
    fixed = SEM[tag](vs, 8, capacity_blocks=1024)
    for grid in (grown, fixed):
        grid.set_next_object_id(1)
    for i in range(int(g["n_frames"])):
        d, c, T = g[f"depth_{i}"], g[f"color_{i}"], g[f"Tcw_{i}"]
        cls_img, inst_img = g[f"class_image_{i}"], g[f"instance_image_{i}"]
        fr = CameraFrustrum(K[0], K[1], K[2], K[3], d.shape[1], d.shape[0], T, depth_max=8.0, depth_min=1e-2)
        maps = [grid.assign_object_ids_to_instance_ids(fr, cls_img, inst_img, d, depth_threshold=0.08, do_carving=True,
                                                       min_vote_ratio=0.5, min_votes=3) for grid in (grown, fixed)]
        assert maps[0] == maps[1]
        for grid in (grown, fixed):
            grid.integrate_rgbd(d, c, K, np.linalg.inv(T), cls_img, remap_instance_ids(inst_img, maps[0]),
                                max_depth=4.0)
    _same_sem(grown, fixed)
    pts = np.random.default_rng(1).uniform(-12, 12, (400, 3)).astype(f32)   # ~400 new blocks: storage grows again
    cols = np.full((400, 3), 0.5, f32)
    for grid in (grown, fixed):
        grid.integrate_segment(pts, cols, 3, 77)
    assert grown.capacity()[1] >= 2
    _same_sem(grown, fixed)
    for by in ("get_object_segments", "get_class_segments"):
        sa, sb = getattr(grown, by)(1, 0.0), getattr(fixed, by)(1, 0.0)
        la = sa.object_vector if hasattr(sa, "object_vector") else sa.class_vector
        lb = sb.object_vector if hasattr(sb, "object_vector") else sb.class_vector
        assert len(la) == len(lb) > 0
        for x, y in zip(la, lb):
            assert (x.class_id, x.confidence_min, x.confidence_max) == (y.class_id, y.confidence_min, y.confidence_max)
            assert np.array_equal(_rows(np.asarray(x.points), np.asarray(x.colors)),
                                  _rows(np.asarray(y.points), np.asarray(y.colors)))
    d, T = g["depth_0"], g["Tcw_0"]
    fr = CameraFrustrum(K[0], K[1], K[2], K[3], d.shape[1], d.shape[0], T, depth_max=3.0, depth_min=0.1)
    bb = BoundingBox3D(-0.5, -0.5, 0.0, 1.0, 1.0, 2.0)
    _same_readout(grown.get_voxels_in_bb(bb, 1, 0.0), fixed.get_voxels_in_bb(bb, 1, 0.0))
    _same_readout(grown.get_voxels_in_camera_frustrum(fr, 1, 0.0), fixed.get_voxels_in_camera_frustrum(fr, 1, 0.0))
    obj = [int(o) for o in np.unique(sort_dump(fixed.dump_blocks(1))["object_id"]) if o > 0]
    assert len(obj) >= 2
    for grid in (grown, fixed):
        grid.merge_segments(obj[0], obj[1])
        grid.remove_segment(77)
        grid.carve(fr, d * 1.5, depth_threshold=0.05)
        grid.remove_low_count_voxels(2)
    _same_sem(grown, fixed)
    _same_readout(grown.get_voxels(1, 0.0), fixed.get_voxels(1, 0.0))


# ---- 4. the ceiling ----------------------------------------------------------------------------------------------------

def _block_points(n):
    """One point in each of n distinct blocks (2^-6 m voxels), in a fixed order."""
    k = np.stack(np.meshgrid(np.arange(8) - 4, np.arange(8) - 4, np.arange(8) - 4, indexing="ij"), -1).reshape(-1, 3)
    return ((k[:n] * 8 + 3.5) * E.VS_EXACT).astype(f32)


def _make(kind, cap, mx):
    if kind == "grid":
        return VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=cap, max_capacity_blocks=mx)
    return VoxelBlockSemanticProbabilisticGrid(E.VS_EXACT, 8, capacity_blocks=cap, max_capacity_blocks=mx)


def _fill(grid, pts, parts=1):
    for idx in np.array_split(np.arange(len(pts)), parts):
        p = pts[idx]
        if isinstance(grid, VoxelBlockGrid):
            grid.integrate(p, np.full_like(p, 0.25))
        else:
            grid.integrate(p, np.full_like(p, 0.25), idx.astype(np.int32) % 5, np.ones(len(p), np.int32))


@pytest.mark.parametrize("kind", ["grid", "sem"])
def test_ceiling(kind):
    n = 200
    pts = _block_points(n + 1)
    g = _make(kind, 4, n)
    _fill(g, pts[:n])
    assert g.num_blocks() == n and g.capacity() == (n, g.capacity()[1]) and g.capacity()[1] >= 1
    g = _make(kind, 4, n)
    with pytest.raises(RuntimeError, match="block pool full"):
        _fill(g, pts)
    assert g.num_blocks() == n
    u = _make(kind, 1 << 10, 0)
    _fill(u, pts)
    dg, du = sort_dump(g.dump_blocks()), sort_dump(u.dump_blocks())
    kk = [tuple(k) for k in du["keys"]]
    sel = np.array([kk.index(tuple(k)) for k in dg["keys"]])
    for name in dg:
        if name != "hashes":
            assert np.array_equal(dg[name], du[name][sel], equal_nan=True), name
    # max = 0 and max = capacity: today's fixed pool
    for mx in (0, n):
        f = _make(kind, n, mx)
        _fill(f, pts[:n])
        assert f.capacity() == (n, 0)
        with pytest.raises(RuntimeError, match="block pool full"):
            _fill(f, pts[n:])
    for cap, mx in ((64, 32), (8, (1 << 22) + 1)):
        with pytest.raises(RuntimeError):
            _make(kind, cap, mx)
    assert _make(kind, 8, 1 << 22).capacity() == (8, 0)


# ---- 5. storage --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["grid", "sem"])
def test_storage_is_kept_by_clear(kind):
    g = _make(kind, 256, 1 << 12)
    _fill(g, _block_points(100))
    assert g.capacity() == (256, 0)
    g = _make(kind, 4, 1 << 12)
    pts = _block_points(500)
    _fill(g, pts, parts=3)
    grown = g.capacity()
    assert grown[1] >= 2 and grown[0] >= 500
    g.clear()
    assert g.capacity() == grown and g.num_blocks() == 0
    fresh = _make(kind, 1 << 12, 0)
    for grid in (g, fresh):
        _fill(grid, pts[::-1].copy())
    assert g.capacity() == grown
    if kind == "grid":
        _same_point_grids(g, fresh)
    else:
        _same_sem(g, fresh)


# ---- 6. plugins ----------------------------------------------------------------------------------------------------------

def _camera(cfg):
    from types import SimpleNamespace
    return SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)


def _drain(integ):
    integ.add_update_output_task()
    integ.step()
    out = None
    while True:
        o = integ.pop_output()
        if o is None:
            return out
        out = o


@pytest.mark.parametrize("plugin", ["voxel_grid", "semantic"])
def test_plugins_with_a_growth_ceiling(plugin):
    cfg = S.CONFIGS["T0"]
    outs = []
    for cap, mx in ((16, 4096), (4096, 0)):
        kw = dict(kVolumetricIntegrationVoxelLength=0.03, kVolumetricIntegrationB200CapacityBlocks=cap,
                  kVolumetricIntegrationB200MaxCapacityBlocks=mx)
        if plugin == "voxel_grid":
            Cls = P.standalone_voxel_grid_integrator_class()
            integ = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_VOXEL_GRID", **kw)
        else:
            Cls = P.standalone_semantic_integrator_class()
            integ = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_SEMANTIC",
                        use_semantic_probabilistic=True, **kw)
        for i in range(4):
            d, c, T = S.render_frame(cfg, i)
            data = dict(id=i, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=d)
            if plugin == "semantic":
                data.update(semantic_img=S.render_class_ids(cfg, i))
            integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(**data))
            integ.step()
        if mx:
            assert integ.volume.capacity()[1] >= 2
        out = _drain(integ)
        outs.append((out, sort_dump(integ.volume.dump_blocks())))
        integ.quit()
    (a, da), (b, db) = outs
    assert np.array_equal(da["keys"], db["keys"]) and np.array_equal(da["count"], db["count"])
    if plugin == "semantic":
        for k in DUMP_KEYS:
            if k in da:
                assert np.array_equal(da[k], db[k], equal_nan=True), k
        assert np.array_equal(_rows(a.point_cloud.points, a.point_cloud.colors),
                              _rows(b.point_cloud.points, b.point_cloud.colors))
        assert np.array_equal(np.sort(a.point_cloud.semantics), np.sort(b.point_cloud.semantics))
    else:
        # real frames: float atomics may add a voxel's points in another order in any two runs, grown or not
        assert np.allclose(da["pos_sum"], db["pos_sum"], rtol=1e-5, atol=1e-6)
        pa, pb = np.asarray(a.point_cloud.points), np.asarray(b.point_cloud.points)
        assert pa.shape == pb.shape and np.allclose(pa[np.lexsort(pa.T[::-1])], pb[np.lexsort(pb.T[::-1])],
                                                    rtol=1e-5, atol=1e-6)
