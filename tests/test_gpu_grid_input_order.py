"""GPU: the point-average grid's input-order sums (`VoxelBlockGrid(input_order_sums=True)`,
`b2v_grid_set_input_order_sums`).  Each voxel adds its points in input order with IEEE float32 adds, so the grid must
equal, bit for bit, the compiled reference's sequential build (the committed golden, and live when oracle/_ref is
built) and `oracle.numpy_grid`, and be the same on every run, for every input kind, shard layout, growth and state
round trip.  Every comparison is exact (`np.array_equal` on sorted dumps); the scenes are order-sensitive
(tests/_grid_order_scenes.py, checked by tests/test_grid_input_order_cpu.py)."""

import ctypes as C
import os

import numpy as np
import pytest

import oracle
from pyslam_b200 import BoundingBox3D, CameraFrustrum, VoxelBlockGrid, _lib
from pyslam_b200 import synthetic as S
from tests import _block_sizes as BS
from tests import _grid_order_scenes as O
from tests import _grid_prep_scenes as E
from tests._util import GOLDEN, sort_dump

pytestmark = pytest.mark.gpu
FIELDS = ("keys", "hashes", "count", "pos_sum", "col_sum")


def _grid(vs=O.VS, B=8, **kw):
    kw.setdefault("capacity_blocks", 1 << 15)
    return VoxelBlockGrid(vs, B, input_order_sums=True, **kw)


def _same(a, b, fields=FIELDS, what=""):
    a = a if isinstance(a, dict) else sort_dump(a.dump_blocks())
    b = b if isinstance(b, dict) else sort_dump(b.dump_blocks())
    for k in fields:
        assert np.array_equal(a[k], b[k]), (what, k)


def _oracle_dump(G, B=8):
    return BS.grid_dump(G, B)


def _rows(p, c):
    """Read-out rows (point, colour) in a canonical order."""
    r = np.concatenate([p, c], 1)
    return r[np.lexsort(r.T[::-1])]


def _feed_golden(grid, g):
    start = 0
    for n in g["frame_counts"]:
        grid.integrate(g["points"][start:start + n], g["colors"][start:start + n])
        start += int(n)


def _grid_fed_golden(g):
    grid = _grid(float(g["voxel_size"]), capacity_blocks=4096)
    _feed_golden(grid, g)
    return grid


def _same_counts(a, b, what=""):
    """The modes agree on keys, hashes and counts."""
    _same(a, b, ("keys", "hashes", "count"), what)


# ---- the compiled reference -------------------------------------------------------------------------------------

def _golden_frustum(g):
    K = g["query_K"]
    H, W = g["query_depth"].shape
    return CameraFrustrum(K[0], K[1], K[2], K[3], W, H, g["query_Tcw"], depth_max=3.0, depth_min=0.05)


def test_golden_reference_bit_for_bit():
    """refgrid_T0.npz, made by the unmodified compiled reference: dump, read-out, queries and carve all equal."""
    g = np.load(os.path.join(GOLDEN, "refgrid_T0.npz"))
    grid = _grid_fed_golden(g)
    assert grid.input_order_sums
    _same(grid, {k: g[k] for k in FIELDS})
    atomic = VoxelBlockGrid(float(g["voxel_size"]), 8, capacity_blocks=4096)
    _feed_golden(atomic, g)
    _same_counts(grid, atomic)
    out = grid.get_voxels(min_count=2)
    order = np.lexsort((out.points[:, 2], out.points[:, 1], out.points[:, 0]))
    assert np.array_equal(out.points[order], g["voxels_min2_points"])
    assert np.array_equal(out.colors[order], g["voxels_min2_colors"])
    fr = _golden_frustum(g)
    fp = grid.get_voxels_in_camera_frustrum(fr, min_count=1).points
    assert np.array_equal(fp[np.lexsort(fp.T[::-1])], g["frustum_points"])
    bp = grid.get_voxels_in_bb(BoundingBox3D(*g["query_bbox"]), min_count=1).points
    assert np.array_equal(bp[np.lexsort(bp.T[::-1])], g["bbox_points"])
    grid.carve(fr, g["query_depth"], depth_threshold=0.05)
    assert np.array_equal(sort_dump(grid.dump_blocks())["count"], g["carved_count"])


def test_integrate_rgbd_equals_the_golden():
    """integrate_rgbd on the three tsdf_T0 frames refgrid_T0 was made from: the whole dump equals the golden."""
    g = np.load(os.path.join(GOLDEN, "refgrid_T0.npz"))
    t = np.load(os.path.join(GOLDEN, "tsdf_T0.npz"))
    grid = _grid(float(g["voxel_size"]), capacity_blocks=4096)
    atomic = VoxelBlockGrid(float(g["voxel_size"]), 8, capacity_blocks=4096)
    for i in range(len(g["frame_counts"])):
        for x in (grid, atomic):
            x.integrate_rgbd(t["depth"][i], t["color"][i], t["K"], S.inv_T(t["Tcw"][i]),
                             max_depth=float(t["depth_trunc"]))
    _same(grid, {k: g[k] for k in FIELDS})
    _same_counts(grid, atomic)


@pytest.mark.skipif(not oracle.have_ref(), reason="compiled reference (oracle/_ref) not built")
def test_live_reference_on_real_frames():
    ref = oracle.RefGrid(O.VS, 8)
    grid = _grid()
    for p, c in O.frame_points():
        ref.integrate(p, c)
        grid.integrate(p, c)
    _same(grid, sort_dump(ref.dump_blocks()))


# ---- order-sensitive scenes against numpy_grid ------------------------------------------------------------------

def _scene_batches(kind):
    pts, u8, fl = O.stress_scene()
    if kind == "uint8":
        return [(pts, u8)]
    if kind == "float":
        return [(pts, fl)]
    if kind == "none":
        return [(pts, None)]
    if kind == "calls12":
        return [(pts[i], fl[i]) for i in np.array_split(np.arange(len(pts)), 12)]
    if kind == "float64":
        return [O.float64_scene()]
    return [O.subnormal_scene()]


@pytest.mark.parametrize("B", BS.BLOCK_SIZES)
@pytest.mark.parametrize("kind", ["uint8", "float", "none", "calls12", "float64", "subnormal"])
def test_scenes_equal_numpy_grid(kind, B):
    batches = _scene_batches(kind)
    grid, atomic = _grid(B=B), VoxelBlockGrid(O.VS, B, capacity_blocks=1 << 15)
    for p, c in batches:
        grid.integrate(p, c)
        atomic.integrate(p, c)
    _same(grid, _oracle_dump(O.numpy_grid_of(batches), B), ("keys", "count", "pos_sum", "col_sum"), (kind, B))
    _same_counts(grid, atomic, (kind, B))


# ---- reproducible on real frames --------------------------------------------------------------------------------

def _feed_frames(grids, frames=None):
    for d, c, Twc in (frames or O.frames()):
        for x in grids:
            x.integrate_rgbd(d, c, O.frame_K(), Twc, max_depth=O.frame_max_depth())


def _feed_device_frames(grid):
    """The frames as torch CUDA tensors through the C ABI, read in place."""
    import torch
    K = np.asarray(O.frame_K(), np.float64)
    for d, c, Twc in O.frames():
        dd, cd = torch.from_numpy(d).cuda(), torch.from_numpy(c).cuda()
        torch.cuda.synchronize()   # the library reads device inputs on its own stream
        T = np.ascontiguousarray(Twc, np.float64).reshape(16)
        rc = grid._L.b2v_grid_integrate_rgbd(grid._h, dd.data_ptr(), cd.data_ptr(), d.shape[0], d.shape[1],
                                             K.ctypes.data, T.ctypes.data, O.frame_max_depth(), 0.0, 0)
        assert rc == _lib.B2V_OK
        assert grid._L.b2v_grid_synchronize(grid._h) == _lib.B2V_OK


def _frames_oracle(frames=None):
    return O.numpy_grid_of([E.rgbd_points(d, c, O.frame_K(), Twc, max_depth=O.frame_max_depth())
                            for d, c, Twc in (frames or O.frames())])


def test_real_frames_reproducible_and_equal_numpy_grid():
    a, b, dev, atomic = _grid(), _grid(), _grid(), VoxelBlockGrid(O.VS, 8, capacity_blocks=1 << 15)
    _feed_frames([a, b, atomic])
    _feed_device_frames(dev)
    ref = _oracle_dump(_frames_oracle())
    _same(a, ref, ("keys", "count", "pos_sum", "col_sum"))
    _same(a, b)
    _same(a, dev)
    _same_counts(a, atomic)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_shards_hold_the_unsharded_blocks(world):
    single = _grid()
    shards = [_grid(shard_rank=r, shard_count=world) for r in range(world)]
    _feed_frames([single] + shards)
    whole = sort_dump(single.dump_blocks())
    row = {tuple(k): i for i, k in enumerate(whole["keys"].tolist())}
    n = 0
    for s in shards:
        d = sort_dump(s.dump_blocks())
        idx = np.array([row[tuple(k)] for k in d["keys"].tolist()], np.int64)
        n += len(idx)
        _same(d, {k: v[idx] for k, v in whole.items()}, what=world)
    assert n == len(whole["keys"])


def test_growth_equals_fixed_grid_and_numpy_grid():
    grown, fixed = _grid(capacity_blocks=4, max_capacity_blocks=1 << 15), _grid()
    _feed_frames([grown, fixed])
    assert grown.capacity()[1] >= 2
    _same(grown, fixed)
    _same(grown, _oracle_dump(_frames_oracle()), ("keys", "count", "pos_sum", "col_sum"))
    # integrate (points) grows the same way
    pts = O.frame_points()
    g2 = _grid(capacity_blocks=4, max_capacity_blocks=1 << 15)
    for p, c in pts:
        g2.integrate(p, c)
    assert g2.capacity()[1] >= 2
    _same(g2, fixed)


def test_state_round_trip_into_one_and_three_grids(tmp_path):
    fr = O.frames()
    whole = _grid()
    _feed_frames([whole], fr)
    first = _grid()
    _feed_frames([first], fr[:5])
    path = str(tmp_path / "half.npz")
    first.save_state(path)
    one = _grid()
    three = [_grid(shard_rank=r, shard_count=3) for r in range(3)]
    atomic_loaded = VoxelBlockGrid(O.VS, 8, capacity_blocks=1 << 15)   # a map loads into either mode
    for x in [one, atomic_loaded] + three:
        x.load_state(path)
    _same(atomic_loaded, first)
    _feed_frames([one] + three, fr[5:])
    _same(one, whole)
    ref = sort_dump(whole.dump_blocks())
    row = {tuple(k): i for i, k in enumerate(ref["keys"].tolist())}
    for s in three:
        d = sort_dump(s.dump_blocks())
        idx = np.array([row[tuple(k)] for k in d["keys"].tolist()], np.int64)
        _same(d, {k: v[idx] for k, v in ref.items()})


# ---- staged frames ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("flt", [False, True])
def test_staged_raw_frames_equal_host_prepared(flt):
    pytest.importorskip("cv2")
    from tests.test_gpu_grid_frames import host_prepare, tum_maps
    cfg = S.CONFIGS[O.FRAME_CFG]
    mx, my = tum_maps(cfg)
    staged, host = _grid(), _grid()
    staged.set_rectification(mx, my, swap_rb=True)
    scale = 1.0 / 5000.0
    for d, c, Twc in O.frames()[:4]:
        raw = np.round(d * 5000.0).astype(np.uint16)
        bgr = np.ascontiguousarray(c[..., ::-1])
        f = staged.set_frame(raw, bgr, depth_scale=scale, filter_shadow_points=flt)
        staged.integrate_rgbd(f.filtered_depth, f.color, O.frame_K(), Twc, max_depth=O.frame_max_depth())
        h = host_prepare(mx, my, raw, bgr, scale=scale, flt=flt)
        host.integrate_rgbd(h["filtered_depth"], h["color"], O.frame_K(), Twc, max_depth=O.frame_max_depth())
    _same(staged, host)


def test_edits_and_queries_on_real_frames_equal_numpy_grid():
    grid = _grid()
    _feed_frames([grid])
    G = _frames_oracle()
    d, c, Twc = O.frames()[3]
    cfg = S.CONFIGS[O.FRAME_CFG]
    Tcw = S.inv_T(Twc)
    K = (cfg.fx, cfg.fy, cfg.cx, cfg.cy)
    fr = CameraFrustrum(*K, cfg.width, cfg.height, Tcw, depth_max=3.0, depth_min=0.05)
    out = grid.get_voxels_in_camera_frustrum(fr, min_count=2)
    assert len(out.points) > 1000
    assert np.array_equal(_rows(out.points, out.colors),
                          _rows(*G.get_voxels_in_frustum(fr._args()[0], cfg.width, cfg.height, Tcw, 3.0, 0.05, 2)))
    mean = (G.pos / G.count[:, None].astype(np.float32)).astype(np.float64)
    lo, hi = np.percentile(mean, 20, axis=0), np.percentile(mean, 70, axis=0)
    bb = np.concatenate([lo, hi])
    ob = grid.get_voxels_in_bb(BoundingBox3D(*bb), min_count=1)
    assert len(ob.points) > 100
    assert np.array_equal(_rows(ob.points, ob.colors), _rows(*G.get_voxels_in_bb(bb, 1)))
    grid.remove_low_count_voxels(3)
    G.remove_low_count_voxels(3)
    _same(grid, _oracle_dump(G), ("keys", "count", "pos_sum", "col_sum"))
    carve_depth = np.where(d > 0, d * np.float32(1.25), d).astype(np.float32)   # the map lies in front of it
    grid.carve(fr, carve_depth, depth_threshold=0.03)
    gone = G.carve(fr._args()[0], cfg.width, cfg.height, Tcw, carve_depth, 0.03, 3.0, 0.05)
    assert len(gone) > 100
    _same(grid, _oracle_dump(G), ("keys", "count", "pos_sum", "col_sum"))


# ---- the modes agree where they must ----------------------------------------------------------------------------

def test_modes_bit_equal_on_exact_scenes():
    """Dyadic scenes, whose float32 sums are exact in any order: both modes hold the same bits."""
    a, b = VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=1 << 12), _grid(E.VS_EXACT, capacity_blocks=1 << 12)
    for _, p, c in E.exact_batches():
        a.integrate(p, c)
        b.integrate(p, c)
    _same(a, b)
    a, b = VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=1 << 12), _grid(E.VS_EXACT, capacity_blocks=1 << 12)
    for d, c, Twc in E.rgbd_frames():
        for x in (a, b):
            x.integrate_rgbd(d, c, E.RGBD_K, Twc)
    _same(a, b)


# ---- API and plugin ---------------------------------------------------------------------------------------------

def test_api_default_toggle_null_and_point_limit():
    L = _lib.load()
    assert L.b2v_version() >= 109
    assert L.b2v_grid_set_input_order_sums(None, 1) == _lib.B2V_ERR_INVALID_ARGUMENT
    g = VoxelBlockGrid(O.VS, 8, capacity_blocks=1 << 12)
    assert not g.input_order_sums
    with pytest.raises(AttributeError):
        g.input_order_sums = True
    p, _, c = O.stress_scene()
    # enabled mid-stream: applies from the next call, and clear() keeps it
    assert L.b2v_grid_set_input_order_sums(g._h, 1) == _lib.B2V_OK
    g.integrate(p, c)
    g.clear()
    g.integrate(p, c)
    _same(g, _oracle_dump(O.numpy_grid_of([(p, c)])), ("keys", "count", "pos_sum", "col_sum"))
    before = sort_dump(g.dump_blocks())
    # past 0x7FFFFFF0 points: rejected before anything is read, the grid unchanged
    rc = L.b2v_grid_integrate_ex(g._h, C.c_void_p(p.ctypes.data), 0, None, 0, 0x7FFFFFF1)
    assert rc == _lib.B2V_ERR_INVALID_ARGUMENT and "0x7FFFFFF0" in L.b2v_grid_last_error(g._h).decode()
    _same(g, before)


def _run_voxel_plugin(**kw):
    from tests import plugin_standins as P
    cfg = S.CONFIGS["T0"]
    from types import SimpleNamespace
    cam = SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)
    Cls = P.standalone_voxel_grid_integrator_class()
    integ = Cls(cam, P.DatasetEnvironmentType.INDOOR, None, "B200_VOXEL_GRID", kVolumetricIntegrationVoxelLength=0.015,
                **kw)
    frames = []
    for i in range(4):
        d, c, T = S.render_frame(cfg, i)
        frames.append((d, c, T))
        integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(
            id=i, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=d))
        integ.step()
    integ.add_update_output_task()
    integ.step()
    out = None
    while True:
        o = integ.pop_output()
        if o is None:
            break
        out = o
    return integ, frames, out


@pytest.mark.parametrize("on", [True, False])
def test_voxel_grid_plugin_parameter(on):
    kw = {"kVolumetricIntegrationB200InputOrderSums": True} if on else {}
    integ, frames, out = _run_voxel_plugin(**kw)
    assert integ.volume.input_order_sums is on
    cfg = S.CONFIGS["T0"]
    ref = VoxelBlockGrid(0.015, 8, capacity_blocks=1 << 17, input_order_sums=True)
    for d, c, T in frames:   # the plugin's host path: shadow filter, depth truncation 4 m
        ref.integrate_rgbd(d, c, cfg.K, np.linalg.inv(T), max_depth=4.0, filter_shadow_points=True)
    if on:
        _same(integ.volume, ref)
        v = ref.get_voxels(min_count=3)
        assert np.array_equal(_rows(out.point_cloud.points, out.point_cloud.colors), _rows(v.points, v.colors))
    else:
        _same_counts(integ.volume, ref)
    integ.quit()
