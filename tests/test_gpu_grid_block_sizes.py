"""GPU: the point-average and semantic grids at every supported block size B (1, 2, 16, and 8 as the control).

A voxel's state does not depend on B, so the B = 8 oracles pin every value: `oracle.numpy_grid` keeps its state per
voxel key and `tests/_block_sizes.grid_dump` lays it out in blocks of side B (block key floor_div(v, B), local index
lx + B ly + B^2 lz); the semantic oracle's B = 8 dump is re-keyed by voxel the same way.  Dumps (keys, BlockKeyHash,
counts, sums, labels) must be equal bit for bit after every call, on the exact-sum scenes of tests/test_gpu_grid_prep_edges.py
and tests/test_gpu_semantic_edges.py."""

import numpy as np
import pytest

import oracle
from pyslam_b200 import (BoundingBox3D, CameraFrustrum, VoxelBlockGrid, VoxelBlockSemanticGrid,
                         VoxelBlockSemanticProbabilisticGrid, sharding)
from tests import _block_sizes as BS
from tests import _grid_prep_scenes as E
from tests import _semantic_scenes as SC
from tests._util import sort_dump

pytestmark = pytest.mark.gpu
f32 = np.float32
SIZES = (1, 2, 16)
KINDS = ("voting", "probabilistic")


def _rows(p, c):
    a = np.concatenate([p, c], 1)
    return a[np.lexsort(a.T[::-1])]


def _same_voxels(got, ref):
    assert got.points.dtype == np.float32 and len(got.points) == len(ref[0])
    assert np.array_equal(_rows(got.points, got.colors), _rows(*ref))


def _same_dump(grid, G, B):
    d = sort_dump(grid.dump_blocks())
    r = BS.grid_dump(G, B)
    assert d["count"].shape[1:] == (B ** 3,)
    assert np.array_equal(d["keys"], r["keys"])
    assert np.array_equal(d["hashes"], BS.block_key_hash(d["keys"]))
    for f in ("count", "pos_sum", "col_sum"):
        assert np.array_equal(d[f], r[f]), f
    return d


# ---- point-average grid ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B", SIZES + (8,))
def test_exact_scene_after_every_call(B):
    grid = VoxelBlockGrid(E.VS_EXACT, B, capacity_blocks=1 << 15)
    assert grid.get_block_size() == B
    G = oracle.numpy_grid(E.VS_EXACT)
    for _, p, c in E.exact_batches():
        grid.integrate(p, c)
        G.integrate(p, c)
        _same_dump(grid, G, B)
    top = int(G.count.max())
    for m in (1, 2, top, top + 1):
        _same_voxels(grid.get_voxels(min_count=m), G.get_voxels(m))
    assert grid.size() == int((G.count > 0).sum())
    grid.remove_low_count_voxels(3)
    G.remove_low_count_voxels(3)
    _same_dump(grid, G, B)
    for m in (1, 3):
        _same_voxels(grid.get_voxels(min_count=m), G.get_voxels(m))


@pytest.mark.parametrize("B", SIZES)
def test_colour_kinds_float64_points_and_far_keys(B):
    rng = np.random.default_rng(3)
    p = E.edge_points_ref_voxel()
    c8 = rng.integers(0, 256, p.shape, dtype=np.uint8)
    for vs, pts, cols in ((E.VS_REF, p, c8), (E.VS_REF, p, None), (E.VS_EXACT, E.far_points(), None),
                          (0.005, E.float64_points(), None)):
        grid = VoxelBlockGrid(vs, B, capacity_blocks=1 << 16)
        G = oracle.numpy_grid(vs)
        grid.integrate(pts, cols)
        G.integrate(pts, cols)
        _same_dump(grid, G, B)
        _same_voxels(grid.get_voxels(1), G.get_voxels(1))


@pytest.mark.parametrize("B", SIZES)
def test_box_frustum_and_carve(B):
    for box, bb in enumerate(E.BOXES):
        pts = E.box_probe_points(bb)
        cols = E.dyadic_colors(np.random.default_rng(box), len(pts))
        grid = VoxelBlockGrid(E.VS_EXACT, B, capacity_blocks=1 << 14)
        G = oracle.numpy_grid(E.VS_EXACT)
        grid.integrate(pts, cols)
        G.integrate(pts, cols)
        _same_voxels(grid.get_voxels_in_bb(BoundingBox3D(*bb), min_count=1), G.get_voxels_in_bb(bb))
    for T in E.cam_poses():
        pts = E.frustum_probe_points(T)
        pts = np.concatenate([pts, pts[:20]])
        cols = E.dyadic_colors(np.random.default_rng(7), len(pts))
        grid = VoxelBlockGrid(E.VS_EXACT, B, capacity_blocks=1 << 14)
        G = oracle.numpy_grid(E.VS_EXACT)
        grid.integrate(pts, cols)
        G.integrate(pts, cols)
        fr = CameraFrustrum(*E.CAM_K, E.CAM_W, E.CAM_H, T, depth_max=E.DEPTH_MAX, depth_min=E.DEPTH_MIN)
        for m in (1, 2):
            _same_voxels(grid.get_voxels_in_camera_frustrum(fr, min_count=m),
                         G.get_voxels_in_frustum(E.CAM_K, E.CAM_W, E.CAM_H, T, E.DEPTH_MAX, E.DEPTH_MIN, m))
        pts, img = E.carve_scene(T)
        grid = VoxelBlockGrid(E.VS_EXACT, B, capacity_blocks=1 << 14)
        G = oracle.numpy_grid(E.VS_EXACT)
        grid.integrate(pts)
        G.integrate(pts)
        grid.carve(fr, img, depth_threshold=E.CARVE_THR)
        assert len(G.carve(E.CAM_K, E.CAM_W, E.CAM_H, T, img, E.CARVE_THR, E.DEPTH_MAX, E.DEPTH_MIN)) >= 10
        _same_dump(grid, G, B)


@pytest.mark.parametrize("B", SIZES)
@pytest.mark.parametrize("flt", [False, True])
def test_integrate_rgbd_and_staged_frames(B, flt):
    grid = VoxelBlockGrid(E.VS_EXACT, B, capacity_blocks=1 << 16)
    staged = VoxelBlockGrid(E.VS_EXACT, B, capacity_blocks=1 << 16)
    G = oracle.numpy_grid(E.VS_EXACT)
    for d, c, Twc in E.rgbd_frames():
        grid.integrate_rgbd(d, c, E.RGBD_K, Twc, filter_shadow_points=flt)
        f = staged.set_frame(d, c, filter_shadow_points=flt)
        staged.integrate_rgbd(f.filtered_depth if flt else f.depth, f.color, E.RGBD_K, Twc)
        dd = oracle.numpy_shadow_filter(d, 2, 2, -1.0)[0] if flt else d
        G.integrate(*E.rgbd_points(dd, c, E.RGBD_K, Twc))
        _same_dump(grid, G, B)
        _same_dump(staged, G, B)
    _same_voxels(grid.get_voxels(1), G.get_voxels(1))


# ---- semantic grids -------------------------------------------------------------------------------------------------

SEM_FIELDS = ("count", "pos_sum", "col_sum", "object_id", "class_id", "confidence", "aux", "lab_obj", "lab_cls",
              "lab_logp")
SEM_CLEARED = dict(count=0, pos_sum=0.0, col_sum=0.0, object_id=-1, class_id=-1, confidence=0.0, aux=0, lab_obj=-1,
                   lab_cls=-1, lab_logp=-np.inf)


def _sem_grid(kind, B, **kw):
    cls_t = VoxelBlockSemanticGrid if kind == "voting" else VoxelBlockSemanticProbabilisticGrid
    kw.setdefault("capacity_blocks", 1 << 14)
    return cls_t(SC.VS, B, **kw)


def _same_semantic(grids, ref8, B, where):
    """The B grids' dump equals the B = 8 reference dump (`ref8`, sorted, labels K = 8) re-keyed by voxel, in every
    voxel with observations (count > 0).  At B >= 8 the blocks are those of the B = 8 blocks; at B < 8 they lie inside
    them and cover every voxel with observations.  A voxel without observations holds the cleared state except, maybe,
    its object id: the edits apply to every voxel of every block (merge_segments(a, -1) gives every empty voxel the
    object a), and which empty voxels a grid holds, and since when, depends on B by that rule."""
    d = sharding.merge_dumps([sort_dump(g.dump_blocks(8)) for g in grids])
    assert np.array_equal(d["hashes"], BS.block_key_hash(d["keys"])), where
    vk, vals = BS.voxels(ref8, 8, SEM_FIELDS)
    seen = vals["count"] > 0
    k8 = np.asarray(ref8["keys"], np.int64)
    if B >= 8:
        blocks = np.unique(BS.block_keys_of(k8 * 8, B), axis=0).reshape(-1, 3)
    else:
        blocks = np.asarray(d["keys"], np.int64)
        inside = np.unique(BS.block_keys_of(blocks * B, 8), axis=0)
        assert set(map(tuple, inside.tolist())) <= set(map(tuple, k8.tolist())), where
        need = np.unique(BS.block_keys_of(vk[seen], B), axis=0)
        assert set(map(tuple, need.tolist())) <= set(map(tuple, blocks.tolist())), where
    exp = BS.layout(vk[seen], {f: v[seen] for f, v in vals.items()}, B, SEM_CLEARED, blocks=blocks)
    assert np.array_equal(d["keys"], exp["keys"]), where
    obs = (d["count"] > 0) | (exp["count"] > 0)
    for f in SEM_FIELDS:
        assert np.array_equal(d[f][obs], exp[f][obs]), (where, f)
        if f != "object_id":
            assert np.array_equal(d[f][~obs], exp[f][~obs]), (where, f, "empty")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("B", SIZES)
def test_semantic_scenes_equal_the_oracle_after_every_step(B, kind):
    """Every scene of tests/_semantic_scenes.py (eviction, softmax fold, edits, association edges, box / frustum /
    carve), each step checked against the B = 8 oracle re-keyed by voxel."""
    for name, scene in sorted(SC.scenes().items()):
        g = _sem_grid(kind, B)
        G = oracle.numpy_semantic_grid(SC.VS, kind)
        for t in (g, G):
            if "depth_threshold" in scene:
                t.set_depth_threshold(scene["depth_threshold"])
            if "depth_decay_rate" in scene:
                t.set_depth_decay_rate(scene["depth_decay_rate"])
        for i, (op, step) in enumerate(scene["steps"]):
            m = SC.apply(g, "gpu", op, step)
            mo = SC.apply(G, "oracle", op, step)
            if op == "assign":
                assert m == mo, (name, i)
            if scene.get("rtol"):
                continue
            _same_semantic([g], G.dump(), B, (name, kind, B, i, op))
            assert g.get_next_object_id() == G.next_object_id
            assert g.label_overflows() == G.label_overflows
        g.close()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("B", SIZES)
def test_semantic_random_stream_equals_block_size_8(B, kind):
    """The 50 000-point randomised stream with edits: the B grid equals a B = 8 grid voxel for voxel, bit for bit."""
    T0, _ = E.cam_poses()
    scene = SC.scene_random(T0)
    g, g8 = _sem_grid(kind, B), _sem_grid(kind, 8)
    for i, (op, step) in enumerate(scene["steps"]):
        assert SC.apply(g, "gpu", op, step) == SC.apply(g8, "gpu", op, step)
        _same_semantic([g], sort_dump(g8.dump_blocks(8)), B, (kind, B, i, op))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("B", SIZES)
def test_association_remap_and_rgbd_equal_block_size_8(B, kind):
    """Labelled RGBD frames through association -> remap_instance_ids -> integrate_rgbd: the same instance maps,
    next_object_id, voxels, and object and class segments as a B = 8 grid."""
    g, g8 = _sem_grid(kind, B), _sem_grid(kind, 8)
    cls_img, obj_img = SC.rgbd_labels()
    for i, (d, c, Twc) in enumerate(E.rgbd_frames(n=8)):
        fr = CameraFrustrum(*E.RGBD_K, d.shape[1], d.shape[0], np.linalg.inv(Twc), depth_max=10.0, depth_min=1e-2)
        maps = []
        for t in (g, g8):
            f = t.set_frame(d, c, cls_img, obj_img)
            maps.append(t.assign_object_ids_to_instance_ids(fr, f.class_image, f.instance_image, f.depth, 0.1, True,
                                                            0.5, 1))
            obj = t.remap_instance_ids() if i else f.instance_image
            t.integrate_rgbd(f.depth, f.color, E.RGBD_K, Twc, class_image=f.class_image, object_image=obj)
        assert maps[0] == maps[1], (kind, B, i)
        assert g.get_next_object_id() == g8.get_next_object_id()
        _same_semantic([g], sort_dump(g8.dump_blocks(8)), B, (kind, B, i))
    for seg in ("get_object_segments", "get_class_segments"):
        a, b = getattr(g, seg)(), getattr(g8, seg)()
        sa, sb = vars(a), vars(b)
        assert sa.keys() == sb.keys()
        for k in sa:
            xa, xb = sa[k], sb[k]
            if isinstance(xa, list):
                assert len(xa) == len(xb), (seg, k)
                for u, v in zip(xa, xb):
                    for name in ("object_id", "class_id", "confidence_min", "confidence_max"):
                        assert getattr(u, name, None) == getattr(v, name, None), (seg, name)
                    assert np.array_equal(_rows(u.points, u.colors), _rows(v.points, v.colors)), seg
                    if hasattr(u, "oriented_bounding_box") and u.oriented_bounding_box is not None:
                        for q in ("center", "extent", "R"):
                            if hasattr(u.oriented_bounding_box, q):
                                assert np.allclose(getattr(u.oriented_bounding_box, q),
                                                   getattr(v.oriented_bounding_box, q), rtol=0, atol=1e-9), (seg, q)


# ---- growth, ceiling, sharding, map state, invalid sizes ------------------------------------------------------------

@pytest.mark.parametrize("B", (2, 16))
def test_growth_equals_fixed_grid(B):
    _, p, c = E.exact_batches()[3]
    fixed = VoxelBlockGrid(E.VS_EXACT, B, capacity_blocks=1 << 12)
    grown = VoxelBlockGrid(E.VS_EXACT, B, capacity_blocks=4, max_capacity_blocks=1 << 12)
    for t in (fixed, grown):
        t.integrate(p, c)
    a, b = sort_dump(fixed.dump_blocks()), sort_dump(grown.dump_blocks())
    assert grown.capacity()[1] > 0
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    T0, _ = E.cam_poses()
    scene = SC.scene_random(T0)
    for kind in KINDS:
        fx, gr = _sem_grid(kind, B, capacity_blocks=1 << 12), _sem_grid(kind, B, capacity_blocks=4,
                                                                        max_capacity_blocks=1 << 12)
        for op, step in scene["steps"]:
            SC.apply(fx, "gpu", op, step)
            SC.apply(gr, "gpu", op, step)
        a, b = sort_dump(fx.dump_blocks(8)), sort_dump(gr.dump_blocks(8))
        for k in a:
            assert np.array_equal(a[k], b[k]), (kind, k)


@pytest.mark.parametrize("B", SIZES)
def test_ceiling(B):
    cap = 27
    k = np.stack(np.meshgrid(*[np.arange(3) - 1] * 3, indexing="ij"), -1).reshape(-1, 3)
    pts = ((k * B + 0.5) * E.VS_EXACT).astype(f32)
    grid = VoxelBlockGrid(E.VS_EXACT, B, capacity_blocks=cap)
    grid.integrate(pts)
    assert grid.num_blocks() == cap
    with pytest.raises(RuntimeError, match="block pool full"):
        grid.integrate(np.array([[5 * B * E.VS_EXACT, 0, 0]], f32))


@pytest.mark.parametrize("B", SIZES)
def test_three_shards_partition_the_grid(B):
    _, p, c = E.exact_batches()[3]
    whole = VoxelBlockGrid(E.VS_EXACT, B, capacity_blocks=1 << 12)
    whole.integrate(p, c)
    ref = sort_dump(whole.dump_blocks())
    parts = []
    for r in range(3):
        s = VoxelBlockGrid(E.VS_EXACT, B, capacity_blocks=1 << 12, shard_rank=r, shard_count=3)
        s.integrate(p, c)
        d = sort_dump(s.dump_blocks())
        assert np.all(BS.block_key_hash(d["keys"]) % np.uint64(3) == np.uint64(r))
        assert np.array_equal(sharding.owner_of(d["keys"], 3), np.full(len(d["keys"]), r))
        parts.append(d)
    m = sharding.merge_dumps(parts)
    for k in ref:
        assert np.array_equal(m[k], ref[k]), k


def test_map_state_round_trip_resharding_and_mismatch(tmp_path):
    _, p, c = E.exact_batches()[3]
    a = VoxelBlockGrid(E.VS_EXACT, 16, capacity_blocks=1 << 10)
    a.integrate(p, c)
    a.save_state(str(tmp_path / "g16.npz"))
    b = VoxelBlockGrid(E.VS_EXACT, 16, capacity_blocks=1 << 10)
    b.load_state(str(tmp_path / "g16.npz"))
    x, y = sort_dump(a.dump_blocks()), sort_dump(b.dump_blocks())
    for k in x:
        assert np.array_equal(x[k], y[k]), k
    g8 = VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=1 << 10)
    g8.integrate(p[:100], c[:100])
    before = sort_dump(g8.dump_blocks())
    with pytest.raises(ValueError):
        g8.load_state(str(tmp_path / "g16.npz"))
    after = sort_dump(g8.dump_blocks())
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    # 1 -> 3 at B = 2, semantic
    T0, _ = E.cam_poses()
    one = _sem_grid("probabilistic", 2)
    for op, step in SC.scene_random(T0)["steps"]:
        SC.apply(one, "gpu", op, step)
    one.save_state(str(tmp_path / "s2.npz"))
    parts = []
    for r in range(3):
        s = _sem_grid("probabilistic", 2, shard_rank=r, shard_count=3)
        s.load_state(str(tmp_path / "s2.npz"))
        parts.append(sort_dump(s.dump_blocks(8)))
    m, ref = sharding.merge_dumps(parts), sort_dump(one.dump_blocks(8))
    for k in ref:
        assert np.array_equal(m[k], ref[k]), k


@pytest.mark.parametrize("B", BS.INVALID_BLOCK_SIZES)
def test_invalid_block_sizes_raise(B):
    for make in (lambda: VoxelBlockGrid(0.05, B, capacity_blocks=64),
                 lambda: VoxelBlockSemanticGrid(0.05, B, capacity_blocks=64),
                 lambda: VoxelBlockSemanticProbabilisticGrid(0.05, B, capacity_blocks=64)):
        with pytest.raises(RuntimeError, match="1, 2, 8, 16"):
            make()


def test_semantic_capacity_bound_follows_the_block_size():
    for B in BS.BLOCK_SIZES:
        bound = min(1 << 30, (1 << 31) // B ** 3)
        with pytest.raises(RuntimeError):
            VoxelBlockSemanticGrid(0.05, B, capacity_blocks=bound + 1)


# ---- plugins --------------------------------------------------------------------------------------------------------

def _plugin_camera(cfg):
    from types import SimpleNamespace
    return SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)


def _run_semantic_plugin(B, gpu_rect, probabilistic):
    import os
    from tests import plugin_standins as P
    from tests._util import GOLDEN
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    r = np.load(os.path.join(GOLDEN, "remap_T0.npz"))
    from pyslam_b200 import synthetic as S
    kw = dict(kVolumetricIntegrationVoxelLength=float(g["voxel_size"]), kVolumetricIntegrationVoxelGridUseCarving=True,
              kVolumetricIntegrationVoxelGridShadowPointsFilter=False,
              kVolumetricIntegrationVoxelGridCarvingDepthThreshold=0.08, kVolumetricIntegrationBlockSize=B,
              kVolumetricIntegrationB200GpuRectify=gpu_rect, use_semantic_probabilistic=probabilistic,
              calib_maps=(r["map1"], r["map2"]))
    Cls = P.standalone_semantic_integrator_class()
    integ = Cls(_plugin_camera(S.CONFIGS["T0"]), P.DatasetEnvironmentType.INDOOR, None, "B200_SEMANTIC", **kw)
    maps = []
    for i in range(int(g["n_frames"])):
        integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(
            id=i, pose=g[f"Tcw_{i}"], img=np.ascontiguousarray(g[f"color_{i}"][..., ::-1]), depth=g[f"depth_{i}"],
            semantic_img=g[f"class_image_{i}"], semantic_instances_img=g[f"instance_image_{i}"]))
        integ.step()
        maps.append(integ.last_instance_map)
    integ.add_update_output_task()
    integ.step()
    out = None
    while True:
        o = integ.pop_output()
        if o is None:
            break
        out = o
    return integ, maps, out


@pytest.mark.parametrize("gpu_rect", [True, False])
@pytest.mark.parametrize("B", (2, 16))
def test_semantic_plugin_honours_the_block_size(B, gpu_rect):
    """The semantic plugin with kVolumetricIntegrationBlockSize B equals the B = 8 plugin: instance maps, object
    ids, the objects' points and class ids, and every observed voxel; the default capacity keeps the B = 8 budget."""
    if not gpu_rect:
        pytest.importorskip("cv2")
    from pyslam_b200 import integrator_semantic
    for probabilistic in (False, True):
        a, ma, oa = _run_semantic_plugin(B, gpu_rect, probabilistic)
        b, mb, ob = _run_semantic_plugin(8, gpu_rect, probabilistic)
        default = integrator_semantic.DEFAULT_PARAMETERS["kVolumetricIntegrationB200CapacityBlocks"]
        assert a.volume.get_block_size() == B and a.volume.capacity_blocks == -(-default * 512 // B ** 3)
        assert ma == mb and a.volume.get_next_object_id() == b.volume.get_next_object_id()
        _same_semantic([a.volume], sort_dump(b.volume.dump_blocks(8)), B, (B, gpu_rect, probabilistic))
        la = sorted(oa.objects.object_list, key=lambda o: o.object_id)
        lb = sorted(ob.objects.object_list, key=lambda o: o.object_id)
        assert len(la) == len(lb) > 0
        for x, y in zip(la, lb):
            assert (x.object_id, x.class_id) == (y.object_id, y.class_id)
            assert np.array_equal(_rows(x.points, x.colors), _rows(y.points, y.colors))
        a.quit()
        b.quit()


@pytest.mark.parametrize("gpu_rect", [True, False])
@pytest.mark.parametrize("B", (2, 16))
def test_voxel_grid_plugin_honours_the_block_size(B, gpu_rect):
    """The point-average plugin with kVolumetricIntegrationBlockSize B holds the B = 8 plugin's voxels with the same
    counts; the sums are float atomics in arrival order, so they agree to the tolerance of the grid tests."""
    if not gpu_rect:
        pytest.importorskip("cv2")
    import os
    from pyslam_b200 import synthetic as S
    from tests import plugin_standins as P
    from tests._util import GOLDEN
    r = np.load(os.path.join(GOLDEN, "remap_T0.npz"))
    cfg = S.CONFIGS["T0"]
    vox = []
    for b in (B, 8):
        Cls = P.standalone_voxel_grid_integrator_class()
        integ = Cls(_plugin_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_VOXEL_GRID",
                    kVolumetricIntegrationVoxelLength=0.03, kVolumetricIntegrationVoxelGridUseCarving=True,
                    kVolumetricIntegrationBlockSize=b, kVolumetricIntegrationB200GpuRectify=gpu_rect,
                    calib_maps=(r["map1"], r["map2"]))
        for i in range(4):
            d, c, T = S.render_frame(cfg, i)
            integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(
                id=i, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=d))
            integ.step()
        assert integ.volume.get_block_size() == b
        k, v = BS.voxels(sort_dump(integ.volume.dump_blocks()), b, ("count", "pos_sum"))
        seen = v["count"] > 0
        vox.append((k[seen], v["count"][seen], v["pos_sum"][seen]))
        integ.quit()
    (ka, ca, pa), (kb, cb, pb) = vox
    assert len(ka) > 1000
    assert np.array_equal(ka, kb) and np.array_equal(ca, cb)
    assert np.allclose(pa, pb, rtol=1e-5, atol=1e-6)
