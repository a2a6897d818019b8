"""GPU: point-average and semantic grids sharded by block-key hash (`shard_rank` / `shard_count`, DESIGN.md §7).

For N in {1, 2, 3, 4, 8}, N shard grids and one unsharded grid live on one device and are fed the same inputs.  Every
shard must hold only the blocks it owns, the shards' blocks must partition the unsharded grid's, and every block must
equal, bit for bit, the unsharded grid's block.  The point-grid scenes keep every float32 sum exact in any order
(tests/_grid_prep_scenes.py); the semantic grids update each voxel in input order, so they are exact on any input.  The
association runs in its two steps on the shards (`sharding.association_votes` on every shard, then
`sharding.resolve_association` of all shards' triples on every shard) and must give every shard the unsharded map."""

import os
import socket

import numpy as np
import pytest
import torch

from pyslam_b200 import (BoundingBox3D, CameraFrustrum, VoxelBlockGrid, VoxelBlockSemanticGrid,
                         VoxelBlockSemanticProbabilisticGrid, remap_instance_ids, sharding)
from pyslam_b200 import synthetic as S
from pyslam_b200.volume import _as_K4, segment_min_count, segments
from tests import _grid_prep_scenes as E
from tests._util import GOLDEN, sort_dump
from tests.test_gpu_grid_growth import _many_blocks, _rgbd_frames, _rows

pytestmark = pytest.mark.gpu
f32 = np.float32
WORLDS = [1, 2, 3, 4, 8]
SEM = {"vote": VoxelBlockSemanticGrid, "prob": VoxelBlockSemanticProbabilisticGrid}
POINT_KEYS = ("keys", "hashes", "count", "pos_sum", "col_sum")
SEM_KEYS = ("keys", "hashes", "count", "pos_sum", "col_sum", "object_id", "class_id", "confidence", "aux", "lab_obj",
            "lab_cls", "lab_logp")
ASSOC = dict(depth_threshold=0.08, do_carving=True)
VOTE = dict(min_vote_ratio=0.5, min_votes=3)


def _grids(cls, world, *args, **kw):
    """(unsharded grid, [shard 0 .. shard world-1])"""
    return cls(*args, **kw), [cls(*args, shard_rank=r, shard_count=world, **kw) for r in range(world)]


def _dump(grid):
    return grid.dump_blocks(8) if isinstance(grid, VoxelBlockSemanticGrid) else grid.dump_blocks()


def _same_blocks(single, shards):
    """Partition by owner, and every block equal to the unsharded grid's (label overflows summed over ranks)."""
    world = len(shards)
    dumps = [_dump(s) for s in shards]
    for r, d in enumerate(dumps):
        assert (sharding.owner_of(d["keys"], world) == r).all(), r
    keys = np.concatenate([d["keys"] for d in dumps])
    assert len(np.unique(keys, axis=0)) == len(keys)
    whole = sort_dump(_dump(single))
    merged = sharding.merge_dumps(dumps)
    names = SEM_KEYS if isinstance(single, VoxelBlockSemanticGrid) else POINT_KEYS
    for k in names:
        assert np.array_equal(merged[k], whole[k], equal_nan=True), k
    assert sum(s.num_blocks() for s in shards) == single.num_blocks()
    if isinstance(single, VoxelBlockSemanticGrid):
        assert sum(s.label_overflows() for s in shards) == single.label_overflows()
    return whole


def _cat(parts):
    """The read-outs of every shard concatenated rank-major, like `sharding.get_voxels_sharded` on dst."""
    out = parts[0]
    for k in ("points", "colors", "class_ids", "object_ids", "confidences"):
        if getattr(out, k) is not None:
            setattr(out, k, np.concatenate([np.asarray(getattr(p, k)) for p in parts]))
    return out


def _same_readout(a, b):
    """Equal as sets keyed by voxel (a voxel's mean position is unique), with exact values."""
    assert len(a.points) == len(b.points)
    ka, kb = np.lexsort(np.asarray(a.points).T[::-1]), np.lexsort(np.asarray(b.points).T[::-1])
    for k in ("points", "colors", "class_ids", "object_ids", "confidences"):
        if getattr(b, k) is not None:
            assert np.array_equal(np.asarray(getattr(a, k))[ka], np.asarray(getattr(b, k))[kb]), k


# ---- 1-2. point-average grid -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("world", WORLDS)
def test_point_grid_points_and_colour_kinds(world):
    p, fc = _many_blocks(0, 1500)
    u8 = (np.random.default_rng(5).integers(0, 2, p.shape) * 255).astype(np.uint8)
    for cols in (fc, u8, None):
        single, shards = _grids(VoxelBlockGrid, world, E.VS_EXACT, 8, capacity_blocks=1 << 12)
        for part in np.array_split(np.arange(len(p)), 3):
            for g in [single] + shards:
                g.integrate(p[part], None if cols is None else cols[part])
        _same_blocks(single, shards)
        for m in (1, 2):
            _same_readout(_cat([s.get_voxels(m) for s in shards]), single.get_voxels(m))
    q = E.float64_points()   # float64 points: keys from the float64 coordinates
    single, shards = _grids(VoxelBlockGrid, world, 0.005, 8, capacity_blocks=1 << 15)
    for g in [single] + shards:
        g.integrate(q)
    _same_blocks(single, shards)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("flt", [False, True])
def test_point_grid_rgbd_and_staged_frames(world, flt):
    frames, K = _rgbd_frames()
    for staged in (False, True):
        single, shards = _grids(VoxelBlockGrid, world, E.VS_EXACT, 8, capacity_blocks=1 << 15)
        for d, c, Twc in frames:
            for g in [single] + shards:
                if staged:
                    f = g.set_frame(d, c, filter_shadow_points=flt)
                    g.integrate_rgbd(f.filtered_depth, f.color, K, Twc)
                else:
                    g.integrate_rgbd(d, c, K, Twc, filter_shadow_points=flt)
        _same_blocks(single, shards)


@pytest.mark.parametrize("world", WORLDS)
def test_point_grid_queries_carve_and_low_count(world):
    fp, fc = _many_blocks(6, 1200, lo=-20, hi=20)
    T = E.cam_poses()[0]
    fr = CameraFrustrum(*E.CAM_K, E.CAM_W, E.CAM_H, T, depth_max=E.DEPTH_MAX, depth_min=E.DEPTH_MIN)
    probe = E.frustum_probe_points(T)
    pcols = E.dyadic_colors(np.random.default_rng(1), len(probe))
    cpts, img = E.carve_scene(T)
    single, shards = _grids(VoxelBlockGrid, world, E.VS_EXACT, 8, capacity_blocks=1 << 13)
    for g in [single] + shards:
        g.integrate(fp, fc)
        g.integrate(probe, pcols)
        g.integrate(cpts)
    for bb in E.BOXES:
        box = BoundingBox3D(*bb)
        _same_readout(_cat([s.get_voxels_in_bb(box, 1) for s in shards]), single.get_voxels_in_bb(box, 1))
    for m in (1, 2):
        _same_readout(_cat([s.get_voxels_in_camera_frustrum(fr, m) for s in shards]),
                      single.get_voxels_in_camera_frustrum(fr, m))
    for g in [single] + shards:
        g.carve(fr, img, depth_threshold=E.CARVE_THR)
    _same_blocks(single, shards)
    for g in [single] + shards:
        g.integrate(fp[:300], fc[:300])
        g.remove_low_count_voxels(4)
    _same_blocks(single, shards)
    assert sum(s.size() for s in shards) == single.size()


# ---- 3. semantic grids ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("tag", ["vote", "prob"])
def test_semantic_golden_stream(tag, world):
    g = np.load(os.path.join(GOLDEN, "semantic_T0.npz"))
    single, shards = _grids(SEM[tag], world, float(g["voxel_size"]), 8, capacity_blocks=1024)
    for grid in [single] + shards:
        grid.set_depth_threshold(float(g[f"{tag}_depth_threshold"]))
        grid.set_depth_decay_rate(float(g[f"{tag}_depth_decay_rate"]))
        for i in range(int(g["n_frames"])):
            grid.integrate(g[f"{tag}_points_{i}"], g[f"{tag}_colors_{i}"], g[f"{tag}_cls_{i}"], g[f"{tag}_inst_{i}"],
                           g[f"{tag}_depths_{i}"])
    _same_blocks(single, shards)


def _associate(single, shards, fr, cls, inst, depth):
    """The unsharded association and the two-step association of the shards; every shard's map, next_object_id and
    voxels must equal the unsharded grid's."""
    want = single.assign_object_ids_to_instance_ids(fr, cls, inst, depth, **ASSOC, **VOTE)
    votes = [sharding.association_votes(s, fr, cls, inst, depth, ASSOC["depth_threshold"], ASSOC["do_carving"])
             for s in shards]
    for v in votes:
        assert v.dtype == np.int32 and v.shape[1] == 3 and (v[:, 2] > 0).all()
        assert len(np.unique(v[:, :2], axis=0)) == len(v)
    for s in shards:
        got = sharding.resolve_association(s, votes[::-1], cls, inst, **VOTE)   # the order of the ranks is free
        assert got == want
        assert s.get_next_object_id() == single.get_next_object_id()
    return want


def _c3_frames(n):
    cfg = S.CONFIGS["C3"]
    out = []
    for i in range(n):
        d, c, Tcw = S.render_frame(cfg, 12 * i)
        cls = S.render_class_ids(cfg, 12 * i).astype(np.int32)
        inst = np.where(cls % 3 == 0, -1, cls * 7 + (np.arange(cls.shape[1])[None, :] // 400) + i % 2)
        inst[:40] = 0   # instance 0 takes object id 0
        out.append((d, c, Tcw, cls, inst.astype(np.int32)))
    return cfg, out


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("tag", ["vote", "prob"])
def test_semantic_c3_association_frame_by_frame(tag, world):
    """8 C3 frames through the plugin's loop: association (with carving) -> remap_instance_ids of the staged frame ->
    integrate_rgbd with the object image, on every grid."""
    cfg, frames = _c3_frames(8)
    K4 = _as_K4(cfg.K)
    single, shards = _grids(SEM[tag], world, 0.015, 8, capacity_blocks=1 << 10, max_capacity_blocks=1 << 17)
    for grid in [single] + shards:
        grid.set_depth_threshold(1.5)
    n_maps = 0
    for d, c, Tcw, cls, inst in frames:
        fr = CameraFrustrum(*K4, d.shape[1], d.shape[0], Tcw, depth_max=cfg.depth_trunc, depth_min=1e-2)
        staged = [g.set_frame(d, c, cls, inst) for g in [single] + shards]
        want = single.assign_object_ids_to_instance_ids(fr, staged[0].class_image, staged[0].instance_image,
                                                        staged[0].depth, **ASSOC, **VOTE)
        votes = [sharding.association_votes(s, fr, f.class_image, f.instance_image, f.depth,
                                            ASSOC["depth_threshold"], ASSOC["do_carving"])
                 for s, f in zip(shards, staged[1:])]
        for s, f in zip(shards, staged[1:]):
            assert sharding.resolve_association(s, votes, f.class_image, f.instance_image, **VOTE) == want
            assert s.get_next_object_id() == single.get_next_object_id()
        n_maps += any(o > 0 for o in want.values())
        objs = [g.remap_instance_ids() for g in [single] + shards]
        ref = objs[0].numpy()
        for o in objs[1:]:
            assert np.array_equal(o.numpy(), ref)
        _same_blocks(single, shards)   # the association's carving and deferred ids
        for g, f, o in zip([single] + shards, staged, objs):
            g.integrate_rgbd(f.depth, f.color, cfg.K, S.inv_T(Tcw), f.class_image, o, max_depth=cfg.depth_trunc)
        _same_blocks(single, shards)
    assert n_maps >= 4 and single.get_next_object_id() > 2 and single.num_blocks() > 500


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("tag", ["vote", "prob"])
def test_semantic_segments_readouts_and_edits(tag, world):
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    vs, K = float(g["voxel_size"]), g["K"]
    single, shards = _grids(SEM[tag], world, vs, 8, capacity_blocks=1024)
    for i in range(int(g["n_frames"])):
        d, c, T = g[f"depth_{i}"], g[f"color_{i}"], g[f"Tcw_{i}"]
        cls_img, inst_img = g[f"class_image_{i}"], g[f"instance_image_{i}"]
        fr = CameraFrustrum(K[0], K[1], K[2], K[3], d.shape[1], d.shape[0], T, depth_max=8.0, depth_min=1e-2)
        m = _associate(single, shards, fr, cls_img, inst_img, d)
        obj_img = remap_instance_ids(inst_img, m)
        for grid in [single] + shards:
            grid.integrate_rgbd(d, c, K, np.linalg.inv(T), cls_img, obj_img, max_depth=4.0)
    _same_blocks(single, shards)
    for by_class in (False, True):
        for mc, conf in ((1, 0.0), (2, 0.3)):
            want = single.get_class_segments(mc, conf) if by_class else single.get_object_segments(mc, conf)
            got = segments(_cat([s.get_voxels(segment_min_count(mc), conf) for s in shards]), by_class)
            lw = want.class_vector if by_class else want.object_vector
            lg = got.class_vector if by_class else got.object_vector
            assert len(lw) == len(lg) > 0
            for x, y in zip(lg, lw):
                # an object segment's class id is its first voxel's, and the read-out order is unspecified
                assert (x.confidence_min, x.confidence_max) == (y.confidence_min, y.confidence_max)
                assert not by_class or x.class_id == y.class_id
                assert np.array_equal(_rows(np.asarray(x.points), np.asarray(x.colors)),
                                      _rows(np.asarray(y.points), np.asarray(y.colors)))
                if not by_class:
                    assert x.object_id == y.object_id
                    bx, by = x.oriented_bounding_box, y.oriented_bounding_box
                    assert np.allclose(bx.center, by.center, rtol=0, atol=1e-9)
                    assert np.allclose(bx.size, by.size, rtol=0, atol=1e-9)
                    assert np.allclose(np.abs(np.sum(bx.R * by.R, axis=0)), 1.0, rtol=0, atol=1e-9)
    d, T = g["depth_0"], g["Tcw_0"]
    fr = CameraFrustrum(K[0], K[1], K[2], K[3], d.shape[1], d.shape[0], T, depth_max=3.0, depth_min=0.1)
    bb = BoundingBox3D(-0.5, -0.5, 0.0, 1.0, 1.0, 2.0)
    for mc, conf in ((1, 0.0), (2, 0.5)):
        _same_readout(_cat([s.get_voxels(mc, conf) for s in shards]), single.get_voxels(mc, conf))
        _same_readout(_cat([s.get_voxels_in_bb(bb, mc, conf) for s in shards]), single.get_voxels_in_bb(bb, mc, conf))
        _same_readout(_cat([s.get_voxels_in_camera_frustrum(fr, mc, conf) for s in shards]),
                      single.get_voxels_in_camera_frustrum(fr, mc, conf))
    obj = [int(o) for o in np.unique(sort_dump(single.dump_blocks(1))["object_id"]) if o > 0]
    assert len(obj) >= 3
    edits = [lambda x: x.merge_segments(obj[0], obj[1]), lambda x: x.remove_segment(obj[2]),
             lambda x: x.carve(fr, d * 1.5, depth_threshold=0.05), lambda x: x.remove_low_count_voxels(2),
             lambda x: x.remove_low_confidence_segments(1)]
    for edit in edits:
        for grid in [single] + shards:
            edit(grid)
        _same_blocks(single, shards)


# ---- 5. growth --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("world", [2, 3, 8])
def test_grown_shards_equal_fixed_shards(world):
    p, fc = _many_blocks(2, 2500)
    for start in (4, 16):
        _, grown = _grids(VoxelBlockGrid, world, E.VS_EXACT, 8, capacity_blocks=start, max_capacity_blocks=1 << 13)
        single, fixed = _grids(VoxelBlockGrid, world, E.VS_EXACT, 8, capacity_blocks=1 << 13)
        for part in np.array_split(np.arange(len(p)), 4):
            for x in [single] + grown + fixed:
                x.integrate(p[part], fc[part])
        assert all(x.capacity()[1] >= 1 for x in grown) and single.num_blocks() == 2500
        _same_blocks(single, grown)
        _same_blocks(single, fixed)
    g = np.load(os.path.join(GOLDEN, "semantic_T0.npz"))
    for tag in ("vote", "prob"):
        _, grown = _grids(SEM[tag], world, float(g["voxel_size"]), 8, capacity_blocks=4, max_capacity_blocks=1024)
        single, fixed = _grids(SEM[tag], world, float(g["voxel_size"]), 8, capacity_blocks=1024)
        for x in [single] + grown + fixed:
            for i in range(int(g["n_frames"])):
                x.integrate(g[f"{tag}_points_{i}"], g[f"{tag}_colors_{i}"], g[f"{tag}_cls_{i}"], g[f"{tag}_inst_{i}"],
                            g[f"{tag}_depths_{i}"])
        _same_blocks(single, grown)
        _same_blocks(single, fixed)


# ---- 6. arguments -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["point", "vote", "prob"])
def test_set_shard_arguments_and_a_stale_resolve(kind):
    make = (lambda **kw: VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=1 << 12, **kw)) if kind == "point" else \
        (lambda **kw: SEM[kind](E.VS_EXACT, 8, capacity_blocks=1 << 12, **kw))
    for rank, count in ((0, 0), (-1, 2), (2, 2), (3, 1)):
        with pytest.raises(RuntimeError, match="set_shard"):
            make(shard_rank=rank, shard_count=count)
    p, c = _many_blocks(4, 300)
    grid = make(shard_rank=1, shard_count=3)
    grid.integrate(p, c)
    before = sort_dump(_dump(grid))
    for rank, count in ((0, 1), (0, 2), (1, 3), (5, 3), (0, 0)):
        with pytest.raises(RuntimeError, match="set_shard"):
            grid.set_shard(rank, count)
    assert (grid.shard_rank, grid.shard_count) == (1, 3)
    after = sort_dump(_dump(grid))
    assert all(np.array_equal(before[k], after[k], equal_nan=True) for k in before)
    assert (sharding.owner_of(after["keys"], 3) == 1).all()
    grid.clear()                                   # clear keeps the setting; an empty grid takes a new one
    grid.integrate(p, c)
    assert (sharding.owner_of(_dump(grid)["keys"], 3) == 1).all()
    grid.clear()
    grid.set_shard(0, 2)
    grid.integrate(p, c)
    assert (sharding.owner_of(_dump(grid)["keys"], 2) == 0).all()
    if kind == "point":
        return
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    K, d, T = g["K"], g["depth_0"], g["Tcw_0"]
    cls, inst = g["class_image_0"], g["instance_image_0"]
    fr = CameraFrustrum(K[0], K[1], K[2], K[3], d.shape[1], d.shape[0], T, depth_max=8.0, depth_min=1e-2)
    grid = SEM[kind](float(g["voxel_size"]), 8, capacity_blocks=1024, shard_rank=0, shard_count=2)
    grid.integrate_rgbd(d, g["color_0"], K, np.linalg.inv(T), cls, inst, max_depth=4.0)
    for between in (lambda: grid.integrate_rgbd(d, g["color_0"], K, np.linalg.inv(T), cls, inst, max_depth=4.0),
                     lambda: grid.remove_low_count_voxels(1), lambda: grid.clear(),
                     lambda: grid.carve(fr, d, 0.05),
                     lambda: sharding.resolve_association(grid, [v], cls, inst)):
        v = sharding.association_votes(grid, fr, cls, inst, d, 0.08, False)
        between()
        with pytest.raises(RuntimeError, match="no votes"):
            sharding.resolve_association(grid, [v], cls, inst)


# ---- 7. the collective wrappers: gloo with two processes on one GPU, NCCL with two GPUs --------------------------------

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, backend, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    try:
        g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
        vs, K = float(g["voxel_size"]), g["K"]
        ok = True
        grid = VoxelBlockSemanticProbabilisticGrid(vs, 8, capacity_blocks=1024, device=dev, shard_rank=rank,
                                                   shard_count=world)
        single = VoxelBlockSemanticProbabilisticGrid(vs, 8, capacity_blocks=1024, device=dev) if rank == 0 else None
        for i in range(int(g["n_frames"])):
            d, c, T = g[f"depth_{i}"], g[f"color_{i}"], g[f"Tcw_{i}"]
            cls, inst = g[f"class_image_{i}"], g[f"instance_image_{i}"]
            fr = CameraFrustrum(K[0], K[1], K[2], K[3], d.shape[1], d.shape[0], T, depth_max=8.0, depth_min=1e-2)
            m = sharding.assign_object_ids_to_instance_ids_sharded(grid, fr, cls, inst, d, **ASSOC, **VOTE)
            if single is not None:
                ok = ok and m == single.assign_object_ids_to_instance_ids(fr, cls, inst, d, **ASSOC, **VOTE)
            for x in (grid, single):
                if x is not None:
                    x.integrate_rgbd(d, c, K, np.linalg.inv(T), cls, remap_instance_ids(inst, m), max_depth=4.0)
        fr = CameraFrustrum(K[0], K[1], K[2], K[3], d.shape[1], d.shape[0], T, depth_max=3.0, depth_min=0.1)
        bb = BoundingBox3D(-0.5, -0.5, 0.0, 1.0, 1.0, 2.0)
        got = [sharding.get_voxels_sharded(grid, 1, 0.0), sharding.get_voxels_in_bb_sharded(grid, bb, 1, 0.0),
               sharding.get_voxels_in_camera_frustrum_sharded(grid, fr, 1, 0.0)]
        segs = [sharding.get_object_segments_sharded(grid, 1, 0.0), sharding.get_class_segments_sharded(grid, 1, 0.0)]
        nb, size = sharding.num_blocks_sharded(grid), sharding.size_sharded(grid)
        pgrid = VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=1 << 12, device=dev, shard_rank=rank, shard_count=world)
        p, pc = _many_blocks(0, 800)
        pgrid.integrate(p, pc)
        pv = sharding.get_voxels_sharded(pgrid, 1)
        pnb = sharding.num_blocks_sharded(pgrid)
        if rank == 0:
            want = [single.get_voxels(1, 0.0), single.get_voxels_in_bb(bb, 1, 0.0),
                    single.get_voxels_in_camera_frustrum(fr, 1, 0.0)]
            for a, b in zip(got, want):
                _same_readout(a, b)
            for by_class, sg in ((False, segs[0]), (True, segs[1])):
                sw = single.get_class_segments(1, 0.0) if by_class else single.get_object_segments(1, 0.0)
                la = sg.class_vector if by_class else sg.object_vector
                lb = sw.class_vector if by_class else sw.object_vector
                ok = ok and len(la) == len(lb) > 0 and all(
                    np.array_equal(_rows(x.points, x.colors), _rows(y.points, y.colors))
                    for x, y in zip(la, lb))
            ok = ok and nb == single.num_blocks() and size == single.size()
            ps = VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=1 << 12, device=dev)
            ps.integrate(p, pc)
            _same_readout(pv, ps.get_voxels(1))
            ok = ok and pnb == ps.num_blocks()
            q.put("ok" if ok else "mismatch")
        else:
            q.put("ok" if all(x is None for x in got + segs + [pv]) else "mismatch")
    except Exception as e:   # reported through the queue: the parent asserts on it
        q.put(f"{type(e).__name__}: {e}")
    finally:
        dist.destroy_process_group()


def _two_processes(backend):
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=300) for _ in range(world)]
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.terminate()
                p.join()
    assert res == ["ok", "ok"]
    assert all(p.exitcode == 0 for p in procs)


def test_gloo_two_processes_on_one_gpu():
    _two_processes("gloo")


def test_nccl_two_gpus():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _two_processes("nccl")
