"""GPU: sharded mesh / point-cloud extraction over the face-halo exchange (DESIGN.md §7).

N shard volumes live on one device in one process, fed the same frames (or the same uploaded blocks) as one unsharded
volume.  Their halo records must equal the numpy restatement bit for bit; the welded mesh pieces must equal the
unsharded `extract_mesh()` after `canonical_mesh`, with every triangle on exactly one rank; the point pieces must be
disjoint and together equal `extract_point_cloud()`; the live volumes must be left untouched."""

import os
import socket

import numpy as np
import pytest
import torch

import oracle
from pyslam_b200 import B200TsdfVolume, sharding
from pyslam_b200 import synthetic as S
from tests import _edge_scenes as E
from tests import _halo_oracle as H

pytestmark = pytest.mark.gpu


def _vol(cfg, cap=1 << 15, **kw):
    return B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=cap, **kw)


def _frames(name, n):
    cfg = S.CONFIGS[name]
    return cfg, [S.render_frame(cfg, i) for i in range(n)]


def _integrated(name, n, world, unit=16, **kw):
    cfg, frames = _frames(name, n)
    vols = [_vol(cfg, volume_unit_resolution=unit, **kw)] + \
        [_vol(cfg, shard_rank=r, shard_count=world, volume_unit_resolution=unit, **kw) for r in range(world)]
    for v in vols:
        d = np.stack([f[0] for f in frames])
        c = np.stack([f[1] for f in frames])
        T = np.stack([f[2] for f in frames])
        v.integrate_batch(d, c, cfg.K, T)
        v.synchronize()
    return cfg, vols[0], vols[1:]


def _uploaded(keys, vox, world, unit=16):
    cfg = S.CONFIGS["T0"]
    single = _vol(cfg, volume_unit_resolution=unit)
    single.upload_blocks(keys, vox)
    own = sharding.owner_of(keys, world)
    shards = []
    for r in range(world):
        v = _vol(cfg, shard_rank=r, shard_count=world, volume_unit_resolution=unit)
        v.upload_blocks(keys[own == r], vox[own == r])
        shards.append(v)
    return cfg, single, shards


def _run(shards, world):
    """(mesh pieces, point pieces, records per sender) of one in-process sharded extraction"""
    recs = [sharding.halo_records(v, world) for v in shards]
    mesh = [sharding.mesh_piece(v, [recs[s][r] for s in range(world)]) for r, v in enumerate(shards)]
    pts = [sharding.point_piece(v, [recs[s][r] for s in range(world)]) for r, v in enumerate(shards)]
    return mesh, pts, recs


def _canon(m):
    return oracle.canonical_mesh(m.vertices, m.vertex_colors, m.edge_ids, m.triangles)


def _by_key(d):
    o = np.lexsort(d["keys"].T[::-1])
    return {k: v[o] for k, v in d.items()}


def _check(single, shards, world):
    world = len(shards)
    before = [v.dump_blocks() for v in shards]
    mesh, pts, recs = _run(shards, world)
    # records: the numpy restatement of the shard's own dump (pool order), bit for bit
    for s, v in enumerate(shards):
        want = H.numpy_halo_records(before[s]["keys"], before[s]["vox"], world)
        for r in range(world):
            assert np.array_equal(recs[s][r][0].cpu().numpy(), want[r][0]), (s, r)
            assert np.array_equal(recs[s][r][1].cpu().numpy().view(np.uint32), want[r][1].view(np.uint32)), (s, r)
    # mesh: the pieces partition the triangles, and weld to the single-volume mesh
    full = single.extract_mesh()
    assert sum(len(m.triangles) for m in mesh) == len(full.triangles)
    for r, m in enumerate(mesh):
        assert H.triangle_roots_ok(m.edge_ids, m.triangles, before[r]["keys"])
    welded = sharding.weld(mesh, device=shards[0].device)
    a, b = _canon(welded), _canon(full)
    for k in b:
        assert np.array_equal(a[k], b[k]), k
    # the GPU weld equals its numpy restatement exactly (order included)
    nw = H.numpy_weld([dict(vertices=m.vertices, colors=m.vertex_colors, edges=m.edge_ids, triangles=m.triangles)
                       for m in mesh])
    assert np.array_equal(welded.edge_ids, nw["edges"]) and np.array_equal(welded.triangles, nw["triangles"])
    assert np.array_equal(welded.vertices, nw["vertices"]) and np.array_equal(welded.vertex_colors, nw["colors"])
    # point cloud: disjoint pieces whose union is the single-volume cloud, as a set keyed by (voxel, axis)
    fpc = single.extract_point_cloud()
    fe = np.asarray(single.extract_point_cloud_with_halo(np.zeros((0, 4), np.int32), np.zeros((0, 5), np.float32))
                    .edge_ids)
    assert len(fe) == len(fpc.points)
    ge = np.concatenate([p.edge_ids for p in pts])
    gp = np.concatenate([p.points for p in pts])
    gc = np.concatenate([p.colors for p in pts])
    assert len(np.unique(ge, axis=0)) == len(ge) == len(fe)
    o1, o2 = np.lexsort(ge.T[::-1]), np.lexsort(fe.T[::-1])
    assert np.array_equal(ge[o1], fe[o2])
    assert np.array_equal(gp[o1], fpc.points[o2]) and np.array_equal(gc[o1], fpc.colors[o2])
    # the live volumes are untouched
    for v, d in zip(shards, before):
        after = v.dump_blocks()
        assert all(np.array_equal(after[k], d[k]) for k in d)
    # determinism: a second extraction gives the same arrays in the same order
    mesh2, pts2, _ = _run(shards, world)
    for m1, m2 in zip(mesh + pts, mesh2 + pts2):
        for k in ("edge_ids",):
            assert np.array_equal(getattr(m1, k), getattr(m2, k))
    w2 = sharding.weld(mesh2, device=shards[0].device)
    assert np.array_equal(w2.vertices, welded.vertices) and np.array_equal(w2.triangles, welded.triangles)
    return welded


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_frames_T0(world):
    cfg, single, shards = _integrated("T0", 3, world)
    m = _check(single, shards, world)
    assert len(m.triangles) > 1000


@pytest.mark.parametrize("world", [2, 8])
def test_frames_C1_and_C2(world):
    for name, n in (("C1", 2), ("C2", 30)):
        cfg, single, shards = _integrated(name, n, world, cap=1 << 17)
        _check(single, shards, world)


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("shift", [0, (1 << 20) - 5, -(1 << 20)])
def test_random_blocks(world, shift):
    keys, vox = E.random_blocks(seed=3)
    keys = (keys + np.int32(shift)).astype(np.int32)
    cfg, single, shards = _uploaded(keys, vox, world)
    _check(single, shards, world)


@pytest.mark.parametrize("unit", [8, 16])
def test_unit_resolutions(unit):
    cfg, single, shards = _integrated("T0", 2, 4, unit=unit)
    _check(single, shards, 4)


def test_more_ranks_than_blocks_and_an_empty_rank():
    keys, vox = E.max_output_blocks()
    cfg, single, shards = _uploaded(keys[:3], vox[:3], 8)
    assert any(v.num_blocks() == 0 for v in shards)
    _check(single, shards, 8)


def test_growable_after_growth():
    cfg, single, shards = _integrated("T0", 3, 2, cap=64, max_capacity_blocks=1 << 15)
    assert all(v.capacity()[1] > 0 for v in shards)
    _check(single, shards, 2)


def test_extraction_does_not_change_later_integration():
    cfg, frames = _frames("T0", 4)
    a = _vol(cfg, shard_rank=0, shard_count=2)
    b = _vol(cfg, shard_rank=0, shard_count=2)
    other = _vol(cfg, shard_rank=1, shard_count=2)
    for v in (a, b, other):
        for d, c, T in frames[:2]:
            v.integrate(d, c, cfg.K, T)
        v.synchronize()
    _run([a, other], 2)
    for v in (a, b):
        for d, c, T in frames[2:]:
            v.integrate(d, c, cfg.K, T)
        v.synchronize()
    da, db = _by_key(a.dump_blocks()), _by_key(b.dump_blocks())   # pool order differs between two volumes
    assert all(np.array_equal(da[k], db[k]) for k in da)
    ma, mb = _canon(a.extract_mesh()), _canon(b.extract_mesh())
    assert all(np.array_equal(ma[k], mb[k]) for k in ma)


def test_single_volume_extraction_is_unchanged_by_a_halo_extraction():
    cfg, single, shards = _integrated("T0", 2, 2)
    m0 = single.extract_mesh()
    p0 = single.extract_point_cloud()
    _run(shards, 2)
    single.extract_mesh_with_halo(np.zeros((0, 4), np.int32), np.zeros((0, 5), np.float32))
    m1 = single.extract_mesh()
    p1 = single.extract_point_cloud()
    assert np.array_equal(m0.vertices, m1.vertices) and np.array_equal(m0.triangles, m1.triangles)
    assert np.array_equal(p0.points, p1.points)


def test_bad_records_are_rejected():
    cfg, single, shards = _integrated("T0", 1, 2)
    recs = sharding.halo_records(shards[0], 2)[1]
    h = recs[0].clone()
    h[0, 3] = 0
    with pytest.raises(RuntimeError, match="invalid mask"):
        shards[1].extract_mesh_with_halo(h, recs[1])
    h = torch.cat([recs[0], recs[0][:1]])
    x = torch.cat([recs[1], recs[1][:len(H.halo_shape(int(recs[0][0, 3])))]])
    with pytest.raises(RuntimeError, match="twice"):
        shards[1].extract_mesh_with_halo(h, x)


# ---- the collective wrappers: gloo with two processes on one GPU, NCCL with two GPUs ------------------------------

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
        cfg, frames = _frames("T0", 3)
        v = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 15, device=dev,
                           shard_rank=rank, shard_count=world)
        for d, c, T in frames:
            v.integrate(d, c, cfg.K, T)
        v.synchronize()
        mesh = sharding.extract_mesh_sharded(v, dst=0)
        pc = sharding.extract_point_cloud_sharded(v, dst=0)
        if rank == 0:
            s = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 15, device=dev)
            for d, c, T in frames:
                s.integrate(d, c, cfg.K, T)
            a, b = _canon(mesh), _canon(s.extract_mesh())
            ok = all(np.array_equal(a[k], b[k]) for k in b)
            fpc = s.extract_point_cloud()
            ok = ok and len(pc.points) == len(fpc.points) and np.array_equal(np.sort(pc.points, axis=0),
                                                                               np.sort(fpc.points, axis=0))
            ok = ok and min(v.last_halo_bytes) > 0
            q.put("ok" if ok else "mismatch")
        else:
            q.put("ok" if mesh is None and pc is None else "mismatch")
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
