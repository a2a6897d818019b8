"""CPU: the face-halo exchange of a sharded volume (DESIGN.md §7), restated in numpy and checked on per-rank twins.

Each rank's twin holds its own blocks plus the halo blocks the numpy records give it.  Its mesh must hold exactly the
triangles of the cubes rooted in its own blocks, and the welded pieces must equal the whole-map twin mesh; the point
pieces, rooted at the own blocks only, must partition the whole-map point cloud.  The gloo test runs the collective
wrapper's host logic (sizes, routing, reassembly on dst) with a stand-in volume."""

import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import oracle
from pyslam_b200 import sharding
from pyslam_b200 import synthetic as S
from tests import _edge_scenes as E
from tests import _halo_oracle as H


def _twin_map(name, frames):
    cfg = S.CONFIGS[name]
    tw = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    for i in range(frames):
        d, c, T = S.render_frame(cfg, i)
        tw.integrate(d, c, cfg.K, T)
    return (cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc), tw


def _scenes():
    for name, frames in (("T0", 2), ("C1", 1), ("C2", 2)):
        args, tw = _twin_map(name, frames)
        yield name, args, tw.dump_blocks(), tw.extract_mesh()
    cfg = S.CONFIGS["T0"]
    args = (cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    for seed in (3, 7):
        keys, vox = E.random_blocks(seed=seed)
        tw = oracle.TsdfOracle(*args)
        for k, v in zip(keys, vox):
            tw.set_block(k, v)
        yield f"random{seed}", args, tw.dump_blocks(), tw.extract_mesh()


SCENES = list(_scenes())


def test_halo_shapes():
    sizes = {m: len(H.halo_shape(m)) for m in range(1, 128)}
    # bit o-1 = offset o (x = 1, y = 2, z = 4): faces o = 1, 2, 4; lines o = 3, 5, 6; the corner o = 7
    assert sizes[1] == sizes[2] == sizes[8] == 64 and sizes[4] == sizes[16] == sizes[32] == 8 and sizes[64] == 1
    assert sizes[127] == max(sizes.values()) == 169 == 512 - 7 ** 3
    # the shapes of a 2-axis / 3-axis offset lie inside the 1-axis faces
    assert np.array_equal(H.halo_shape(1 | 2 | 8), H.halo_shape(127))


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("scene", range(len(SCENES)), ids=[s[0] for s in SCENES])
def test_rank_meshes_weld_to_the_whole_map_mesh(scene, world):
    name, args, dump, full = SCENES[scene]
    shards = H.shard_dumps(dump["keys"], dump["vox"], world)
    pieces, n_tri = [], 0
    for r in range(world):
        recs = H.numpy_halo_records(*shards[r], world)
        assert len(recs[r][0]) == 0                               # nothing for itself
        per_block = {}
        for h, _ in recs:
            assert len(h) == len(np.unique(h[:, :3], axis=0))     # one record per (block, destination)
            for row in h:
                per_block[tuple(row[:3])] = per_block.get(tuple(row[:3]), 0) + len(H.halo_shape(int(row[3])))
                assert len(H.halo_shape(int(row[3]))) <= 169
        assert max(per_block.values(), default=0) <= 217
        hdr, pay = H.received(shards, world, r)
        tw = H.twin_piece(args, *shards[r], hdr, pay)
        m = tw.extract_mesh()
        assert H.triangle_roots_ok(m["edges"], m["triangles"], shards[r][0]), (name, r)
        n_tri += len(m["triangles"])
        pieces.append(m)
    assert n_tri == len(full["triangles"])                        # no triangle on two ranks, none lost
    got = oracle.canonical_mesh(**H.numpy_weld(pieces))
    want = oracle.canonical_mesh(full["vertices"], full["colors"], full["edges"], full["triangles"])
    for k in want:
        assert np.array_equal(got[k], want[k]), (name, world, k)


@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("scene", range(len(SCENES)), ids=[s[0] for s in SCENES])
def test_rank_point_clouds_partition_the_whole_map_cloud(scene, world):
    name, args, dump, _ = SCENES[scene]
    full = oracle.numpy_point_cloud(dump, args[0], 16)
    shards = H.shard_dumps(dump["keys"], dump["vox"], world)
    parts = []
    for r in range(world):
        hdr, pay = H.received(shards, world, r)
        hk, hv = H.halo_blocks(hdr, pay)
        keys = np.concatenate([shards[r][0], hk])
        pc = oracle.numpy_point_cloud(dict(keys=keys, vox=np.concatenate([shards[r][1], hv])), args[0], 16)
        root = sharding.owner_of(pc["edges"][:, :3] >> 3, world) == r   # roots limited to the own blocks
        parts.append({k: v[root] for k, v in pc.items()})
    got = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    assert len(np.unique(got["edges"], axis=0)) == len(got["edges"]) == len(full["edges"])

    def by_edge(d):
        o = np.lexsort(d["edges"].T[::-1])
        return {k: v[o] for k, v in d.items()}
    a, b = by_edge(got), by_edge(full)
    for k in a:
        assert np.array_equal(a[k], b[k]), (name, world, k)


# ---- gloo: the collective wrapper's host logic ------------------------------------------------------------------

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


class _StandInShard:
    """Stand-in for one shard of B200TsdfVolume on the CPU: numpy records of its blocks, twin mesh pieces."""
    device = 0

    def __init__(self, args, keys, vox, world):
        self.args, self.keys, self.vox, self.world = args, keys, vox, world

    def export_halo_torch(self, world):
        recs = H.numpy_halo_records(self.keys, self.vox, world)
        return (torch.from_numpy(np.concatenate([h for h, _ in recs])),
                torch.from_numpy(np.concatenate([x for _, x in recs])),
                [len(h) for h, _ in recs], [len(x) for _, x in recs])

    def extract_mesh_with_halo(self, headers, payload):
        from pyslam_b200.volume import TriangleMesh
        m = H.twin_piece(self.args, self.keys, self.vox, headers.numpy(), payload.numpy()).extract_mesh()
        return TriangleMesh(m["vertices"], m["triangles"], m["colors"], m["edges"])

    def extract_point_cloud_with_halo(self, headers, payload):
        from pyslam_b200.volume import PointCloud
        hk, hv = H.halo_blocks(headers.numpy(), payload.numpy())
        pc = oracle.numpy_point_cloud(dict(keys=np.concatenate([self.keys, hk]), vox=np.concatenate([self.vox, hv])),
                                      self.args[0], 16)
        root = np.all((pc["edges"][:, None, :3] >> 3) == self.keys[None], axis=2).any(axis=1)
        return PointCloud(pc["points"][root], pc["colors"][root], pc["edges"][root])


def _gloo_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        def weld(pieces, device=0):   # the GPU weld is checked on the GPU; here its numpy restatement
            from pyslam_b200.volume import TriangleMesh
            w = H.numpy_weld([dict(vertices=p.vertices, colors=p.vertex_colors, edges=p.edge_ids,
                                   triangles=p.triangles) for p in pieces])
            return TriangleMesh(w["vertices"], w["triangles"], w["colors"], w["edges"])
        sharding.weld = weld
        cfg = S.CONFIGS["T0"]
        args = (cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
        keys, vox = E.random_blocks(seed=3)
        mine = sharding.owner_of(keys, world) == rank
        vol = _StandInShard(args, keys[mine], vox[mine], world)
        mesh = sharding.extract_mesh_sharded(vol, dst=0)
        pc = sharding.extract_point_cloud_sharded(vol, dst=0)
        own = sharding.extract_mesh_sharded(vol, gather=False)
        sent = vol.last_halo_bytes
        if rank == 0:
            tw = oracle.TsdfOracle(*args)
            for k, v in zip(keys, vox):
                tw.set_block(k, v)
            full = tw.extract_mesh()
            got = oracle.canonical_mesh(mesh.vertices, mesh.vertex_colors, mesh.edge_ids, mesh.triangles)
            want = oracle.canonical_mesh(full["vertices"], full["colors"], full["edges"], full["triangles"])
            ok = all(np.array_equal(got[k], want[k]) for k in want)
            fpc = oracle.numpy_point_cloud(dict(keys=keys, vox=vox), cfg.voxel_size, 16)
            o1, o2 = np.lexsort(pc.edge_ids.T[::-1]), np.lexsort(fpc["edges"].T[::-1])
            ok = ok and np.array_equal(pc.edge_ids[o1], fpc["edges"][o2]) and np.array_equal(pc.points[o1],
                                                                                              fpc["points"][o2])
            recs = [H.numpy_halo_records(keys[sharding.owner_of(keys, world) == s],
                                         vox[sharding.owner_of(keys, world) == s], world) for s in range(world)]
            ok = ok and sent == [sum(len(h) * 16 + len(x) * 20 for h, x in r) for r in recs] and min(sent) > 0
            q.put(("ok" if ok else "mismatch", len(own.triangles)))
        else:
            q.put(("ok" if mesh is None and pc is None else "mismatch", len(own.triangles)))
    finally:
        dist.destroy_process_group()


def test_sharded_extraction_wrappers_over_gloo():
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert [r[0] for r in res] == ["ok", "ok"]
    assert all(r[1] > 0 for r in res)
