"""Cost of the sharded extraction (face-halo exchange) against gather-to-one, C2's 300 frames (device-resident).

One GPU: N in {2, 4, 8} shard volumes held in one process emulate N ranks.  Per rank: halo export, import + mesh
extraction (b2v_extract_mesh_with_halo, which imports the shard and the records into its scratch first) and point
extraction times, halo bytes sent; then the weld time of the N pieces.  Against it: the bytes gather-to-one moves for
the same map ((N-1)/N of the blocks at 10 240 B each, `extract_mesh_distributed`), the extraction-scratch memory
(shard + received halo blocks) against the gather scratch (the whole map), and the single-volume extract_mesh time.
Under torchrun on N GPUs (`torchrun --nproc-per-node N tools/sharded_extract_cost.py --dist`): wall time of
extract_mesh_sharded against extract_mesh_distributed.  Prints one JSON line (rank 0).
python tools/sharded_extract_cost.py [--frames 300]"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from pyslam_b200 import B200TsdfVolume, sharding

BLOCK_BYTES = 5 * 512 * 4


def _sync_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, round((time.perf_counter() - t0) * 1e3, 3)


def one_gpu(frames):
    cfg, depth, color, Tcw = bench.load_frames("C2", frames, 0, 1)
    d, c = torch.from_numpy(depth).cuda(), torch.from_numpy(color).cuda()
    out = {"gpu": torch.cuda.get_device_name(0), "frames": frames, "config": "C2"}

    def vol(**kw):
        v = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 19, **kw)
        v.integrate_batch(d, c, cfg.K, Tcw)
        v.synchronize()
        return v

    single = vol()
    nb = single.num_blocks()
    single.extract_mesh()
    m, t = _sync_ms(single.extract_mesh)
    out["single"] = {"blocks": nb, "extract_mesh_ms": t, "triangles": len(m.triangles)}
    for world in (2, 4, 8):
        shards = [vol(shard_rank=r, shard_count=world) for r in range(world)]
        for _ in range(2):   # the second round is timed (scratch volumes exist, tables uploaded)
            r = {"ranks": []}
            recs = []
            for s in shards:
                rec, t_exp = _sync_ms(lambda: sharding.halo_records(s, world))
                recs.append(rec)
                sent = sum(h.numel() * 4 + x.numel() * 4 for i, (h, x) in enumerate(rec))
                r["ranks"].append({"blocks": s.num_blocks(), "export_ms": t_exp, "halo_bytes_sent": sent})
            pieces = []
            for i, s in enumerate(shards):
                inbox = [recs[j][i] for j in range(world)]
                piece, t_mesh = _sync_ms(lambda: sharding.mesh_piece(s, inbox))
                _, t_pts = _sync_ms(lambda: sharding.point_piece(s, inbox))
                n_halo = sum(h.shape[0] for h, _ in inbox)
                r["ranks"][i].update(import_and_mesh_ms=t_mesh, import_and_points_ms=t_pts, halo_blocks=n_halo,
                                     scratch_gb=round((s.num_blocks() + n_halo) * BLOCK_BYTES / 1e9, 4))
                pieces.append(piece)
            welded, t_weld = _sync_ms(lambda: sharding.weld(pieces))
        r["weld_ms"] = t_weld
        r["triangles"] = len(welded.triangles)
        r["halo_bytes_total"] = sum(x["halo_bytes_sent"] for x in r["ranks"])
        r["gather_bytes_total"] = sum(x["blocks"] for x in r["ranks"][1:]) * BLOCK_BYTES   # dst = rank 0
        r["halo_over_gather"] = round(r["halo_bytes_total"] / max(r["gather_bytes_total"], 1), 4)
        r["gather_scratch_gb"] = round(nb * BLOCK_BYTES / 1e9, 4)
        r["max_rank_mesh_ms"] = max(x["import_and_mesh_ms"] for x in r["ranks"])
        out[f"N{world}"] = r
        for s in shards:
            s.close()
    print(json.dumps(out))


def distributed(frames):
    import torch.distributed as dist
    dist.init_process_group("nccl")
    rank, world = dist.get_rank(), dist.get_world_size()
    torch.cuda.set_device(rank)
    cfg, depth, color, Tcw = bench.load_frames("C2", frames, 0, 1)
    d, c = torch.from_numpy(depth).cuda(), torch.from_numpy(color).cuda()
    v = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 19, device=rank,
                       shard_rank=rank, shard_count=world)
    v.integrate_batch(d, c, cfg.K, Tcw)
    v.synchronize()
    res = {}
    for name, fn in (("sharded", lambda: sharding.extract_mesh_sharded(v)),
                     ("gather_to_one", lambda: sharding.extract_mesh_distributed(v))):
        ts = []
        for _ in range(3):
            dist.barrier()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            dist.barrier()
            ts.append(time.perf_counter() - t0)
        res[name + "_s"] = round(min(ts[1:]), 4)
    if rank == 0:
        print(json.dumps({"gpu": torch.cuda.get_device_name(0), "world": world, "frames": frames, **res}))
    dist.destroy_process_group()


if __name__ == "__main__":
    n = int(sys.argv[sys.argv.index("--frames") + 1]) if "--frames" in sys.argv else 300
    distributed(n) if "--dist" in sys.argv else one_gpu(n)
