"""Per-rank cost of hash-sharded grids, N = 2, 4, 8 ranks emulated by N shard grids in one process on one GPU (the
ranks share nothing on the data path, so each rank's work can be timed alone), against the unsharded grid (N = 1):
    grid      the bench's grid leg: C2, 300 device-resident frames through b2v_grid_integrate_rgbd, fixed 2^17 blocks
    semantic  the bench's semantic leg: C3, 16 frames with class and instance images through the Bayesian grid at
              0.015 m (growable 2^10 -> 2^16), each frame associated (votes + resolve, carving on) and then integrated
              with its object image
Per N: blocks per rank, integrate ms per frame (max and mean over ranks, each rank timed alone), association ms per
frame (votes: max over ranks; resolve of all ranks' triples: max over ranks; the triples exchanged per frame), storage
each rank holds (blocks with storage x bytes per block), and whether the shards equal the unsharded grid (keys, counts
and, for the semantic grid, the whole dump).  Prints one JSON line with the card's name and power limit.
python tools/sharded_grid_cost.py"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from pyslam_b200 import (CameraFrustrum, VoxelBlockGrid, VoxelBlockSemanticProbabilisticGrid, remap_instance_ids,
                         sharding)
from pyslam_b200.volume import _as_K4
from pyslam_b200 import synthetic as S
from tests._util import sort_dump

GRID_BLOCK_BYTES = 7 * 512 * 4          # count, position sum, colour sum planes
BAYES_BLOCK_BYTES = 512 * (4 + 24 + 12 + 4 + 4 + 4 + 4 + 4 + 3 * 8 * 4)   # DESIGN.md §4: 79 872 B


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def grid_leg(world):
    cfg, depth, color, Tcw = bench.load_frames("C2", 300, 0, 1)
    d_dev, c_dev = torch.from_numpy(depth).cuda(), torch.from_numpy(color).cuda()
    K4 = np.array(cfg.K, np.float64)
    Twc = [np.ascontiguousarray(S.inv_T(Tcw[i])).reshape(16) for i in range(len(depth))]

    def run(g):
        for i in range(len(depth)):
            rc = g._L.b2v_grid_integrate_rgbd(g._h, d_dev[i].data_ptr(), c_dev[i].data_ptr(), depth.shape[1],
                                              depth.shape[2], K4.ctypes.data, Twc[i].ctypes.data,
                                              float(cfg.depth_trunc), 0.0, 0)
            assert rc == 0
        g._check(g._L.b2v_grid_synchronize(g._h), "sync")

    grids = [VoxelBlockGrid(cfg.voxel_size, 8, capacity_blocks=1 << 17, shard_rank=r, shard_count=world)
             for r in range(world)]
    run(grids[0])   # module load and warm-up
    grids[0].clear()
    ms = []
    for g in grids:
        ms.append(1e3 * wall(lambda: run(g)) / len(depth))
    blocks = [g.num_blocks() for g in grids]
    dumps = [g.dump_blocks() for g in grids]
    for g in grids:
        g.close()
    return {"blocks_per_rank": blocks, "integrate_ms_per_frame_max": round(max(ms), 4),
            "integrate_ms_per_frame_mean": round(float(np.mean(ms)), 4),
            "storage_gb_per_rank_used_blocks": round(max(blocks) * GRID_BLOCK_BYTES / 1e9, 3)}, dumps


def semantic_leg(world):
    cfg, depth, color, Tcw = bench.load_frames("C3", 16, 0, 1)
    step = max(cfg.n_frames // len(depth), 1)
    cls = [S.render_class_ids(cfg, i * step).astype(np.int32) for i in range(len(depth))]
    inst = [np.where(c % 3 == 0, -1, c * 7 + np.arange(c.shape[1])[None, :] // 400).astype(np.int32) for c in cls]
    K4 = _as_K4(cfg.K)
    grids = [VoxelBlockSemanticProbabilisticGrid(0.015, 8, capacity_blocks=1 << 10, max_capacity_blocks=1 << 16,
                                                 shard_rank=r, shard_count=world) for r in range(world)]
    t_int, t_votes, t_res, n_triples = np.zeros(world), np.zeros(world), np.zeros(world), []
    for i in range(len(depth)):
        fr = CameraFrustrum(*K4, depth.shape[2], depth.shape[1], Tcw[i], depth_max=cfg.depth_trunc, depth_min=1e-2)
        votes = [None] * world
        for r, g in enumerate(grids):
            t_votes[r] += wall(lambda: votes.__setitem__(r, sharding.association_votes(
                g, fr, cls[i], inst[i], depth[i], 0.08, True)))
        n_triples.append(sum(len(v) for v in votes))
        maps = [None] * world
        for r, g in enumerate(grids):
            t_res[r] += wall(lambda: maps.__setitem__(r, sharding.resolve_association(g, votes, cls[i], inst[i])))
        assert all(m == maps[0] for m in maps)
        obj = remap_instance_ids(inst[i], maps[0])
        for r, g in enumerate(grids):
            t_int[r] += wall(lambda: g.integrate_rgbd(depth[i], color[i], cfg.K, S.inv_T(Tcw[i]), cls[i], obj,
                                                      max_depth=cfg.depth_trunc))
    n = len(depth)
    blocks = [g.num_blocks() for g in grids]
    storage = [g.capacity()[0] for g in grids]
    dumps = [g.dump_blocks(8) for g in grids]
    for g in grids:
        g.close()
    return {"blocks_per_rank": blocks, "integrate_ms_per_frame_max": round(1e3 * t_int.max() / n, 3),
            "integrate_ms_per_frame_mean": round(1e3 * t_int.mean() / n, 3),
            "votes_ms_per_frame_max": round(1e3 * t_votes.max() / n, 3),
            "resolve_ms_per_frame_max": round(1e3 * t_res.max() / n, 3),
            "triples_per_frame_all_ranks": int(np.mean(n_triples)),
            "storage_blocks_per_rank_max": max(storage),
            "storage_gb_per_rank_max": round(max(storage) * BAYES_BLOCK_BYTES / 1e9, 3)}, dumps


def main():
    out = {"gpu": card()}
    for name, leg in (("grid_C2_300_frames", grid_leg), ("semantic_C3_16_frames", semantic_leg)):
        ref = None
        for world in (1, 2, 4, 8):
            r, dumps = leg(world)
            merged = sharding.merge_dumps(dumps)
            if ref is None:
                ref = sort_dump(dumps[0])
            else:
                keys = ("keys", "count") if name.startswith("grid") else tuple(ref)
                r["equal_to_unsharded"] = bool(all(np.array_equal(merged[k], ref[k], equal_nan=True) for k in keys))
            out.setdefault(name, {})[f"N={world}"] = r
    print(json.dumps(out))


if __name__ == "__main__":
    main()
