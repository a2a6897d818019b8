"""Cost of the grids' block size B in (1, 2, 8, 16), on the bench's frames:
    point     VoxelBlockGrid.integrate_rgbd of C2 and C3 frames (device-resident), then get_voxels(1)
    bayes     VoxelBlockSemanticProbabilisticGrid.integrate_rgbd of C2 and C3 frames with class images at 0.015 m,
              then get_voxels(1)
Per grid and B: integrate_rgbd ms per frame (a warm pass into a cleared grid), get_voxels ms, blocks held and the
device memory the grid holds (drop of free memory from before create to the end).  Every B holds the same voxels, so
get_voxels returns the same count at every B (reported).  Prints one JSON line with the card's name and power limit.
python tools/grid_block_size_cost.py [--frames N]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from pyslam_b200 import VoxelBlockGrid, VoxelBlockSemanticProbabilisticGrid
from pyslam_b200 import synthetic as S

SIZES = (1, 2, 8, 16)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def measure(make, frames, labels, cfg):
    depth, color, Tcw = frames
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    g = make()

    def run():
        for i in range(len(depth)):
            kw = dict(class_image=labels[i]) if labels is not None else {}
            g.integrate_rgbd(depth[i], color[i], cfg.K, S.inv_T(Tcw[i]), max_depth=cfg.depth_trunc, **kw)
        torch.cuda.synchronize()

    run()            # module loads and storage
    g.clear()
    t0 = time.perf_counter()
    run()
    ms = 1e3 * (time.perf_counter() - t0) / len(depth)
    g.get_voxels(1)
    t0 = time.perf_counter()
    v = g.get_voxels(1)
    gv = 1e3 * (time.perf_counter() - t0)
    r = dict(integrate_rgbd_ms_per_frame=round(ms, 3), get_voxels_ms=round(gv, 3), voxels=len(v.points),
             blocks=g.num_blocks(), held_gb=round((free0 - torch.cuda.mem_get_info()[0]) / 1e9, 3))
    g.close()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=32)
    a = ap.parse_args()
    out = {"gpu": card()}
    for conf in ("C2", "C3"):
        cfg, depth, color, Tcw = bench.load_frames(conf, a.frames, 0, 1)
        labels = [S.render_class_ids(cfg, i * max(cfg.n_frames // len(depth), 1)) for i in range(len(depth))]
        for B in SIZES:
            # the same voxel budget at every B: 2^17 blocks of 8^3 voxels (point), 2^16 (Bayesian)
            out[f"point_{conf}_B{B}"] = measure(
                lambda: VoxelBlockGrid(cfg.voxel_size, B, capacity_blocks=-(-(1 << 17) * 512 // B ** 3)),
                (depth, color, Tcw), None, cfg)
            out[f"bayes_{conf}_B{B}"] = measure(
                lambda: VoxelBlockSemanticProbabilisticGrid(0.015, B, capacity_blocks=-(-(1 << 16) * 512 // B ** 3)),
                (depth, color, Tcw), labels, cfg)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
