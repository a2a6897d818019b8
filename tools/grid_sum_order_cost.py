"""Cost of the point-average grid's input-order sums (VoxelBlockGrid(input_order_sums=True)) against the default
float-atomic sums, through integrate_rgbd on device frames, on C2, C3 (5 mm voxels, the bench's grid leg) and C5
(10 cm voxels: the longest runs).  Per configuration:
    timing     both modes fed the same frames, alternated frame by frame, each into its own grid, after a warm pass
               (--steps frames per mode, cycling over --frames rendered frames); median and p90 ms per frame, host
               clock around each call, which ends in a device synchronise
    split      a separate run under torch.profiler (CUDA kernel activity): device ms per frame of the RGBD front-end
               and insert, the keys, the sort (CUB radix sort kernels), the runs, and the atomic accumulate
    runs       the longest and the 99th-percentile run (points of one voxel in one call: the work of one thread of
               grid_runs_kernel), from the front-end points of the rendered frames
    staging    bytes per pixel the input-order mode keeps: point record 12 + colour 12 + mask 1 + two key and two
               order buffers of 4 each, times the pixels of a frame (the radix sort's temporary storage comes on top)
Prints one JSON line with the card's name, power limit and clocks, read in the same run.
python tools/grid_sum_order_cost.py [--frames N] [--steps K]"""
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
from pyslam_b200 import VoxelBlockGrid
from pyslam_b200 import synthetic as S

CONFIGS = ("C2", "C3", "C5")
RECORD_BYTES = 12 + 12 + 1 + 2 * 4 + 2 * 4


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def run_lengths(cfg, depth, color, Tcw):
    """(longest, p99) of the points per voxel and frame."""
    inv = np.float32(1.0) / np.float32(cfg.voxel_size)
    runs = []
    for i in range(len(depth)):
        p = S.inv_T(Tcw[i])
        fx, fy, cx, cy = cfg.K
        d = depth[i]
        ok = (d > 0) & (d < cfg.depth_trunc)
        rows, cols = np.nonzero(ok)
        z = d[ok].astype(np.float64)
        x, y = ((cols - cx) * z) * (1.0 / fx), ((rows - cy) * z) * (1.0 / fy)
        w = np.stack([((x * p[a, 0] + y * p[a, 1]) + z * p[a, 2]) + p[a, 3] for a in range(3)], 1).astype(np.float32)
        k = np.floor(w * inv).astype(np.int64) + (1 << 20)
        key = (k[:, 0] << 42) | (k[:, 1] << 21) | k[:, 2]
        runs.append(np.unique(key, return_counts=True)[1])
    r = np.concatenate(runs)
    return int(r.max()), float(np.percentile(r, 99))


def rgbd(g, d, c, cfg, Tcw):
    """integrate_rgbd of device images through the C ABI (read in place), ending in a device synchronise."""
    K4 = np.array(cfg.K, np.float64)
    T = np.ascontiguousarray(S.inv_T(Tcw)).reshape(16)
    rc = g._L.b2v_grid_integrate_rgbd(g._h, d.data_ptr(), c.data_ptr(), d.shape[0], d.shape[1], K4.ctypes.data,
                                      T.ctypes.data, float(cfg.depth_trunc), 0.0, 0)
    assert rc == 0, rc
    g._check(g._L.b2v_grid_synchronize(g._h), "b2v_grid_synchronize")


def make_grids(cfg):
    return {m: VoxelBlockGrid(cfg.voxel_size, 8, capacity_blocks=1 << 18, input_order_sums=m == "input_order")
            for m in ("atomic", "input_order")}


def timing(cfg, d_dev, c_dev, Tcw, steps):
    grids = make_grids(cfg)
    n = len(d_dev)

    def call(g, i):
        rgbd(g, d_dev[i % n], c_dev[i % n], cfg, Tcw[i % n])

    for g in grids.values():   # module loads, staging buffers, the map's blocks
        for i in range(n):
            call(g, i)
    ms = {m: [] for m in grids}
    for i in range(steps):
        for m, g in grids.items():
            t0 = time.perf_counter()
            call(g, i)
            ms[m].append(1e3 * (time.perf_counter() - t0))
    out = {m: dict(median_ms=round(float(np.median(v)), 4), p90_ms=round(float(np.percentile(v, 90)), 4),
                   frames=len(v)) for m, v in ms.items()}
    for g in grids.values():
        g.close()
    return out


def split(cfg, d_dev, c_dev, Tcw, frames=20):
    """Device ms per frame of each kernel group, from torch.profiler's CUDA kernel activity."""
    from torch.profiler import ProfilerActivity, profile
    groups = {"front_end_and_insert": ("grid_rgbd_points_kernel", "point_insert_kernel", "grid_rgbd_insert_kernel"),
              "keys": ("voxel_keys_kernel",), "sort": ("DeviceRadixSort",), "runs": ("grid_runs_kernel",),
              "atomic_accumulate": ("grid_rgbd_accumulate_kernel",)}
    out = {}
    for m, g in make_grids(cfg).items():
        for i in range(len(d_dev)):
            rgbd(g, d_dev[i], c_dev[i], cfg, Tcw[i])
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(frames):
                j = i % len(d_dev)
                rgbd(g, d_dev[j], c_dev[j], cfg, Tcw[j])
            torch.cuda.synchronize()
        tot = {k: 0.0 for k in groups}
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            for k, names in groups.items():
                if any(s in e.key for s in names):
                    tot[k] += us
        out[m] = {k: round(v / 1e3 / frames, 4) for k, v in tot.items() if v}
        g.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--steps", type=int, default=300)
    a = ap.parse_args()
    out = {"gpu": card()}
    for name in CONFIGS:
        cfg, depth, color, Tcw = bench.load_frames(name, a.frames, 0, 1)
        d_dev = [torch.from_numpy(x).cuda() for x in depth]
        c_dev = [torch.from_numpy(x).cuda() for x in color]
        torch.cuda.synchronize()
        longest, p99 = run_lengths(cfg, depth, color, Tcw)
        out[name] = dict(voxel_size=cfg.voxel_size, pixels=int(cfg.width * cfg.height),
                         staging_bytes=RECORD_BYTES * cfg.width * cfg.height, longest_run=longest,
                         p99_run=round(p99, 1), timing=timing(cfg, d_dev, c_dev, Tcw, a.steps),
                         split_ms_per_frame=split(cfg, d_dev, c_dev, Tcw))
    out["gpu_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
