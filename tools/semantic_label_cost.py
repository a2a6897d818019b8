"""Cost of the Bayesian grid's overflow label store (max_label_overflow_pairs), on C3 frames through integrate_rgbd
with class images at 0.015 m (the bench's semantic leg):
    bench    the bench's stream: class images, no object images (object id 0), so a voxel holds one pair per class
    churn    the same frames with object images whose ids change every frame (class * 1000 + frame + a 0..2 jitter per
             pixel), the pattern of an instance association that cannot match
Per stream and ceiling (0 = no store, and 2^24 pairs): integrate_rgbd ms per frame (a warm pass into a cleared grid),
the device memory the grid holds (drop of free memory from before create to the end), the histogram of pairs per voxel,
chunks in use and mapped, and label overflows.  Prints one JSON line with the card's name, power limit and clock.
python tools/semantic_label_cost.py [--frames N]"""
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
from pyslam_b200 import VoxelBlockSemanticProbabilisticGrid
from pyslam_b200 import synthetic as S

CEILINGS = (0, 1 << 24)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def measure(ceiling, frames, labels, objects, cfg):
    depth, color, Tcw = frames
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    g = VoxelBlockSemanticProbabilisticGrid(0.015, 8, capacity_blocks=1 << 16, max_label_overflow_pairs=ceiling)

    def run():
        for i in range(len(depth)):
            g.integrate_rgbd(depth[i], color[i], cfg.K, S.inv_T(Tcw[i]), class_image=labels[i],
                             object_image=None if objects is None else objects[i], max_depth=cfg.depth_trunc)
        torch.cuda.synchronize()

    run()            # module loads and storage
    g.clear()
    t0 = time.perf_counter()
    run()
    ms = 1e3 * (time.perf_counter() - t0) / len(depth)
    held = (free0 - torch.cuda.mem_get_info()[0]) / 1e9
    st = g.export_blocks()
    pairs = st["counter"][st["count"] > 0]
    hist = np.bincount(pairs, minlength=9)
    r = dict(integrate_rgbd_ms_per_frame=round(ms, 3), held_gb=round(held, 3), voxels=int(len(pairs)),
             pairs_histogram={str(k): int(v) for k, v in enumerate(hist) if v},
             label_storage=g.label_storage(), label_overflows=g.label_overflows())
    g.close()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=32)
    a = ap.parse_args()
    out = {"gpu": card()}
    cfg, depth, color, Tcw = bench.load_frames("C3", a.frames, 0, 1)
    labels = [S.render_class_ids(cfg, i * max(cfg.n_frames // len(depth), 1)) for i in range(len(depth))]
    rng = np.random.default_rng(0)
    churn = [(lab * 1000 + i + rng.integers(0, 3, lab.shape)).astype(np.int32) for i, lab in enumerate(labels)]
    for name, objects in (("bench", None), ("churn", churn)):
        for ceiling in CEILINGS:
            out[f"{name}_ceiling_{ceiling}"] = measure(ceiling, (depth, color, Tcw), labels, objects, cfg)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
