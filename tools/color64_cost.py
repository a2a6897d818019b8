"""Cost of the float64-colour volume (B200TsdfVolume(color_float64=True)) against the default float32-colour volume.

C2, 300 frames, fused in groups of 32, both modes alternated in one run.  Per mode and repetition: frames/s of the
whole integrate_batch call (host clock around work that ends in a synchronise) and the update kernel's device time per
32-frame group (CUDA events, b2v_profile_*).  Prints one JSON line with the card name and power limit.

    python tools/color64_cost.py [--reps 5] [--frames 300]
"""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pyslam_b200 import B200TsdfVolume  # noqa: E402
from pyslam_b200 import synthetic as S  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _run(cfg, d, c, T, f64):
    v = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 19, color_float64=f64)
    v.set_group_size(32)
    v.integrate_batch(d[:32], c[:32], cfg.K, T[:32])   # warm-up: module load, staging buffers
    v.synchronize()
    v.reset()
    v.profile_enable(True)
    t0 = time.perf_counter()
    v.integrate_batch(d, c, cfg.K, T)
    v.synchronize()
    dt = time.perf_counter() - t0
    alloc_ms, int_ms, frames, launches = v.profile_read()
    v.close()
    return len(d) / dt, 1000.0 * int_ms / max(1, -(-len(d) // 32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=300)
    a = ap.parse_args()
    cfg = S.CONFIGS["C2"]
    frames = [S.render_frame(cfg, i % cfg.n_frames) for i in range(a.frames)]
    d, c, T = (np.ascontiguousarray(np.stack([f[k] for f in frames])) for k in range(3))
    res = {"f32": [], "f64": []}
    for _ in range(a.reps):
        for name, f64 in (("f32", False), ("f64", True)):
            res[name].append(_run(cfg, d, c, T, f64))
    out = {"card": _card(), "config": "C2", "frames": a.frames, "group": 32}
    for name, rows in res.items():
        fps = [r[0] for r in rows]
        us = [r[1] for r in rows]
        out[name] = dict(frames_per_s=[round(x, 1) for x in fps], update_us_per_group=[round(x, 1) for x in us],
                         median_frames_per_s=round(float(np.median(fps)), 1),
                         median_update_us_per_group=round(float(np.median(us)), 1))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
