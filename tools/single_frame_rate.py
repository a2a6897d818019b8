"""Single-frame integration rate: the 300 C2 frames through `vol.integrate(...)`, one call per frame (the frame-by-frame
kernels, allocate / update overlap on), from device memory and from pinned host memory.  Each timed pass starts from
an empty volume and ends with a full synchronise.  python tools/single_frame_rate.py [--reps N]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import argparse, json, time, torch, bench
from pyslam_b200 import B200TsdfVolume

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
args = ap.parse_args()
cfg, depth, color, Tcw = bench.load_frames("C2", 300, 0, 1)
vol = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 19)
pinned = [torch.from_numpy(a).pin_memory() for a in (depth, color)]  # kept alive: the numpy views below share them
sources = {"device": (torch.from_numpy(depth).cuda(), torch.from_numpy(color).cuda()),
           "pinned_host": tuple(t.numpy() for t in pinned)}


def one_pass(d, c):
    """(frames/s, host enqueue time per frame in us)"""
    vol.reset()
    t0 = time.perf_counter()
    for i in range(len(Tcw)):
        vol.integrate(d[i], c[i], cfg.K, Tcw[i])
    t1 = time.perf_counter()
    vol.synchronize()
    return len(Tcw) / (time.perf_counter() - t0), 1e6 * (t1 - t0) / len(Tcw)


for name, (d, c) in sources.items():
    one_pass(d, c)  # warm-up
    runs = [one_pass(d, c) for _ in range(args.reps)]
    print(json.dumps({"source": name, "gpu": torch.cuda.get_device_name(0),
                      "frames_per_s": [round(r, 1) for r, _ in runs],
                      "enqueue_us_per_frame": [round(e, 1) for _, e in runs]}))
