"""Per-keyframe cost of the grid plugins with the frame preparation on the host (the base class: cv2.remap, cvtColor,
depth widening, label remap in numpy) against on the device (set_frame, kVolumetricIntegrationB200GpuRectify).

Seeded C2 (640x480) and C3 (1200x680) frames, raw BGR + uint16 depth in C++-core mode, TUM1-like distortion maps,
through the semantic plugin (voting grid, class and instance images, association with carving, shadow filter) and the
voxel-grid plugin (carving, shadow filter).  Each path runs in its own plugin instance; the two are alternated frame by
frame in one run.  Wall ms per frame is a host clock around one plugin step followed by a device synchronise; the
first frames are warm-up.  H2D bytes per frame are the image bytes each path's calls upload, computed from the image
sizes (the host path also downloads the filtered depth once).  Both paths' grids are compared at the end.  Prints one
JSON line with the card's name, power limit and SM clock read in the same run.
python tools/grid_frame_cost.py [--frames N] [--warmup W]"""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from pyslam_b200 import integrator_semantic as IS
from pyslam_b200 import synthetic as S
from tests import plugin_standins as P
from tests._util import sort_dump
from tests.test_gpu_grid_frames import RectifyingBase, raw_labels, tum_maps


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def h2d_bytes_per_pixel(kind, device):
    """Uploads of one frame: device path = set_frame (uint16 depth 2, BGR 3, class 4, instance 4); host path =
    filter_shadow_points (depth 4), association (class, instance, depth 12), integrate_rgbd (depth, RGB, class, object
    15) for the semantic plugin, carve (depth 4) + integrate_rgbd (depth 4, RGB 3) for the voxel-grid plugin."""
    if kind == "semantic":
        return 13 if device else 31
    return 5 if device else 11


def make_plugin(kind, cfg, maps, device):
    base = type("Base", (RectifyingBase,), {"use_cpp": True})
    api = SimpleNamespace(**vars(P.API), USE_CPP=True)
    make = IS.make_semantic_integrator_class if kind == "semantic" else IS.make_voxel_grid_integrator_class
    cam = SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None,
                          depth_factor=1.0 / 5000)
    return make(base, api)(cam, P.DatasetEnvironmentType.INDOOR, None, "B200", calib_maps=maps,
                           kVolumetricIntegrationB200GpuRectify=device, kVolumetricIntegrationVoxelGridUseCarving=True,
                           kVolumetricIntegrationOutputTimeInterval=1e9, kVolumetricIntegrationVoxelLength=0.015,
                           kVolumetricIntegrationB200CapacityBlocks=1 << 17)


def run(kind, name, n, warmup):
    cfg = S.CONFIGS[name]
    maps = tum_maps(cfg)
    frames = []
    for i in range(n):
        d, c, Tcw = S.render_frame(cfg, 3 * i)
        cls, inst = raw_labels(cfg, 3 * i, d)
        frames.append(P.VolumetricIntegrationKeyframeData(
            id=i, pose=Tcw, img=np.ascontiguousarray(c[..., ::-1]), depth=np.round(d * 5000).astype(np.uint16),
            semantic_img=cls, semantic_instances_img=inst))
    plugins = {"host": make_plugin(kind, cfg, maps, False), "device": make_plugin(kind, cfg, maps, True)}
    assert plugins["device"]._gpu_rectify and not plugins["host"]._gpu_rectify
    ms = {"host": [], "device": []}
    for i, kd in enumerate(frames):
        for path in (("host", "device") if i % 2 == 0 else ("device", "host")):
            integ = plugins[path]
            integ.add_keyframe_data(kd)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            integ.step()
            torch.cuda.synchronize()
            if i >= warmup:
                ms[path].append((time.perf_counter() - t0) * 1e3)
    dumps = {p: sort_dump(v.volume.dump_blocks(8) if kind == "semantic" else v.volume.dump_blocks())
             for p, v in plugins.items()}
    same_keys = bool(np.array_equal(dumps["host"]["keys"], dumps["device"]["keys"])
                     and np.array_equal(dumps["host"]["count"], dumps["device"]["count"]))
    for v in plugins.values():
        v.quit()
    px = cfg.width * cfg.height
    out = {"plugin": kind, "config": name, "frames_timed": len(ms["host"]), "same_keys_and_counts": same_keys}
    for p in ("host", "device"):
        out[f"{p}_ms_per_frame_median"] = round(float(np.median(ms[p])), 3)
        out[f"{p}_ms_per_frame_min_max"] = [round(float(np.min(ms[p])), 3), round(float(np.max(ms[p])), 3)]
        out[f"{p}_h2d_bytes_per_frame"] = h2d_bytes_per_pixel(kind, p == "device") * px
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=4)
    a = ap.parse_args()
    card_before = card()
    rows = [run(kind, name, a.frames, a.warmup) for name in ("C2", "C3") for kind in ("semantic", "voxel")]
    print(json.dumps({"card_before": card_before, "card_after": card(), "rows": rows}))


if __name__ == "__main__":
    main()
