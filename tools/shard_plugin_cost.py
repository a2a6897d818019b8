"""Cost of the multi-process plugin (kVolumetricIntegrationB200Devices): the TSDF plugin on C2-shape keyframes (raw
uint16 depth, GPU rectification) at N = 1 and at every N the machine allows.  Prints one JSON line:

  keyframe_ms_median   wall time per keyframe, task in to output out (integrate + mesh, OutputTimeInterval 0)
  backlog_fps          frames per second a 300-frame backlog drains at (fused batches of MaxBatch), output included

N = 2 over gloo with both ranks on GPU 0 measures the protocol's overhead on a one-GPU machine; NCCL rows appear only
with two or more GPUs.  The card's name and power limit are read in the same run.

    python tools/shard_plugin_cost.py [--keyframes 20] [--backlog 300]
"""

import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    except Exception:
        q = []
    return dict(name=torch.cuda.get_device_name(0), nvidia_smi=q, device_count=torch.cuda.device_count())


def _run(devices, frames, n_key, n_backlog, cfg):
    from pyslam_b200.integrator import make_integrator_class
    from tests import plugin_standins as P
    api = SimpleNamespace(**{**vars(P.API), "USE_CPP": True})
    Cls = make_integrator_class(P.StandaloneIntegratorBase, api)
    y, x = np.mgrid[:cfg.height, :cfg.width].astype(np.float32)
    cam = SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None,
                          depth_factor=1.0 / 5000.0)
    integ = Cls(cam, P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF", calib_maps=(x, y),
                kVolumetricIntegrationVoxelLength=cfg.voxel_size, kVolumetricIntegrationTSdfTrunc=cfg.sdf_trunc,
                kVolumetricIntegrationB200CapacityBlocks=1 << 17, kVolumetricIntegrationOutputTimeInterval=0.0,
                kVolumetricIntegrationB200Devices=list(devices))

    def kd(i):
        d, c, T = frames[i % len(frames)]
        return P.VolumetricIntegrationKeyframeData(id=i, pose=T, img=c, depth=d)

    try:
        times = []
        for i in range(n_key + 3):
            t0 = time.perf_counter()
            integ.add_keyframe_data(kd(i))
            integ.step()
            assert integ.pop_output() is not None
            times.append(time.perf_counter() - t0)
        integ.reset()
        for i in range(n_backlog):
            integ.add_keyframe_data(kd(i))
        t0 = time.perf_counter()
        integ.run_pending()
        integ.add_update_output_task()
        integ.step()
        while integ.pop_output() is not None:
            pass
        dt = time.perf_counter() - t0
    finally:
        integ.quit()
    return dict(devices=list(devices), backend=None if len(devices) < 2 else integ._shards.backend,
                keyframe_ms_median=round(1e3 * float(np.median(times[3:])), 3), backlog_fps=round(n_backlog / dt, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, default=20)
    ap.add_argument("--backlog", type=int, default=300)
    a = ap.parse_args()
    import torch
    from pyslam_b200 import synthetic as S
    cfg = S.CONFIGS["C2"]
    frames = []
    for i in range(24):
        d, c, T = S.render_frame(cfg, i)
        frames.append((np.round(d * 5000.0).astype(np.uint16), np.ascontiguousarray(c[..., ::-1]), T))
    n = torch.cuda.device_count()
    layouts = [[], [0, 0]] + [list(range(k)) for k in range(2, n + 1)]
    rows = [_run(d, frames, a.keyframes, a.backlog, cfg) for d in layouts]
    print(json.dumps(dict(tool="shard_plugin_cost", config="C2", card=_card(), rows=rows)))


if __name__ == "__main__":
    main()
