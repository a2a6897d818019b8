"""Cost of saving and loading the dense map's state (`save_state` / `load_state`, DESIGN.md §7 "Map state"):
    tsdf      C2, 300 frames through the TSDF volume (integrate_batch, unit resolution 16, fixed 2^19 blocks)
    grid      C2, 300 frames through the point-average grid (b2v_grid_integrate_rgbd, fixed 2^17 blocks)
    semantic  C3, 16 frames with class and instance images through the Bayesian grid at 0.015 m (growable 2^10 ->
              2^16), each frame associated (carving on) and integrated with its object image
Per map: blocks, file bytes, and wall time of the two halves of a save (device -> host export; file write) and of a
load (file read + validation; clear + chunked host -> device upload), each ending in a device synchronise, best of
three; and whether the loaded map equals the saved one.  The file goes to a temporary directory.  Prints one JSON line
with the card's name, power limit and maximum SM clock.
python tools/map_state_cost.py"""
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from pyslam_b200 import (B200TsdfVolume, CameraFrustrum, VoxelBlockGrid, VoxelBlockSemanticProbabilisticGrid,
                         map_state)
from pyslam_b200 import synthetic as S
from pyslam_b200.volume import _as_K4
from tests._util import sort_dump


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def best(fn, reps=3):
    t, out = min((wall(fn) for _ in range(reps)), key=lambda x: x[0])
    return round(1e3 * t, 1), out


def tsdf_map():
    cfg, depth, color, Tcw = bench.load_frames("C2", 300, 0, 1)
    vol = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 19)
    vol.integrate_batch(depth, color, cfg.K, Tcw)
    vol.synchronize()
    return vol, lambda: B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 19)


def grid_map():
    cfg, depth, color, Tcw = bench.load_frames("C2", 300, 0, 1)
    g = VoxelBlockGrid(cfg.voxel_size, 8, capacity_blocks=1 << 17)
    for i in range(len(depth)):
        g.integrate_rgbd(depth[i], color[i], cfg.K, S.inv_T(Tcw[i]), max_depth=cfg.depth_trunc)
    return g, lambda: VoxelBlockGrid(cfg.voxel_size, 8, capacity_blocks=1 << 17)


def semantic_map():
    cfg, depth, color, Tcw = bench.load_frames("C3", 16, 0, 1)
    step = max(cfg.n_frames // len(depth), 1)
    K4 = _as_K4(cfg.K)

    def make():
        return VoxelBlockSemanticProbabilisticGrid(0.015, 8, capacity_blocks=1 << 10, max_capacity_blocks=1 << 16)

    g = make()
    for i in range(len(depth)):
        cls = S.render_class_ids(cfg, i * step).astype(np.int32)
        inst = np.where(cls % 3 == 0, -1, cls * 7 + np.arange(cls.shape[1])[None, :] // 400).astype(np.int32)
        fr = CameraFrustrum(*K4, depth.shape[2], depth.shape[1], Tcw[i], depth_max=cfg.depth_trunc, depth_min=1e-2)
        st = g.set_frame(depth[i], color[i], cls, inst)
        g.assign_object_ids_to_instance_ids(fr, st.class_image, st.instance_image, st.depth, depth_threshold=0.08,
                                            do_carving=True)
        g.integrate_rgbd(st.depth, st.color, cfg.K, S.inv_T(Tcw[i]), st.class_image, g.remap_instance_ids(),
                         max_depth=cfg.depth_trunc)
    return g, make


def blocks_of(m):
    d = m.export_blocks() if hasattr(m, "export_blocks") else m._export_state()
    return sort_dump(d)


def measure(m, make, path):
    t_export, arrays = best(m._export_state)
    t_write, _ = best(lambda: map_state.write(path, m._STATE_KIND, m._state_semantic_kind(), m._state_config(),
                                              m._state_settings(), m.shard_rank, m.shard_count, arrays))
    n = make()
    spec = n._state_arrays()
    block_bytes = sum(np.dtype(dt).itemsize * int(np.prod(shape)) for dt, shape in spec.values())
    t_read, (settings, blocks) = best(lambda: map_state.read(
        path, n._STATE_KIND, n._state_semantic_kind(), n._state_config(),
        {k: np.asarray(v).dtype for k, v in n._state_settings().items()}, spec, n.shard_rank, n.shard_count,
        n._state_capacity(), n._STATE_BOUNDS))

    def upload():
        n._clear_state()
        for a, b in map_state.chunks(len(blocks["keys"]), block_bytes):
            n._upload_state({k: x[a:b] for k, x in blocks.items()})
        n._restore_settings(settings)

    t_upload, _ = best(upload)
    x, y = blocks_of(m), blocks_of(n)
    same = all(np.array_equal(x[k], y[k], equal_nan=True) for k in x)
    return {"blocks": int(len(arrays["keys"])), "file_bytes": os.path.getsize(path),
            "save_export_ms": t_export, "save_write_ms": t_write, "load_read_ms": t_read, "load_upload_ms": t_upload,
            "bit_exact": bool(same)}


def main():
    out = {"gpu": card()}
    with tempfile.TemporaryDirectory() as tmp:
        for name, build in (("tsdf_C2_300_frames", tsdf_map), ("grid_C2_300_frames", grid_map),
                            ("bayesian_C3_16_frames", semantic_map)):
            m, make = build()
            path = os.path.join(tmp, name + ".npz")
            out[name] = measure(m, make, path)
            os.remove(path)
            m.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
