"""Cost of growable grid storage, on the bench's grid and semantic legs:
    grid      C2, 300 frames (device-resident) through b2v_grid_integrate_rgbd: fixed 2^17 vs growable 2^10 -> 2^17
    semantic  C3, 16 frames + class images through VoxelBlockSemanticProbabilisticGrid.integrate_rgbd at 0.015 m:
              fixed 2^16 vs growable 2^10 -> 2^16
Per grid: ms per frame of the first pass (where the storage grows) and of a second, steady pass, growths, storage at the
end, device memory held (drop of free memory at creation and at the end) and whether the grown grid's outputs equal the
fixed grid's: keys and counts bit for bit (the point grid's float sums are compared to float-atomic tolerance on these
real frames, where the order of the adds differs between any two runs), the semantic dump bit for bit.  Prints one JSON
line with the card's name and power limit.
python tools/grid_growth_cost.py"""
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
from tests._util import sort_dump


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed_grid(make, run, passes=2):
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    g = make()
    r = {"held_gb_at_create": round((free0 - torch.cuda.mem_get_info()[0]) / 1e9, 3), "ms_per_frame": []}
    for k in range(passes):
        if k:
            g.clear()   # same frames again into the storage the first pass grew
        t0 = time.perf_counter()
        n = run(g)
        r["ms_per_frame"].append(round(1e3 * (time.perf_counter() - t0) / n, 3))
    r["storage_blocks"], r["growths"] = g.capacity()
    r["blocks"] = g.num_blocks()
    r["held_gb_final"] = round((free0 - torch.cuda.mem_get_info()[0]) / 1e9, 3)
    return g, r


def main():
    out = {"gpu": card()}
    # ---- point-average grid: the bench's grid leg on 300 device frames
    cfg, depth, color, Tcw = bench.load_frames("C2", 300, 0, 1)
    d_dev, c_dev = torch.from_numpy(depth).cuda(), torch.from_numpy(color).cuda()
    K4 = np.array(cfg.K, np.float64)
    Twc = [np.ascontiguousarray(S.inv_T(Tcw[i])).reshape(16) for i in range(len(depth))]

    def grid_pass(g):
        for i in range(len(depth)):
            rc = g._L.b2v_grid_integrate_rgbd(g._h, d_dev[i].data_ptr(), c_dev[i].data_ptr(), depth.shape[1],
                                              depth.shape[2], K4.ctypes.data, Twc[i].ctypes.data,
                                              float(cfg.depth_trunc), 0.0, 0)
            assert rc == 0
        g._check(g._L.b2v_grid_synchronize(g._h), "sync")
        return len(depth)

    warm = VoxelBlockGrid(cfg.voxel_size, 8, capacity_blocks=1 << 12, max_capacity_blocks=1 << 17)  # module loads
    grid_pass(warm)
    warm.close()
    dumps = {}
    for name, (cap, mx) in {"fixed_2^17": (1 << 17, None), "grow_2^10_2^17": (1 << 10, 1 << 17)}.items():
        g, r = timed_grid(lambda: VoxelBlockGrid(cfg.voxel_size, 8, capacity_blocks=cap, max_capacity_blocks=mx),
                          grid_pass)
        dumps[name] = sort_dump(g.dump_blocks())
        g.close()
        out.setdefault("grid_C2_300_frames", {})[name] = r
    a, b = dumps["fixed_2^17"], dumps["grow_2^10_2^17"]
    out["grid_C2_300_frames"]["keys_counts_equal"] = bool(np.array_equal(a["keys"], b["keys"]) and
                                                          np.array_equal(a["count"], b["count"]))
    out["grid_C2_300_frames"]["sums_max_abs_diff"] = float(max(np.abs(a["pos_sum"] - b["pos_sum"]).max(),
                                                               np.abs(a["col_sum"] - b["col_sum"]).max()))
    del dumps, a, b, d_dev, c_dev
    # ---- semantic grid: the bench's semantic leg
    cfg, depth, color, Tcw = bench.load_frames("C3", 16, 0, 1)
    labels = [S.render_class_ids(cfg, i * max(cfg.n_frames // len(depth), 1)) for i in range(len(depth))]

    def sem_pass(g):
        for i in range(len(depth)):
            g.integrate_rgbd(depth[i], color[i], cfg.K, S.inv_T(Tcw[i]), class_image=labels[i],
                             max_depth=cfg.depth_trunc)
        return len(depth)

    dumps = {}
    for name, (cap, mx) in {"fixed_2^16": (1 << 16, None), "grow_2^10_2^16": (1 << 10, 1 << 16)}.items():
        g, r = timed_grid(lambda: VoxelBlockSemanticProbabilisticGrid(0.015, 8, capacity_blocks=cap,
                                                                      max_capacity_blocks=mx), sem_pass)
        dumps[name] = sort_dump(g.dump_blocks(8))
        r["label_overflows"] = g.label_overflows()
        g.close()
        out.setdefault("semantic_C3_16_frames", {})[name] = r
    a, b = dumps["fixed_2^16"], dumps["grow_2^10_2^16"]
    out["semantic_C3_16_frames"]["dumps_equal"] = bool(all(np.array_equal(a[k], b[k], equal_nan=True) for k in a))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
