"""Cost of a growable block pool: C2's 300 frames (device-resident), three passes, into three volumes
    fixed      capacity 2^19
    grow12_19  capacity 2^12, growth ceiling 2^19
    grow19_22  capacity 2^19, growth ceiling 2^22 (hash table and bookkeeping sized for 2^22)
Per volume: wall time of the first pass (where the pool grows) and of the two steady passes, growths, first-pass time
over the fixed volume's per growth, final capacity, device memory held (drop of free memory), allocate-kernel time of
every pass (b2v_profile_read), and whether the three final volumes are equal bit for bit.  Prints one JSON line.
python tools/growth_cost.py"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from pyslam_b200 import B200TsdfVolume


def sorted_blocks(vol):
    keys, vox = vol.export_blocks_torch()
    k = keys[:, :3].to(torch.int64) + (1 << 20)
    order = torch.argsort((k[:, 0] << 42) | (k[:, 1] << 21) | k[:, 2])
    return keys[order], vox[order].view(torch.int32)


def main():
    cfg, depth, color, Tcw = bench.load_frames("C2", 300, 0, 1)
    d, c = torch.from_numpy(depth).cuda(), torch.from_numpy(color).cuda()
    setups = {"fixed": (1 << 19, None), "grow12_19": (1 << 12, 1 << 19), "grow19_22": (1 << 19, 1 << 22)}
    out = {"gpu": torch.cuda.get_device_name(0), "frames": 300, "passes": 3}
    warm = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 16)  # module loads
    warm.integrate_batch(d[:32], c[:32], cfg.K, Tcw[:32])
    warm.synchronize()
    warm.close()
    ref = None
    for name, (cap, mx) in setups.items():
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        vol = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=cap,
                             max_capacity_blocks=mx)
        held_at_create = free0 - torch.cuda.mem_get_info()[0]
        vol.set_group_size(32)
        r = {"pass_s": [], "allocate_ms": []}
        for _ in range(3):
            vol.profile_enable(True)
            t0 = time.perf_counter()
            vol.integrate_batch(d, c, cfg.K, Tcw)
            vol.synchronize()
            r["pass_s"].append(round(time.perf_counter() - t0, 4))
            r["allocate_ms"].append(round(vol.profile_read()[0], 2))
            vol.profile_enable(False)
        r["capacity_blocks"], r["growths"] = vol.capacity()
        r["blocks"] = vol.num_blocks()
        r["held_gb_at_create"] = round(held_at_create / 1e9, 3)
        r["held_gb_final"] = round((free0 - torch.cuda.mem_get_info()[0]) / 1e9, 3)
        keys, vox = sorted_blocks(vol)
        if ref is None:
            ref = (keys, vox)
            r["equal_to_fixed"] = True
        else:
            r["equal_to_fixed"] = bool(torch.equal(keys, ref[0]) and torch.equal(vox, ref[1]))
        del keys, vox
        vol.close()
        out[name] = r
    for name in ("grow12_19", "grow19_22"):
        g = out[name]["growths"]
        extra = out[name]["pass_s"][0] - out["fixed"]["pass_s"][0]
        out[name]["first_pass_extra_s_per_growth"] = round(extra / g, 4) if g else None
    print(json.dumps(out))


if __name__ == "__main__":
    main()
