"""Where a fused group's time goes: the allocation against the update, alone and side by side.
C2's 300 device-resident frames, groups of 32 (the bench's workload), steady state (the map is populated first).
    alone    b2v_set_overlap(0): a group's allocation and its update run one after the other on one stream, so the
             CUDA events around each measure that kernel's work with the whole GPU to itself
    in_situ  b2v_set_overlap(1), the bench's schedule: the allocation of the next groups runs beside the update; the
             events measure spans, which include waiting for SMs
Per schedule: wall time of a pass (CUDA events), and per group the allocation (`allocate_group_kernel` and whatever
else the library counts as the group's allocation) and the update (`integrate_group_kernel` + the mask clear), from
b2v_profile_read.  The card's name, power limit and SM clocks are read in the same run.  Prints one JSON line.
python tools/alloc_split.py [--passes 5]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from pyslam_b200 import B200TsdfVolume


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        name, plim, sm, smax = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit_w": float(plim), "sm_mhz_now": float(sm), "sm_max_mhz": float(smax)}
    except Exception as e:  # the measurement stands without it, but says so
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=5)
    args = ap.parse_args()
    cfg, depth, color, Tcw = bench.load_frames("C2", 300, 0, 1)
    d, c = torch.from_numpy(depth).cuda(), torch.from_numpy(color).cuda()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    vol = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 19)
    vol.set_group_size(32)

    def one_pass():
        vol.integrate_batch(d, c, cfg.K, Tcw, stream=stream.cuda_stream)

    for _ in range(3):  # populate: steady state afterwards
        one_pass()
    vol.synchronize()
    out = {"card": card(), "config": "C2 640x480, 300 resident frames per pass, fused groups of 32",
           "passes": args.passes, "blocks": vol.num_blocks()}
    for name, overlap in (("alone", False), ("in_situ", True), ("alone_again", False)):
        vol.set_overlap(overlap)
        vol.set_fusion(True)
        one_pass()  # the schedule's first groups
        vol.synchronize()
        torch.cuda.synchronize()
        vol.profile_enable(True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.passes):
            one_pass()
        e1.record(stream)
        torch.cuda.synchronize()
        a_ms, i_ms, frames, groups = vol.profile_read()
        vol.profile_enable(False)
        pass_ms = e0.elapsed_time(e1) / args.passes
        out[name] = {"pass_ms": round(pass_ms, 4), "frames_per_s": round(300 / (pass_ms * 1e-3), 1),
                     "groups": groups // args.passes,
                     "allocate_us_per_group": round(1e3 * a_ms / groups, 2),
                     "update_us_per_group": round(1e3 * i_ms / groups, 2)}
    a = out["alone"]
    out["allocate_share_alone"] = round(a["allocate_us_per_group"] /
                                        (a["allocate_us_per_group"] + a["update_us_per_group"]), 4)
    out["card_after"] = card()
    vol.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
