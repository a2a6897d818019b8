"""A worker rank of a multi-GPU dense-mapping plugin (`shard_plugin`): started by the integrator process (rank 0) as

    python -m pyslam_b200.shard_worker --rank r --world N --device d --port p --backend nccl|gloo --timeout s

It joins rank 0's rendezvous store on localhost port p, builds its shard of the map when rank 0 sends SETUP and then
serves rank 0's ops until STOP.  It exits as soon as its parent process is gone."""

from __future__ import annotations

import argparse
import os
import threading
import time


def _exit_with_parent(ppid: int) -> None:
    """Poll the parent pid: a worker reparented to another process has lost rank 0 and ends at once."""
    while True:
        time.sleep(0.25)
        if os.getppid() != ppid:
            os._exit(3)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--rank", type=int, required=True)
    ap.add_argument("--world", type=int, required=True)
    ap.add_argument("--device", type=int, required=True)
    ap.add_argument("--port", type=int, required=True)
    ap.add_argument("--backend", choices=("nccl", "gloo"), required=True)
    ap.add_argument("--timeout", type=float, required=True)
    args = ap.parse_args(argv)
    threading.Thread(target=_exit_with_parent, args=(os.getppid(),), daemon=True).start()

    from datetime import timedelta

    import torch.distributed as dist

    from pyslam_b200 import shard_plugin
    store = dist.TCPStore("127.0.0.1", args.port, args.world, is_master=False,
                          timeout=timedelta(seconds=args.timeout))
    side = shard_plugin.ShardSide(args.rank, args.world, args.device, args.backend, store)
    if args.backend == "nccl":
        import torch
        torch.cuda.set_device(args.device)
    store.set(f"{shard_plugin._UP_KEY}{args.rank}", "1")
    side._init_group(args.timeout)
    try:
        shard_plugin.serve(side)
    finally:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
