"""One dense map over several GPUs behind one pySLAM plugin: the integrator process is rank 0 and drives N - 1 worker
processes (`python -m pyslam_b200.shard_worker`), one per further entry of `kVolumetricIntegrationB200Devices`; every
rank holds the blocks `BlockKeyHash % N` gives it (DESIGN.md §7, "Multi-GPU plugins").

The protocol is SPMD, one op at a time, all started by rank 0 (`ShardGroup.run`):

1. rank 0 publishes a small header in the rendezvous store: op name, scalars and the shape and dtype of each payload
   array.  Workers idle on the store, not in a collective, so an integrator that waits for keyframes for a long time
   never runs into the process group's timeout;
2. rank 0 broadcasts the payload arrays: device tensors over NCCL when the device ids are distinct, host tensors over
   gloo when one repeats (ranks that share a GPU);
3. every rank makes the same call on its shard: the plugin method `_op_<name>(meta, **arrays)`, which is the plugin's
   own loop body (the sharded grids and the volume expect every call on every rank with the same arguments);
4. an all-reduce of a status word ends the op.  If a rank failed, the first failing rank broadcasts its message and
   rank 0 raises it as RuntimeError; the plugin's task loop logs it and goes on.

A collective that fails (a worker died, the timeout expired) takes the whole group down: rank 0 kills the workers and
every later op raises.  A worker exits when its parent process is gone, whatever it is doing.
"""

from __future__ import annotations

import atexit
import os
import pickle
import subprocess
import sys
import time
import traceback
from datetime import timedelta
from types import SimpleNamespace

import numpy as np

# process-group timeout: the longest a rank waits for its peers inside one op
TIMEOUT_S = 300.0
# the longest rank 0 waits for the workers to start (each imports torch and creates a CUDA context)
START_TIMEOUT_S = 300.0
# the longest STOP waits for a worker to exit before it is killed
JOIN_TIMEOUT_S = 30.0
# "module:function" that builds a worker's plugin from the SETUP spec (a test puts a recording stand-in here)
WORKER_FACTORY = "pyslam_b200.shard_plugin:worker_plugin"

_OP_KEY = "b200/op/"
_UP_KEY = "b200/up/"


def device_count() -> int:
    import torch
    return torch.cuda.device_count()


def parse_devices(value) -> list:
    """The device ids of kVolumetricIntegrationB200Devices: a list of ints in [0, device_count()); RuntimeError
    otherwise.  An empty list needs no device query."""
    if not isinstance(value, list):
        raise RuntimeError(f"kVolumetricIntegrationB200Devices must be a list of CUDA device ids, not {value!r}")
    if any(isinstance(d, bool) or not isinstance(d, (int, np.integer)) for d in value):
        raise RuntimeError(f"kVolumetricIntegrationB200Devices must hold integer device ids, not {value!r}")
    ids = [int(d) for d in value]
    if ids:
        n = device_count()
        bad = [d for d in ids if not 0 <= d < n]
        if bad:
            raise RuntimeError(f"kVolumetricIntegrationB200Devices: device ids {bad} outside [0, {n})")
    return ids


def backend_for(devices) -> str:
    """NCCL with device tensors when every rank has its own GPU; gloo with host tensors when an id repeats."""
    return "nccl" if len(set(devices)) == len(devices) else "gloo"


class ShardSide:
    """One rank's end of the group: its rank, the world size, its device, the backend, and the payload and status
    transport of an op."""

    def __init__(self, rank: int, world: int, device: int, backend: str, store):
        self.rank, self.world, self.device, self.backend, self.store = rank, world, int(device), backend, store

    @property
    def _torch_device(self):
        import torch
        return torch.device("cuda", self.device) if self.backend == "nccl" else torch.device("cpu")

    def _init_group(self, timeout: float):
        import torch
        import torch.distributed as dist
        if dist.is_initialized():
            raise RuntimeError("this process already has a default torch.distributed process group")
        kw = dict(device_id=torch.device("cuda", self.device)) if self.backend == "nccl" else {}
        dist.init_process_group(self.backend, store=dist.PrefixStore("pg/", self.store), rank=self.rank,
                                world_size=self.world, timeout=timedelta(seconds=timeout), **kw)

    def _view(self, flat, shape, dtype):
        """The array a flat uint8 tensor holds: a CUDA tensor view over NCCL, a numpy view over gloo."""
        import torch
        if self.backend == "nccl":
            return flat.view(torch.from_numpy(np.zeros(0, dtype)).dtype).reshape(shape)
        return flat.numpy().view(dtype).reshape(shape)

    def send(self, a: np.ndarray):
        """Broadcast `a` from rank 0 (uploaded once over NCCL); returns the array rank 0 itself computes with."""
        import torch
        import torch.distributed as dist
        a = np.ascontiguousarray(a)
        flat = torch.from_numpy(a.reshape(-1).view(np.uint8))
        if self.backend == "nccl":
            flat = flat.to(self._torch_device)
        if flat.numel():
            dist.broadcast(flat, 0)
        return self._view(flat, a.shape, a.dtype) if self.backend == "nccl" else a

    def recv(self, shape, dtype):
        import torch
        import torch.distributed as dist
        dtype = np.dtype(dtype)
        flat = torch.empty(int(np.prod(shape)) * dtype.itemsize, dtype=torch.uint8, device=self._torch_device)
        if flat.numel():
            dist.broadcast(flat, 0)
        return self._view(flat, tuple(shape), dtype)

    def finish(self, err, result=None):
        """The status all-reduce that ends every op; the first failing rank's message (None when all succeeded).
        It also gathers every rank's op result when that is an int (else -1) into `words`, rank by rank: a value each
        rank computes for itself, such as the frame-store slot it filled, which rank 0 can check all ranks agree on."""
        import torch
        import torch.distributed as dist
        flags = torch.zeros(2 * self.world, dtype=torch.int64, device=self._torch_device)
        flags[self.rank] = 1 if err else 0
        word = result if isinstance(result, (int, np.integer)) and not isinstance(result, bool) else -1
        flags[self.world + self.rank] = int(word)
        dist.all_reduce(flags)
        flags = flags.cpu().tolist()
        self.words = flags[self.world:]
        failed = [r for r, f in enumerate(flags[:self.world]) if f]
        if not failed:
            return None
        msg = [err if self.rank == failed[0] else None]
        dist.broadcast_object_list(msg, src=failed[0], device=self._torch_device)
        return msg[0]


def _execute(plugin, op, meta, arrays, rank):
    """(result, None) of `plugin._op_<op>(meta, **arrays)`, or (None, message) when it raised."""
    try:
        return getattr(plugin, "_op_" + op)(meta, **arrays), None
    except Exception as e:
        return None, f"rank {rank}: {type(e).__name__}: {e}"


class ShardGroup(ShardSide):
    """Rank 0's end: starts the workers, runs every op, and shuts them down (`close`).  Whatever happens, no worker
    outlives it: a failed start kills them, `close` joins them with a timeout and kills the rest, and it also runs at
    interpreter exit."""

    def __init__(self, devices, timeout: float | None = None):
        import torch.distributed as dist
        devices = [int(d) for d in devices]
        self.timeout = float(TIMEOUT_S if timeout is None else timeout)
        store = dist.TCPStore("127.0.0.1", 0, len(devices), is_master=True, timeout=timedelta(seconds=self.timeout),
                              wait_for_workers=False)
        super().__init__(0, len(devices), devices[0], backend_for(devices), store)
        self.devices, self.procs, self.plugin = devices, [], None
        self._seq, self._closed, self._broken, self._group = 0, False, None, False
        atexit.register(self.close)
        try:
            root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
            env = dict(os.environ)
            env["PYTHONPATH"] = os.pathsep.join([root] + [p for p in [env.get("PYTHONPATH")] if p])
            for r in range(1, self.world):
                self.procs.append(subprocess.Popen(
                    [sys.executable, "-m", "pyslam_b200.shard_worker", "--rank", str(r), "--world", str(self.world),
                     "--device", str(devices[r]), "--port", str(store.port), "--backend", self.backend,
                     "--timeout", str(self.timeout)], env=env))
            deadline = time.monotonic() + START_TIMEOUT_S
            while not store.check([f"{_UP_KEY}{r}" for r in range(1, self.world)]):
                self._check_alive()
                if time.monotonic() > deadline:
                    raise RuntimeError(f"the shard workers did not start within {START_TIMEOUT_S:.0f} s")
                time.sleep(0.05)
            self._init_group(self.timeout)
            self._group = True
        except BaseException:
            self.close()
            raise

    def _check_alive(self):
        for r, p in enumerate(self.procs, 1):
            if p.poll() is not None:
                raise RuntimeError(f"shard worker {r} exited with status {p.returncode}")

    def agreed(self):
        """The int result every rank returned from the last op, or -1 when the ranks' results differ."""
        w = self.words
        return w[0] if all(x == w[0] for x in w) else -1

    def _fail(self, msg):
        self._broken = msg
        self.close()
        raise RuntimeError(f"the shard group is down: {msg}")

    def run(self, op: str, meta: dict | None = None, arrays: dict | None = None):
        """One op on every rank; rank 0's result (every rank's int result in `words`, see `finish`).  RuntimeError
        when a rank failed (the group stays up) or the group failed (it is then shut down and every later op
        raises)."""
        if self._closed:
            raise RuntimeError(f"the shard group is down: {self._broken or 'stopped'}")
        meta, arrays = meta or {}, arrays or {}
        try:
            self._check_alive()
        except RuntimeError as e:
            self._fail(str(e))
        arrays = {k: None if a is None else np.asarray(a) for k, a in arrays.items()}
        spec = {k: None if a is None else (a.shape, a.dtype.str) for k, a in arrays.items()}
        self._seq += 1
        try:
            self.store.set(f"{_OP_KEY}{self._seq}", pickle.dumps((op, meta, spec)))
            local = {k: None if a is None else self.send(a) for k, a in arrays.items()}
        except Exception as e:
            self._fail(f"{op}: {e}")
        result, err = _execute(self.plugin, op, meta, local, 0)
        try:
            msg = self.finish(err, result)
            if self._seq > 1:   # every worker has read the previous header
                self.store.delete_key(f"{_OP_KEY}{self._seq - 1}")
        except Exception as e:
            self._fail(f"{op}: {e}")
        if msg:
            raise RuntimeError(msg)
        return result

    def close(self):
        """STOP: the workers are told to exit, joined with a timeout and killed if still there; the process group is
        destroyed.  Idempotent."""
        if self._closed:
            return
        self._closed = True
        atexit.unregister(self.close)
        if self._group and not self._broken:
            try:
                self.store.set(f"{_OP_KEY}{self._seq + 1}", pickle.dumps(("stop", {}, {})))
            except Exception:
                pass
        for p in self.procs:
            try:
                p.wait(timeout=JOIN_TIMEOUT_S if self._group and not self._broken else 0.1)
            except subprocess.TimeoutExpired:
                p.kill()
                p.wait()
        if self._group:
            import torch.distributed as dist
            try:
                dist.destroy_process_group()
            except Exception:
                pass
            self._group = False


# ---- worker side ------------------------------------------------------------------------------------------------------

class _WorkerBase:
    """What a worker's plugin instance needs of pySLAM's base class: nothing but a quiet `print` (rank 0 reports)."""
    print = staticmethod(lambda *a, **k: None)


def worker_plugin(spec: dict, side: ShardSide):
    """A worker's plugin: an instance of the same plugin class, built against `_WorkerBase`, carrying rank 0's
    configuration (`spec["attrs"]`); the SETUP op then builds its map (`_op_setup`)."""
    from . import integrator, integrator_semantic
    make = {"tsdf": integrator.make_integrator_class,
            "voxel_grid": integrator_semantic.make_voxel_grid_integrator_class,
            "semantic": integrator_semantic.make_semantic_integrator_class}[spec["kind"]]
    cls = make(_WorkerBase, SimpleNamespace(VolumetricIntegrationTaskType=None))
    plugin = cls.__new__(cls)
    plugin.__dict__.update(spec["attrs"])
    plugin._shards = side
    return plugin


def _wait_key(store, key):
    """The value of `key` once rank 0 has set it (polled, so that an idle worker holds no collective open)."""
    pause = 0.0002
    while not store.check([key]):
        time.sleep(pause)
        pause = min(2 * pause, 0.01)
    return store.get(key)


def serve(side: ShardSide):
    """A worker's command loop: SETUP builds the plugin, every other op runs its `_op_` method, STOP ends it."""
    import importlib
    plugin, seq = None, 0
    try:
        while True:
            seq += 1
            op, meta, spec = pickle.loads(_wait_key(side.store, f"{_OP_KEY}{seq}"))
            if op == "stop":
                return
            arrays = {k: None if s is None else side.recv(*s) for k, s in spec.items()}
            if op == "setup":
                try:
                    mod, fn = meta["factory"].split(":")
                    plugin = getattr(importlib.import_module(mod), fn)(meta, side)
                except Exception as e:
                    traceback.print_exc()
                    side.finish(f"rank {side.rank}: {type(e).__name__}: {e}")
                    continue
            if plugin is None:
                side.finish(f"rank {side.rank}: {op} before setup")
                continue
            result, err = _execute(plugin, op, meta, arrays, side.rank)
            side.finish(err, result)
    finally:
        if plugin is not None and getattr(plugin, "volume", None) is not None:
            plugin.volume.close()
