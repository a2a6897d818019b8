"""Seeded call sequences for the TSDF volume (no torch import): what to feed the volume, step by step, and what the CPU
twin gets instead.  tests/test_gpu_tsdf_sequences.py runs them; tests/test_tsdf_sequences_cpu.py checks that the
committed seeds reach every transition the sequences are for.

A step is a dict with an `op`:

* `frames`: `entry` "integrate" (one frame) or "batch" (`n` frames); `kind` host_f32 | host_u16 | pinned | cuda_f32 |
  cuda_u16 (batches only); `shape` (a key of SHAPES) and `kvar` (intrinsics variant: same size, scaled or shifted
  intrinsics); `frames` (frame indices); `stream` None or caller stream 0 / 1 (device kinds only); `event` (a one-shot
  input event, device kinds only); `offset` (device batches: the frames start `offset` frames into a larger tensor,
  odd offsets leave the colour address unaligned for TMA); `stall` (hold the call's stream back first).
* `group_size` (`value` 1..32), `fusion` / `overlap` (`value` bool), `rectify` (`value` None to remove the maps, else
  the shape the maps are for; `swap` BGR input), `upload` (`n_new` new blocks, `n_replace` existing ones, `seed`),
  `reset`, `save_load`, `extract` (`what` mesh | points | dump | capacity).
"""

from __future__ import annotations

import numpy as np

#: (width, height): the T0 test shape, the C1 shape, a width that is not a multiple of 16, an image below one tile
SHAPES = {"T0": (96, 72), "C1": (320, 240), "W": (104, 72), "S": (28, 20)}
KVARS = ("base", "scaled", "shifted")
KINDS = ("host_f32", "host_u16", "pinned", "cuda_f32", "cuda_u16")
DEVICE_KINDS = ("cuda_f32", "cuda_u16")
SEEDS = (3, 17, 29, 41)
N_FRAME_INDICES = 24   # frames are rendered for indices 0..23 of the T0 trajectory (cached by the runner)
DEPTH_SCALE = 1.0 / 5000.0


def intrinsics(shape: str, kvar: str) -> np.ndarray:
    """(fx, fy, cx, cy) of a shape: T0's field of view at that size, scaled by 1.1 or with the principal point shifted
    by (3, -2) pixels for the variants."""
    w, h = SHAPES[shape]
    f = 80.0 * w / 96.0
    K = np.array([f, f, (w - 1) / 2.0, (h - 1) / 2.0])
    if kvar == "scaled":
        K[:2] *= 1.1
    elif kvar == "shifted":
        K[2:] += (3.0, -2.0)
    return K


def generate(seed: int, n_steps: int = 60) -> list:
    rng = np.random.default_rng(seed)
    steps = []
    shape, kvar, rect = "T0", "base", None
    frame_pos = 0

    def take(n):
        nonlocal frame_pos
        idx = [(frame_pos + k) % N_FRAME_INDICES for k in range(n)]
        frame_pos += n
        return idx

    while len(steps) < n_steps:
        k = len(steps)
        if k and k % 14 == 0:
            steps.append(dict(op="extract", what=str(rng.choice(["mesh", "points"]))))
            continue
        r = rng.random()
        if r < 0.55:
            if rng.random() < 0.2:          # a shape or intrinsics change
                new_shape = str(rng.choice(list(SHAPES), p=[0.4, 0.15, 0.25, 0.2]))
                new_kvar = str(rng.choice(KVARS)) if new_shape == shape else "base"
                if (new_shape, new_kvar) != (shape, kvar):
                    shape, kvar = new_shape, new_kvar
                    if rect is not None and rect != shape:   # maps only fit their own image size
                        rect = shape if rng.random() < 0.5 else None
                        steps.append(dict(op="rectify", value=rect, swap=bool(rng.integers(0, 2))))
            kind = str(rng.choice(KINDS, p=[0.25, 0.15, 0.15, 0.3, 0.15]))
            entry = "batch" if kind == "cuda_u16" or rng.random() < 0.45 else "integrate"
            n = int(rng.choice([2, 3, 5, 7, 17, 19, 33, 40])) if entry == "batch" else 1
            if shape == "C1":
                n = min(n, 5)
            dev = kind in DEVICE_KINDS
            stream = (None if rng.random() < 0.4 else int(rng.integers(0, 2))) if dev else None
            steps.append(dict(op="frames", entry=entry, kind=kind, shape=shape, kvar=kvar, frames=take(n),
                              stream=stream, event=bool(dev and stream is None and rng.random() < 0.3),
                              offset=int(rng.choice([0, 1, 3])) if dev and entry == "batch" else 0,
                              stall=bool(dev and rng.random() < 0.35)))
        elif r < 0.63:
            steps.append(dict(op="group_size", value=int(rng.choice([1, 3, 8, 16, 32]))))
        elif r < 0.69:
            steps.append(dict(op="fusion", value=bool(rng.integers(0, 2))))
        elif r < 0.75:
            steps.append(dict(op="overlap", value=bool(rng.integers(0, 2))))
        elif r < 0.81:
            rect = None if rect is not None else shape
            steps.append(dict(op="rectify", value=rect, swap=bool(rng.integers(0, 2))))
        elif r < 0.86:
            steps.append(dict(op="upload", n_new=int(rng.integers(1, 6)), n_replace=int(rng.integers(0, 4)),
                              seed=int(rng.integers(0, 1 << 30))))
        elif r < 0.89:
            steps.append(dict(op="reset"))
        elif r < 0.93:
            steps.append(dict(op="save_load"))
        else:
            steps.append(dict(op="extract", what=str(rng.choice(["mesh", "points", "dump", "capacity"]))))
    return steps


def transitions(steps) -> set:
    """Names of the transitions a sequence makes (the census of tests/test_tsdf_sequences_cpu.py)."""
    out = set()
    prev = None                 # previous frames step
    modes = dict(group_size=16, fusion=True, overlap=True)
    for s in steps:
        op = s["op"]
        if op in modes:
            if s["value"] != modes[op]:
                out.add(f"{op} change" if op == "group_size" else f"{op} {'on' if s['value'] else 'off'}")
            modes[op] = s["value"]
        elif op == "rectify":
            out.add("rectify on" if s["value"] is not None else "rectify off")
        elif op in ("reset", "upload", "save_load"):
            out.add(op)
        elif op == "extract":
            out.add("extract " + s["what"])
        if op != "frames":
            continue
        if prev is not None:
            ps, cs = prev["stream"], s["stream"]
            switch = None
            if ps is not None and cs is None:
                switch = "caller -> library"
            elif ps is None and cs is not None:
                switch = "library -> caller"
            elif ps is not None and cs is not None and ps != cs:
                switch = "caller -> other caller"
            if switch:
                out.add(switch)
                if s["stall"]:
                    out.add("stall before " + switch)
            pa, ca = np.prod(SHAPES[prev["shape"]]), np.prod(SHAPES[s["shape"]])
            if ca < pa:
                out.add("larger -> smaller")
            elif ca > pa:
                out.add("smaller -> larger")
            elif prev["shape"] == s["shape"] and prev["kvar"] != s["kvar"]:
                out.add("new intrinsics, same size")
            u16 = lambda x: x["kind"] in ("host_u16", "cuda_u16")
            dev = lambda x: x["kind"] in DEVICE_KINDS
            unaligned = lambda x: x["offset"] % 2 == 1
            if u16(prev) != u16(s):
                out.add("uint16 -> float32" if u16(prev) else "float32 -> uint16")
            if dev(prev) != dev(s):
                out.add("device -> host" if dev(prev) else "host -> device")
            if unaligned(prev) != unaligned(s):
                out.add("unaligned -> aligned" if unaligned(prev) else "aligned -> unaligned")
        prev = s
    return out


#: every transition the committed seeds must make at least once (over all seeds)
REQUIRED = {
    "caller -> library", "library -> caller", "caller -> other caller",
    "stall before caller -> library", "stall before library -> caller", "stall before caller -> other caller",
    "larger -> smaller", "smaller -> larger", "new intrinsics, same size",
    "uint16 -> float32", "float32 -> uint16", "device -> host", "host -> device",
    "unaligned -> aligned", "aligned -> unaligned",
    "group_size change", "fusion on", "fusion off", "overlap on", "overlap off", "rectify on", "rectify off",
    "reset", "upload", "save_load", "extract mesh", "extract points", "extract dump", "extract capacity",
}
