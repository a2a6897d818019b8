"""State files of the dense map: the TSDF volume and the point-average and semantic voxel grids (DESIGN.md §7,
"Map state").

One uncompressed `np.savez` file per map or per shard, read without pickle.  Besides the block arrays a file holds the
format version, the map kind (and the semantic kind), the configuration that defines what the voxels mean, the
settings a load restores and the saver's `shard_rank` / `shard_count`.  `read` validates everything before a map is
touched and keeps only the blocks a loading object owns under its own shard setting (`sharding.owner_of`), so a map
saved by N ranks loads into any number of ranks.  This module needs no GPU.

A Bayesian semantic grid with overflow label pairs (`max_label_overflow_pairs`) adds four arrays: `labels_count` int32
[n, B^3] (each voxel's pairs past its 8 in-voxel slots) and `labels_obj` / `labels_cls` int32, `labels_logp` float32
[total] (those pairs, voxel after voxel in block order, each voxel's in slot order).  A file without them is exactly
the file of a grid without overflow pairs.
"""

from __future__ import annotations

import os

import numpy as np

from .sharding import owner_of

IN_VOXEL_PAIRS = 8     # B2V_SEM_MAX_LABELS
LABEL_FIELDS = ("count", "obj", "cls", "logp")

FORMAT_VERSION = 1

# upload chunk of a load: the temporary device copy of a chunk stays near this size whatever the map's
CHUNK_BYTES = 1 << 28


def state_path(ply_path: str) -> str:
    """The state file the plugins write beside `dense_map.ply`: `dense_map.state.npz`."""
    return os.path.splitext(ply_path)[0] + ".state.npz"


def shard_state_path(ply_path: str, rank: int, count: int) -> str:
    """The state file rank `rank` of a `count`-rank plugin writes beside `dense_map.ply`:
    `dense_map.state.<rank>-of-<count>.npz`."""
    return os.path.splitext(ply_path)[0] + f".state.{rank}-of-{count}.npz"


def _shard_sets(ply_path: str) -> dict:
    """count -> {rank: path} of the shard state files beside `ply_path`."""
    head = os.path.basename(os.path.splitext(ply_path)[0]) + ".state."
    folder = os.path.dirname(ply_path) or "."
    sets = {}
    for name in os.listdir(folder) if os.path.isdir(folder) else ():
        if not (name.startswith(head) and name.endswith(".npz")):
            continue
        rank, sep, count = name[len(head):-4].partition("-of-")
        if sep and rank.isdigit() and count.isdigit():
            sets.setdefault(int(count), {})[int(rank)] = os.path.join(os.path.dirname(ply_path), name)
    return sets


def state_files(ply_path: str):
    """What LOAD reads for the map saved as `ply_path`: the single state file when it exists, else the complete set of
    shard files (a list in rank order), else the single file's path (whose load then reports it missing).  ValueError
    when shard files exist but form no complete set, or more than one."""
    single = state_path(ply_path)
    if os.path.exists(single):
        return single
    sets = _shard_sets(ply_path)
    full = [n for n, s in sets.items() if sorted(s) == list(range(n))]
    if sets and len(full) != 1:
        raise ValueError(f"{single} is missing and the shard state files beside it form "
                         f"{'no complete set' if not full else 'more than one set'}: "
                         f"{sorted(os.path.basename(p) for s in sets.values() for p in s.values())}")
    if not sets:
        return single
    return [sets[full[0]][r] for r in range(full[0])]


def remove_other_states(ply_path: str, count: int) -> None:
    """Before a `count`-rank plugin writes its shard files: remove the single file and the shard files of other rank
    counts beside `ply_path`, so that `state_files` finds the new set."""
    if os.path.exists(state_path(ply_path)):
        os.remove(state_path(ply_path))
    for n, s in _shard_sets(ply_path).items():
        if n != count:
            for p in s.values():
                os.remove(p)


def write(path, kind: str, semantic_kind: int, config: dict, settings: dict, shard_rank: int, shard_count: int,
          arrays: dict, labels: dict | None = None) -> None:
    """Write one state file at `path` (exactly that name).  `config` / `settings`: numpy scalars; `arrays`: the
    per-block arrays, keys int32 [n,3] first; `labels`: None, or the overflow label pairs (count, obj, cls, logp)."""
    fields = dict(format_version=np.int32(FORMAT_VERSION), kind=np.str_(kind), semantic_kind=np.int32(semantic_kind),
                  shard_rank=np.int32(shard_rank), shard_count=np.int32(shard_count))
    for name, value in (*config.items(), *settings.items()):
        fields[name] = np.asarray(value)
    for name, a in arrays.items():
        fields["blocks_" + name] = np.ascontiguousarray(a)
    for name, a in (labels or {}).items():
        fields["labels_" + name] = np.ascontiguousarray(a)
    with open(path, "wb") as f:
        np.savez(f, **fields)


def _scalar(z, name, dtype, where):
    if name not in z.files:
        raise ValueError(f"{where}: missing field {name!r}")
    a = z[name]
    if a.shape != () or a.dtype != np.dtype(dtype):
        raise ValueError(f"{where}: field {name!r} must be a {np.dtype(dtype)} scalar, not {a.dtype} {a.shape}")
    return a[()]


def _read_labels(z, blocks, where):
    """The overflow label pairs of one file (None without them), checked against its blocks: counts >= 0, the
    voxels with pairs hold 8 in-voxel pairs (counter = 8 + count), flat arrays as long as the counts' sum, object and
    class ids above INT32_MIN (the association's pending marker) and evidence finite and >= 0."""
    names = {n for n in z.files if n.startswith("labels_")}
    if not names:
        return None
    if names != {"labels_" + n for n in LABEL_FIELDS}:
        raise ValueError(f"{where}: label arrays {sorted(names)} where {['labels_' + n for n in LABEL_FIELDS]} are "
                         "expected")
    lab = {n: z["labels_" + n] for n in LABEL_FIELDS}
    count, counter = lab["count"], blocks.get("counter")
    if counter is None or count.dtype != np.int32 or count.shape != counter.shape:
        raise ValueError(f"{where}: labels_count must be int32 shaped like the counters")
    if count.size and count.min() < 0:
        raise ValueError(f"{where}: negative overflow pair count")
    if np.any((count > 0) & (counter != IN_VOXEL_PAIRS + count)):
        raise ValueError(f"{where}: a voxel with overflow pairs must count {IN_VOXEL_PAIRS} in-voxel pairs plus them")
    total = int(count.sum(dtype=np.int64))
    for n, dt in (("obj", np.int32), ("cls", np.int32), ("logp", np.float32)):
        if lab[n].dtype != dt or lab[n].shape != (total,):
            raise ValueError(f"{where}: labels_{n} must be {np.dtype(dt)} [{total}]")
    if total and (min(lab["obj"].min(), lab["cls"].min()) == np.iinfo(np.int32).min):
        raise ValueError(f"{where}: label ids outside [{np.iinfo(np.int32).min + 1}, {np.iinfo(np.int32).max}]")
    if total and not (np.all(np.isfinite(lab["logp"])) and lab["logp"].min() >= 0):
        raise ValueError(f"{where}: label evidence must be finite and >= 0")
    return lab


def label_slice(labels: dict, a: int, b: int) -> dict:
    """The overflow pairs of blocks [a, b) of `labels` (as `read` returns them)."""
    per_block = labels["count"].reshape(len(labels["count"]), -1).sum(axis=1, dtype=np.int64)
    offs = np.concatenate([[0], np.cumsum(per_block)])
    return dict(count=labels["count"][a:b], **{n: labels[n][offs[a]:offs[b]] for n in LABEL_FIELDS[1:]})


def read(paths, kind: str, semantic_kind: int, config: dict, settings: dict, arrays: dict, shard_rank: int,
         shard_count: int, max_blocks: int, bounds: dict | None = None, labels: bool = False):
    """Validate the state files `paths` (one path or a list) against a loading object and return (settings, blocks):
    the settings every file agrees on and the per-block arrays of the blocks it owns.  `labels` True: (settings,
    blocks, labels) with the overflow label pairs of those blocks (None when no file has any); False: a file with
    them is refused.

    `config`: name -> numpy scalar that must match exactly (dtype and value); `settings`: name -> dtype of the
    restored scalars; `arrays`: name -> (dtype, per-block shape), keys included; `bounds`: name -> (lo, hi) value
    range of an integer array (None: open).  Raises ValueError for a wrong format version, kind, semantic kind or
    configuration, missing or unexpected arrays, wrong dtypes or shapes, a block outside the saver's own shard,
    duplicate keys within or across files, values out of range, disagreeing settings, or more owned blocks than
    `max_blocks`; the label arrays as `_read_labels` checks them.  With label pairs the counter bound applies to the
    in-voxel pairs (counter - labels_count)."""
    if isinstance(paths, (str, os.PathLike)):
        paths = [paths]
    paths = list(paths)
    if not paths:
        raise ValueError("no state file given")
    want = {"blocks_" + n for n in arrays}
    got_settings, parts = None, []
    for path in paths:
        where = os.fspath(path)
        try:
            z = np.load(path, allow_pickle=False)
        except (OSError, ValueError) as e:
            raise ValueError(f"{where}: not a map state file ({e})") from e
        if not isinstance(z, np.lib.npyio.NpzFile):
            raise ValueError(f"{where}: not a map state file")
        with z:
            version = _scalar(z, "format_version", np.int32, where)
            if version != FORMAT_VERSION:
                raise ValueError(f"{where}: format version {version}, this library reads {FORMAT_VERSION}")
            if "kind" not in z.files or z["kind"].shape != () or z["kind"].dtype.kind != "U" or z["kind"][()] != kind:
                raise ValueError(f"{where}: not a {kind} map state")
            sk = _scalar(z, "semantic_kind", np.int32, where)
            if sk != semantic_kind:
                raise ValueError(f"{where}: semantic kind {sk}, expected {semantic_kind}")
            for name, value in config.items():
                v = np.asarray(value)
                got = _scalar(z, name, v.dtype, where)
                if got != v[()]:
                    raise ValueError(f"{where}: {name} = {got} does not match this map's {v[()]}")
            rank = int(_scalar(z, "shard_rank", np.int32, where))
            count = int(_scalar(z, "shard_count", np.int32, where))
            if count < 1 or not 0 <= rank < count:
                raise ValueError(f"{where}: bad shard setting {rank} of {count}")
            s = {name: _scalar(z, name, dt, where) for name, dt in settings.items()}
            if got_settings is None:
                got_settings = s
            else:
                for name in settings:
                    if s[name] != got_settings[name]:
                        raise ValueError(f"{where}: {name} = {s[name]} differs from {got_settings[name]} of "
                                         f"{os.fspath(paths[0])}")
            names = {n for n in z.files if n.startswith("blocks_")}
            if names != want:
                raise ValueError(f"{where}: block arrays {sorted(names)} where {sorted(want)} are expected")
            blocks = {}
            for name, (dt, shape) in arrays.items():
                a = z["blocks_" + name]
                if a.dtype != np.dtype(dt) or a.ndim != 1 + len(shape) or a.shape[1:] != tuple(shape):
                    raise ValueError(f"{where}: block array {name!r} is {a.dtype} {a.shape}, expected {np.dtype(dt)} "
                                     f"[n, {', '.join(map(str, shape))}]")
                blocks[name] = a
            lab = _read_labels(z, blocks, where)
        if lab is not None and not labels:
            raise ValueError(f"{where}: holds overflow label pairs, which this map does not take")
        n = blocks["keys"].shape[0]
        if any(a.shape[0] != n for a in blocks.values()):
            raise ValueError(f"{where}: block arrays of different lengths")
        for name, (lo, hi) in (bounds or {}).items():
            a = blocks[name] if lab is None or name != "counter" else blocks[name] - lab["count"]
            if a.size and ((lo is not None and a.min() < lo) or (hi is not None and a.max() > hi)):
                raise ValueError(f"{where}: {name} outside [{lo}, {hi}]")
        if count > 1 and n and np.any(owner_of(blocks["keys"], count) != rank):
            raise ValueError(f"{where}: holds blocks that shard {rank} of {count} does not own")
        parts.append((blocks, lab))
    keys = np.concatenate([p["keys"] for p, _ in parts])
    if len(keys):
        k = keys[np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))]
        if np.any(np.all(k[1:] == k[:-1], axis=1)):
            raise ValueError("duplicate block keys in the state files")
    own = owner_of(keys, shard_count) == shard_rank if shard_count > 1 else np.ones(len(keys), bool)
    n_own = int(own.sum())
    if n_own > max_blocks:
        raise ValueError(f"the state holds {n_own} blocks for this object, more than its {max_blocks}")
    blocks = {name: np.concatenate([p[name] for p, _ in parts])[own] for name in arrays}
    if not labels:
        return got_settings, blocks
    if all(lab is None for _, lab in parts):
        return got_settings, blocks, None
    # the pairs of the owned blocks, in the order of `blocks`
    labs = [lab or dict(count=np.zeros_like(p["counter"]), obj=np.zeros(0, np.int32), cls=np.zeros(0, np.int32),
                        logp=np.zeros(0, np.float32)) for p, lab in parts]
    count = np.concatenate([lab["count"] for lab in labs])
    per_block = count.reshape(len(count), -1).sum(axis=1, dtype=np.int64)
    keep = np.repeat(own, per_block)
    out = dict(count=count[own], **{n: np.concatenate([lab[n] for lab in labs])[keep] for n in LABEL_FIELDS[1:]})
    return got_settings, blocks, out


def chunks(n: int, block_bytes: int):
    """[start, stop) ranges of an upload of n blocks of block_bytes each in CHUNK_BYTES pieces; one empty range for
    n = 0, so that a load of an empty map still makes its upload call."""
    step = max(1, CHUNK_BYTES // block_bytes)
    return [(s, min(n, s + step)) for s in range(0, n, step)] or [(0, 0)]
