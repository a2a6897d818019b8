"""numpy restatement of the face-halo exchange of a sharded volume (pyslam_b200/csrc/b2v_shard.cu, DESIGN.md §7):
which (block, destination) records exist, their masks and their voxels in canonical order; the per-rank twin maps
built from them; and the weld of mesh pieces by edge id."""

import numpy as np

import oracle
from pyslam_b200 import sharding

OFFSETS = [(o & 1, (o >> 1) & 1, (o >> 2) & 1) for o in range(1, 8)]   # bit o-1 of a mask: offset o


def halo_shape(mask: int) -> np.ndarray:
    """Voxel indices (increasing) with a local coordinate 0 on every axis of some offset in the mask."""
    v = np.arange(512)
    xyz = np.stack([v & 7, (v >> 3) & 7, v >> 6], 1)
    need = np.zeros(512, bool)
    for o, off in enumerate(OFFSETS):
        if (mask >> o) & 1:
            need |= np.all((xyz == 0) | (np.array(off) == 0), axis=1)
    return v[need]


def numpy_halo_records(keys, vox, world: int):
    """The records a shard holding blocks `keys` int32 [nb,3] (pool order) / `vox` float32 [nb,5,512] sends each of
    `world` ranks: a list of (headers int32 [n,4] = {x,y,z,mask}, payload float32 [m,5]) in pool order."""
    keys = np.asarray(keys, np.int32).reshape(-1, 3)
    vox = np.asarray(vox, np.float32).reshape(len(keys), 5, 512)
    own = sharding.owner_of(keys, world)
    owners = [sharding.owner_of(keys - np.array(off, np.int32), world) for off in OFFSETS]
    out = []
    for r in range(world):
        mask = np.zeros(len(keys), np.int64)
        for o, ow in enumerate(owners):
            mask |= ((ow == r) & (own != r)).astype(np.int64) << o
        idx = np.nonzero(mask)[0]
        headers = np.concatenate([keys[idx], mask[idx, None]], 1).astype(np.int32).reshape(-1, 4)
        payload = [vox[b][:, halo_shape(int(mask[b]))].T for b in idx]
        out.append((headers, np.concatenate(payload).astype(np.float32) if payload else np.zeros((0, 5), np.float32)))
    return out


def halo_blocks(headers, payload):
    """Records -> zero-filled blocks (keys int32 [n,3], vox float32 [n,5,512]) holding the records' voxels."""
    headers = np.asarray(headers).reshape(-1, 4)
    payload = np.asarray(payload).reshape(-1, 5)
    vox = np.zeros((len(headers), 5, 512), np.float32)
    o = 0
    for i, h in enumerate(headers):
        shape = halo_shape(int(h[3]))
        vox[i][:, shape] = payload[o:o + len(shape)].T
        o += len(shape)
    assert o == len(payload)
    return headers[:, :3].astype(np.int32), vox


def shard_dumps(keys, vox, world: int):
    """Split a whole-map dump into the `world` shards' (keys, vox) by BlockKeyHash % world."""
    own = sharding.owner_of(keys, world)
    return [(keys[own == r], vox[own == r]) for r in range(world)]


def received(shards, world: int, r: int):
    """The records rank r receives: every other shard's records for r, in sender order."""
    recs = [numpy_halo_records(k, v, world)[r] for k, v in shards]
    return np.concatenate([h for h, _ in recs]), np.concatenate([x for _, x in recs])


def twin_piece(cfg_args, own_keys, own_vox, headers, payload, unit=16):
    """A TsdfOracle holding a rank's own blocks plus its halo blocks."""
    tw = oracle.TsdfOracle(*cfg_args, unit_resolution=unit)
    for k, v in zip(own_keys, own_vox):
        tw.set_block(k, v)
    hk, hv = halo_blocks(headers, payload)
    for k, v in zip(hk, hv):
        tw.set_block(k, v)
    return tw


def numpy_weld(pieces):
    """Weld of mesh pieces (dicts vertices / colors / edges / triangles with piece-local indices) in piece order: the
    first vertex of each edge id, in order of first occurrence; triangles re-indexed, piece-major."""
    V = np.concatenate([p["vertices"] for p in pieces]).reshape(-1, 3)
    Cc = np.concatenate([p["colors"] for p in pieces]).reshape(-1, 3)
    E = np.concatenate([p["edges"] for p in pieces]).reshape(-1, 4)
    base = np.cumsum([0] + [len(p["vertices"]) for p in pieces])
    T = np.concatenate([np.asarray(p["triangles"], np.int64).reshape(-1, 3) + base[i] for i, p in enumerate(pieces)])
    _, first, inv = np.unique(E, axis=0, return_index=True, return_inverse=True)
    inv = inv.reshape(-1)
    keep = np.zeros(len(E), bool)
    keep[first] = True
    newidx = np.cumsum(keep) - 1
    remap = newidx[first[inv]]
    return dict(vertices=V[keep], colors=Cc[keep], edges=E[keep], triangles=remap[T].astype(np.int64))


def triangle_roots_ok(edges, triangles, owned_keys) -> bool:
    """Every triangle lies in the 9^3 tile of one of `owned_keys` (its vertices' owner voxels do)."""
    owned = {tuple(k) for k in np.asarray(owned_keys).tolist()}
    E = np.asarray(edges)[:, :3].astype(np.int64)
    for t in np.asarray(triangles).reshape(-1, 3):
        p = E[t]
        lo, hi = p.min(0), p.max(0)
        ok = False
        for off in [(0, 0, 0)] + OFFSETS:
            b = (lo >> 3) - np.array(off)
            if tuple(b.tolist()) in owned and np.all(lo >= 8 * b) and np.all(hi <= 8 * b + 8):
                ok = True
                break
        if not ok:
            return False
    return True
