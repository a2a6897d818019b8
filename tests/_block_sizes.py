"""Block-size helpers of the grid tests: the reference's key rules for any block side B (voxel_hashing.h:139-161,
voxel_block.h:67-70) in plain Python integers and numpy, and the re-keying of a grid dump between block sizes.

A voxel's state does not depend on B; B only decides which block holds the voxel, the block key and its hash, the
shard owner and the layout.  So a dump at one B is the same map as a dump at another, voxel for voxel: `voxels`
flattens a dump to (voxel keys, per-voxel fields) and `layout` builds the dump of block side B from them, with the
block keys floor_div(v, B), the local index lx + B ly + B^2 lz and the grid's cleared state in the voxels no
observation reached."""

import numpy as np

BLOCK_SIZES = (1, 2, 8, 16)          # the grids' block sizes
RULE_SIZES = (1, 2, 4, 8, 16)        # the key rules hold for every power of two
INVALID_BLOCK_SIZES = (0, 3, 4, 6, 10, 32, -8)


def floor_div(a: int, b: int) -> int:
    """floor(a / b) on Python integers (voxel_hashing.h:139-151)."""
    return a // b


def local_coords(B):
    """[B^3, 3] local key (lx, ly, lz) of each voxel index l = lx + B ly + B^2 lz (voxel_block.h:67-70)."""
    l = np.arange(B ** 3)
    return np.stack([l % B, (l // B) % B, l // (B * B)], 1).astype(np.int64)


def block_keys_of(voxel_keys, B):
    return np.floor_divide(np.asarray(voxel_keys, np.int64), B)


def local_index_of(voxel_keys, B):
    v = np.asarray(voxel_keys, np.int64)
    lk = v - block_keys_of(v, B) * B
    return lk[:, 0] + B * lk[:, 1] + B * B * lk[:, 2]


def block_key_hash(keys):
    """BlockKeyHash (voxel_hashing.h:106-113): h1 ^ (h2 << 1) ^ (h3 << 2) on the sign-extended 64-bit keys."""
    k = np.asarray(keys, np.int64).reshape(-1, 3).astype(np.uint64)
    return k[:, 0] ^ (k[:, 1] << np.uint64(1)) ^ (k[:, 2] << np.uint64(2))


def _sort_keys(k):
    return np.lexsort((k[:, 2], k[:, 1], k[:, 0]))


def voxels(dump, B, fields):
    """(voxel keys [n,3] int64 sorted, {field: [n,...]}) of every voxel of every block of a dump at block side B."""
    keys = np.asarray(dump["keys"], np.int64).reshape(-1, 3)
    vk = (keys[:, None, :] * B + local_coords(B)[None]).reshape(-1, 3)
    order = _sort_keys(vk)
    out = {f: np.asarray(dump[f]).reshape((len(vk),) + np.asarray(dump[f]).shape[2:])[order] for f in fields}
    return vk[order], out


def layout(voxel_keys, values, B, cleared, blocks=None):
    """The sorted dump at block side B of the voxels `voxel_keys` holding `values` ({field: [n,...]}): keys [nb,3]
    (floor_div(v, B), sorted), each field [nb, B^3, ...] with `cleared[field]` in every voxel not listed.  `blocks`:
    the block keys to lay out (default: the blocks of the listed voxels); listed voxels outside them are dropped."""
    vk = np.asarray(voxel_keys, np.int64).reshape(-1, 3)
    bk = block_keys_of(vk, B)
    if blocks is None:
        keys = np.unique(bk, axis=0).reshape(-1, 3)
    else:
        keys = np.asarray(blocks, np.int64).reshape(-1, 3)
    keys = keys[_sort_keys(keys)]
    nv = B ** 3
    out = {"keys": keys.astype(np.int32)}
    row = {tuple(k): i for i, k in enumerate(keys.tolist())}
    b = np.array([row.get(tuple(k), -1) for k in bk.tolist()], np.int64)
    sel = b >= 0
    l = local_index_of(vk, B)
    for f, v in values.items():
        v = np.asarray(v)
        arr = np.empty((len(keys), nv) + v.shape[1:], v.dtype)
        arr[...] = cleared[f]
        arr[b[sel], l[sel]] = v[sel]
        out[f] = arr
    return out


def grid_dump(G, B):
    """`oracle.numpy_grid`'s state as `sort_dump(VoxelBlockGrid(vs, B).dump_blocks())` without the hashes: every
    voxel a point reached, in blocks of side B."""
    return layout(G.keys, dict(count=G.count.astype(np.int32), pos_sum=G.pos, col_sum=G.col), B,
                  dict(count=0, pos_sum=0.0, col_sum=0.0))
