"""Scenes and oracle views of tests/test_gpu_grid_matrix.py and tests/test_grid_matrix_cpu.py: the grids' features
combined - the Bayesian grid's overflow label store at block sides 1, 2 and 16, together with block-pool growth,
shards and state files, and the point-average grid's input-order sums with growth, shards, state files, staged frames
and edits at those block sides.

A voxel's state does not depend on the block side B, so the oracles keep it per voxel and these views lay it out at
B (tests/_block_sizes.py): `unbounded_dump` is what `sort_dump(grid.dump_blocks(K))` of a Bayesian grid with a store
must equal, `unbounded_overflow_pairs` what its `export_labels()` must hold (re-ordered by `sorted_labels`), pair for
pair in slot order, and `BS.grid_dump` is the point-average view."""

import copy
from functools import lru_cache

import numpy as np

from tests import _block_sizes as BS
from tests import _grid_order_scenes as O
from tests import _grid_prep_scenes as E
from tests import _semantic_labels as SL
from tests import _semantic_scenes as SC

f32 = np.float32
SEM_FIELDS = ("count", "pos_sum", "col_sum", "object_id", "class_id", "confidence", "aux", "lab_obj", "lab_cls",
              "lab_logp")
SEM_CLEARED = dict(count=0, pos_sum=0.0, col_sum=0.0, object_id=-1, class_id=-1, confidence=0.0, aux=0, lab_obj=-1,
                   lab_cls=-1, lab_logp=-np.inf)
CTA_VOXELS = 512    # the per-voxel passes run one 512-thread CTA per 512 pool voxels, whatever B


# ---- the oracle and its views at block side B ----------------------------------------------------------------------

class MatrixOracle(SL.UnboundedSemanticGrid):
    """The unbounded label map that also keeps every voxel a point reached since the last clear.  A grid of block side
    B holds the blocks of those voxels; below B = 8 they are not all visible in the B = 8 state once an edit has reset
    voxels."""

    def clear(self):
        super().clear()
        self.reached = np.zeros((0, 3), np.int64)

    def integrate(self, points, colors=None, class_ids=None, instance_ids=None, depths=None):
        p = np.asarray(points)
        if len(p):
            inv = np.float64(self.inv_vs) if p.dtype == np.float64 else self.inv_vs
            vk = np.floor(p * inv).astype(np.int64)
            self.reached = np.unique(np.concatenate([self.reached, vk]), axis=0)
        super().integrate(points, colors, class_ids, instance_ids, depths)


def blocks_at(G, B):
    """The sorted block keys a grid of side B holds after the oracle's calls."""
    return np.unique(BS.block_keys_of(G.reached, B), axis=0).reshape(-1, 3)


def unbounded_dump(G, B, K=None):
    """`G`'s state (a MatrixOracle) laid out at block side B: keys, count, sums, argmax, confidence, aux (pairs per
    voxel) and lab_obj / lab_cls / lab_logp [nb, B^3, K] (each voxel's pairs in (object, class) order), the cleared
    state (-1, -1, -inf, ...) in every voxel without observations.  An empty voxel's object id is not part of the
    state: an edit gives it to every voxel of every block (merge_segments(a, -1)), and which empty voxels a grid holds
    depends on B; `same_semantic` does not compare it."""
    K = max(8, G.max_pairs()) if K is None else K
    vk, vals = BS.voxels(G.dump(K), 8, SEM_FIELDS)
    seen = vals["count"] > 0
    return BS.layout(vk[seen], {f: v[seen] for f, v in vals.items()}, B, SEM_CLEARED, blocks=blocks_at(G, B))


def _sorted_voxel_pairs(keys, lists, B, blocks):
    """(count [nb, B^3], obj, cls, logp) of per-voxel pair lists, voxel after voxel in the order of the sorted
    `blocks` and the local index."""
    row = {tuple(k): i for i, k in enumerate(np.asarray(blocks).tolist())}
    count = np.zeros((len(blocks), B ** 3), np.int32)
    if len(keys) == 0:
        return count, np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, f32)
    vk = np.asarray(keys, np.int64).reshape(-1, 3)
    b = np.array([row[tuple(k)] for k in BS.block_keys_of(vk, B).tolist()], np.int64)
    l = BS.local_index_of(vk, B)
    order = np.lexsort((l, b))
    obj, cls, logp = [], [], []
    for i in order.tolist():
        count[b[i], l[i]] = len(lists[i])
        for o, c, lp in lists[i]:
            obj.append(o)
            cls.append(c)
            logp.append(lp)
    return count, np.array(obj, np.int32), np.array(cls, np.int32), np.array(logp, f32)


def unbounded_overflow_pairs(G, B):
    """Each voxel's pairs past its 8 in-voxel slots, in insertion (slot) order, laid out like `export_labels()` in
    the sorted block order of `unbounded_dump(G, B)`: keys [nb,3], count [nb, B^3], obj / cls / logp [total]."""
    blocks = blocks_at(G, B)
    keys, lists = [], []
    l8 = BS.local_coords(8)
    for (b, l), slots in G.slots.items():
        if len(slots) > 8:
            keys.append(G.keys[b] * 8 + l8[l])
            lists.append(slots[8:])
    count, obj, cls, logp = _sorted_voxel_pairs(keys, lists, B, blocks)
    return dict(keys=blocks.astype(np.int32), count=count, obj=obj, cls=cls, logp=logp)


def sorted_labels(parts):
    """`export_labels()` of one grid or of the shards of a map, [(export_blocks()["keys"], export_labels())], in the
    layout of `unbounded_overflow_pairs`: blocks sorted by key, pairs voxel after voxel in that order."""
    keys = np.concatenate([np.asarray(k, np.int64).reshape(-1, 3) for k, _ in parts])
    count = np.concatenate([lab["count"] for _, lab in parts])
    flat = {n: np.concatenate([lab[n] for _, lab in parts]) for n in ("obj", "cls", "logp")}
    order = np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))
    c = count
    start = (np.cumsum(c.reshape(-1)) - c.reshape(-1)).reshape(c.shape)
    cs, ss = c[order].reshape(-1).astype(np.int64), start[order].reshape(-1)
    total = int(cs.sum())
    idx = np.repeat(ss, cs) + (np.arange(total) - np.repeat(np.cumsum(cs) - cs, cs))
    out = dict(keys=keys[order].astype(np.int32), count=c[order])
    out.update({n: a[idx] for n, a in flat.items()})
    return out


def used_chunks(G):
    return sum(SL.chunks_of(len(s)) for s in G.slots.values())


def same_semantic(d, r, exact, where):
    """A grid's sorted dump `d` equals the oracle view `r`: every field bit for bit in every voxel, but the object id
    of voxels without observations; with `exact` False the depth-decayed evidence and the confidence within the
    allowances of tests/test_gpu_semantic_labels.py."""
    assert np.array_equal(d["keys"], r["keys"]), where
    assert np.array_equal(d["hashes"], BS.block_key_hash(d["keys"])), where
    obs = (d["count"] > 0) | (r["count"] > 0)
    for f in SEM_FIELDS:
        if f == "object_id":
            assert np.array_equal(d[f][obs], r[f][obs]), (where, f)
        elif exact or f not in ("lab_logp", "confidence"):
            assert np.array_equal(d[f], r[f]), (where, f)
    if not exact:
        fin = np.isfinite(r["lab_logp"])
        assert np.array_equal(np.isfinite(d["lab_logp"]), fin), where
        assert np.allclose(d["lab_logp"][fin], r["lab_logp"][fin], rtol=1e-6, atol=0), where
        assert np.allclose(d["confidence"], r["confidence"], rtol=2e-6, atol=1e-9), where


def same_pairs(got, ref, exact, where):
    for k in ("keys", "count", "obj", "cls"):
        assert np.array_equal(got[k], ref[k]), (where, k)
    if exact:
        assert np.array_equal(got["logp"], ref["logp"]), where
    else:
        assert np.allclose(got["logp"], ref["logp"], rtol=1e-6, atol=0), where


# ---- semantic scenes -----------------------------------------------------------------------------------------------

# voxels of the chain scenes: a 9 x 9 x 8 cube around the origin (more than one 512-voxel CTA at B = 1 and 2, the
# last one partial) and, at B = 16, two voxels in each 512-voxel slice of a negative and of a positive block, the
# last voxel (local index 4095) included
CUBE = [(x, y, z) for z in range(-4, 4) for y in range(-4, 5) for x in range(-4, 5)]
SLICE_BLOCKS = ((-2, -1, -3), (1, 2, 0))
SLICE_LOCAL = [512 * s + (67 * s + 5) % 512 for s in range(8)] + [512 * s + 511 for s in range(8)]
SLICE_VOXELS = [tuple(int(q) for q in np.array(bk) * 16 + BS.local_coords(16)[l])
                for bk in SLICE_BLOCKS for l in SLICE_LOCAL]
CHAIN_VOXELS = CUBE + SLICE_VOXELS
PAIR_COUNTS = (9, 17, 40)
# a camera 1 m in front of the cube, looking along +z: the cube projects to u in [12, 21], v in [10, 15]
CUBE_T = np.eye(4)
CUBE_T[2, 3] = 1.0
ARGMAX_OBJECTS = (17, 24, 38)   # the argmax object of the voxels of kinds 1, 2, 3 (SL.pairs(n, first)[0][0])


def chain_streams(voxels=CHAIN_VOXELS):
    """Per voxel (index i): n = 9, 17 or 40 distinct pairs seen once each, so every voxel holds a chain.  Kind i % 4:
      0  (-1, 100) three times first, then n - 1 pairs: the argmax is (-1, 100), a voxel the association gives an id
      1-3  SL.pairs(n, first) with first 1, 2, 4: argmax object 17, 24 or 38, class 101 or 102"""
    s = {}
    for i, k in enumerate(voxels):
        n = PAIR_COUNTS[i % 3]
        if i % 4 == 0:
            s[k] = [(-1, 100, 1.0)] * 3 + [(o, c, 1.0) for o, c in SL.pairs(n - 1)]
        else:
            s[k] = [(o, c, 1.0) for o, c in SL.pairs(n, (1, 2, 4)[i % 4 - 1])]
    return s


def _cube_carve():
    img = np.zeros((E.CAM_H, E.CAM_W), f32)
    img[:, :E.CAM_W // 2] = 1.5      # the voxels left of the cube's middle lie 0.5 m in front of it: carved
    return ("carve", dict(cam=SC.cam(CUBE_T), depth_image=img, depth_threshold=0.25))


def _cube_assign():
    """Class 100 everywhere; instance 0 left of the middle (the voxels without an object take 0 at once), 7 right
    of it (they are pending and take a new id)."""
    cls = np.full((E.CAM_H, E.CAM_W), 100, np.int32)
    inst = np.full((E.CAM_H, E.CAM_W), 7, np.int32)
    inst[:, :E.CAM_W // 2] = 0
    return ("assign", dict(cam=SC.cam(CUBE_T), class_image=cls, instance_image=inst, depth_image=None,
                           depth_threshold=0.1, do_carving=False, min_vote_ratio=0.5, min_votes=1))


def chains_everywhere(assign=True):
    """The chain streams, then each edit that releases chains followed by the same call again, which builds them
    again in released chunks: remove_segment, merge_segments (of an object and of -1), remove_low_count_voxels,
    remove_low_confidence_segments, carve and, with `assign`, the association's set_object_id (left out on shards:
    an association spans every rank).  Then clear and the first call once more.  The same scene serves every B."""
    kw = SC.stream(chain_streams())
    edits = [("remove_segment", dict(object_id=ARGMAX_OBJECTS[0])), ("merge_segments", dict(a=5, b=ARGMAX_OBJECTS[1])),
             ("merge_segments", dict(a=6, b=-1)), ("remove_low_count_voxels", dict(min_count=60)),
             ("remove_low_confidence_segments", dict(min_confidence=1)), _cube_carve()]
    if assign:
        edits.append(_cube_assign())
    steps = [("integrate", kw)]
    for e in edits:
        steps += [e, ("integrate", kw)]
    steps += [("clear", {}), ("integrate", kw)]
    return dict(steps=steps, cams=[SC.cam(CUBE_T)])


GROW_BLOCKS = 4   # the growable grids start with 4 blocks of storage and one chunk of 8 pairs


def _far_row(n=200):
    """One pair in one voxel of each of n new blocks at every B (16 voxels apart, far from the cube)."""
    return {(16 * i + 3, 40, -40): [(7, 101, 1.0)] for i in range(-n // 2, n // 2)}


def grow_both():
    """On a grid with 4 blocks of storage and one chunk: a first call that overflows the block pool and, in the same
    call, needs chunks for voxels in more than 4 blocks (so for blocks past the initial storage); a call that only
    adds blocks (one pair per voxel); one that only adds pairs to chained voxels; then edits that release chains in
    grown blocks, each followed by the pair call again, which reuses the released chunks."""
    kw = SC.stream(chain_streams())
    more = SC.stream({k: [(200 + i, 100 + i % 3, 1.0) for i in range(40)] for k in CHAIN_VOXELS})
    steps = [("integrate", kw), ("integrate", SC.stream(_far_row())), ("integrate", more),
             ("remove_segment", dict(object_id=ARGMAX_OBJECTS[0])), ("integrate", more),
             ("remove_low_count_voxels", dict(min_count=60)), ("integrate", more)]
    return dict(steps=steps)


def scene(name):
    if name == "chains":
        return chains_everywhere()
    if name == "chains_no_assign":
        return chains_everywhere(assign=False)
    if name == "grow_both":
        return grow_both()
    if name == "churn":
        return SL.scene_churn(E.cam_poses()[0])
    if name.startswith("pairs"):
        return SL.scene_many_pairs(int(name[5:]))
    raise KeyError(name)


def new_oracle(sc, vs=SC.VS):
    G = MatrixOracle(vs)
    if "depth_threshold" in sc:
        G.set_depth_threshold(sc["depth_threshold"])
    if "depth_decay_rate" in sc:
        G.set_depth_decay_rate(sc["depth_decay_rate"])
    return G


@lru_cache(maxsize=None)
def played(name):
    """(scene, [(instance map or None, oracle after the step)]): the scene played once on the oracle, a copy of the
    oracle kept after every step; the views at any B are built from them."""
    sc = scene(name)
    G = new_oracle(sc)
    out = []
    for op, kw in sc["steps"]:
        m = SC.apply(G, "oracle", op, kw)
        out.append((m, copy.deepcopy(G)))
    return sc, out


# ---- point-average streams with input-order sums --------------------------------------------------------------------

def point_scenes():
    """name -> list of (points, colours) calls at voxel size O.VS: the order-sensitive scenes of
    tests/_grid_order_scenes.py."""
    pts, u8, fl = O.stress_scene()
    return {"stress_calls12": [(pts[i], fl[i]) for i in np.array_split(np.arange(len(pts)), 12)],
            "stress_u8": [(pts, u8)], "float64": [O.float64_scene()], "subnormal": [O.subnormal_scene()]}


def runs_by_block(batches, B, vs=O.VS):
    """Per call: (block keys at side B, local index, points) of every voxel with more than one point in that call."""
    import oracle
    G = oracle.numpy_grid(vs)
    out = []
    for b in batches:
        k, n = np.unique(G.voxel_keys(b[0]), axis=0, return_counts=True)
        k = k[n > 1]
        out.append((BS.block_keys_of(k, B), BS.local_index_of(k, B), n[n > 1]))
    return out


def last_cta_blocks(nb, B):
    """Blocks in the last, partial 512-voxel CTA of a pool of nb blocks of side B (0 when it is full)."""
    per = CTA_VOXELS // B ** 3 if B ** 3 < CTA_VOXELS else 1
    return nb % per
