"""CPU: the scenes of tests/_grid_matrix.py reach the cases tests/test_gpu_grid_matrix.py is named for, shown on the
oracles alone, and the oracle views at B = 8 are the oracles' own dumps."""

import numpy as np
import pytest

import oracle
from tests import _block_sizes as BS
from tests import _grid_matrix as M
from tests import _grid_order_scenes as O
from tests import _semantic_labels as SL
from tests import _semantic_scenes as SC


def _chained(G):
    """Voxel keys of the voxels holding more than 8 pairs."""
    l8 = BS.local_coords(8)
    k = [G.keys[b] * 8 + l8[l] for (b, l), s in G.slots.items() if len(s) > 8]
    return np.array(k, np.int64).reshape(-1, 3)


def test_chain_voxels_hold_chains_after_the_first_call():
    _, snaps = M.played("chains")
    G = snaps[0][1]
    have = set(map(tuple, _chained(G).tolist()))
    assert set(M.CHAIN_VOXELS) <= have
    n = {len(G.slots[k]) for k in G.slots}
    assert {9, 17, 40} <= n


def test_chains_in_every_slice_of_a_block_16():
    """At B = 16: chained voxels at local indices in each of the 8 slices of 512 of a negative and a positive block,
    index 4095 included (the per-voxel passes run 8 CTAs per block)."""
    _, snaps = M.played("chains")
    vk = _chained(snaps[0][1])
    bk, l = BS.block_keys_of(vk, 16), BS.local_index_of(vk, 16)
    for block in M.SLICE_BLOCKS:
        mine = np.all(bk == block, axis=1)
        assert set((l[mine] // 512).tolist()) == set(range(8)), block
        assert 4095 in set(l[mine].tolist())
    assert any(all(q < 0 for q in b) for b in M.SLICE_BLOCKS) and any(all(q >= 0 for q in b) for b in M.SLICE_BLOCKS)


@pytest.mark.parametrize("B", (1, 2))
def test_chains_in_every_block_and_a_partial_last_cta(B):
    """At B = 1 and 2 a 512-voxel CTA spans 512 / B^3 blocks: every block holds a chained voxel, so whatever pool
    order the blocks take, the first, middle and last block of every CTA hold chains; the pool needs more than one
    CTA and its last one is partial; block keys of both signs."""
    _, snaps = M.played("chains")
    G = snaps[0][1]
    blocks = M.blocks_at(G, B)
    chained = np.unique(BS.block_keys_of(_chained(G), B), axis=0)
    assert np.array_equal(blocks, chained)
    nv = len(blocks) * B ** 3
    assert nv > M.CTA_VOXELS and M.last_cta_blocks(len(blocks), B) > 0
    assert (blocks < 0).all(axis=1).any() and (blocks >= 0).all(axis=1).any()


@pytest.mark.parametrize("name", ["chains", "chains_no_assign", "grow_both"])
def test_every_edit_releases_chunks_that_the_next_call_takes_again(name):
    sc, snaps = M.played(name)
    used = [M.used_chunks(G) for _, G in snaps]
    ops = [op for op, _ in sc["steps"]]
    edits = [i for i, op in enumerate(ops) if op not in ("integrate", "clear")]
    assert len(edits) >= (2 if name == "grow_both" else 6)
    for i in edits:
        assert used[i] < used[i - 1], (name, i, ops[i])
        assert ops[i + 1] == "integrate" and used[i + 1] > used[i], (name, i)
    if name.startswith("chains"):
        assert {"remove_segment", "merge_segments", "remove_low_count_voxels", "remove_low_confidence_segments",
                "carve"} <= set(ops)
        assert ("merge_segments", dict(a=6, b=-1)) in sc["steps"]
        c = ops.index("clear")
        assert used[c] == 0 and used[c + 1] == used[0]


def test_the_association_gives_ids_to_chained_voxels():
    """The association step sets object ids on both of its paths (instance 0 at once, a new id for pending voxels)
    and releases chains doing so."""
    sc, snaps = M.played("chains")
    i = [op for op, _ in sc["steps"]].index("assign")
    m = snaps[i][0]
    assert m[0] == 0 and m[7] >= 1
    before, after = snaps[i - 1][1], snaps[i][1]
    assert M.used_chunks(after) < M.used_chunks(before)
    assert (after.obj == 0).sum() > (before.obj == 0).sum() and (after.obj == m[7]).sum() > 0


@pytest.mark.parametrize("B", (1, 2, 8, 16))
def test_grow_both_overflows_blocks_and_chunks_in_one_call(B):
    """First call: more than 4 blocks, and more than 4 blocks hold chained voxels, so some chained voxel lies past the
    initial 4-block storage whatever the pool order, and its chunks are needed in the call that grows the pool.  Then
    a call that adds blocks and no chunk, and one that adds more than twice the chunks in use and no block."""
    _, snaps = M.played("grow_both")
    G0, G1, G2 = (snaps[i][1] for i in range(3))
    assert len(M.blocks_at(G0, B)) > M.GROW_BLOCKS
    assert len(np.unique(BS.block_keys_of(_chained(G0), B), axis=0)) > M.GROW_BLOCKS
    assert M.used_chunks(G0) > 1
    assert len(M.blocks_at(G1, B)) > len(M.blocks_at(G0, B)) and M.used_chunks(G1) == M.used_chunks(G0)
    assert np.array_equal(M.blocks_at(G2, B), M.blocks_at(G1, B)) and M.used_chunks(G2) > 2 * M.used_chunks(G1)
    if B >= 8:     # a row of far blocks: more blocks than a first growth from 4 maps at B = 8 and 16
        assert len(M.blocks_at(G1, B)) > 2 * len(M.blocks_at(G0, B))


def test_state_file_scene_holds_chains():
    """The state-file test saves the first call of the chain scene at B = 16 and continues with its next steps."""
    sc, snaps = M.played("chains_no_assign")
    assert M.used_chunks(snaps[0][1]) > 0 and len(M.blocks_at(snaps[0][1], 16)) > M.GROW_BLOCKS
    assert [op for op, _ in sc["steps"][1:7]] == ["remove_segment", "integrate", "merge_segments", "integrate",
                                                 "merge_segments", "integrate"]


@pytest.mark.parametrize("name", ["chains", "grow_both", "pairs40"])
def test_unbounded_dump_at_8_is_the_oracle_dump(name):
    _, snaps = M.played(name)
    for _, G in snaps:
        K = max(8, G.max_pairs())
        d, r = M.unbounded_dump(G, 8, K), G.dump(K)
        assert np.array_equal(d["keys"], r["keys"])
        seen = r["count"] > 0
        for f in M.SEM_FIELDS:
            a, b = np.asarray(d[f]), np.asarray(r[f])
            if f == "object_id":
                assert np.array_equal(a[seen], b[seen])
            else:
                assert np.array_equal(a, b), f


@pytest.mark.parametrize("B", (1, 2, 8, 16))
def test_overflow_pairs_are_the_pairs_past_slot_8_in_slot_order(B):
    _, snaps = M.played("chains")
    G = snaps[2][1]
    p = M.unbounded_overflow_pairs(G, B)
    d = M.unbounded_dump(G, B)
    assert np.array_equal(p["keys"], d["keys"])
    assert np.array_equal(p["count"], np.maximum(d["aux"] - 8, 0))
    assert len(p["obj"]) == sum(max(0, len(s) - 8) for s in G.slots.values())
    # the first chained voxel of the sorted layout: its pairs 8.. in insertion order
    f = int(np.argmax(p["count"].reshape(-1) > 0))
    first = p["keys"][f // B ** 3].astype(np.int64) * B + BS.local_coords(B)[f % B ** 3]
    b8, l8 = BS.block_keys_of(first[None], 8)[0], BS.local_index_of(first[None], 8)[0]
    slots = G.slots[(G.block_of[tuple(b8.tolist())], int(l8))]
    n = len(slots) - 8
    assert [tuple(x) for x in zip(p["obj"][:n].tolist(), p["cls"][:n].tolist())] == [(o, c) for o, c, _ in slots[8:]]
    # insertion order is not the (object, class) order the dump shows
    assert any([q[:2] for q in s[8:]] != sorted(q[:2] for q in s[8:]) for s in G.slots.values())


def test_sorted_labels_reorders_a_pool_order_export():
    """`sorted_labels` on an export in a shuffled block order (as a pool holds them), split in shards, gives the
    sorted layout back."""
    _, snaps = M.played("chains")
    G = snaps[0][1]
    B = 2
    p = M.unbounded_overflow_pairs(G, B)
    rng = np.random.default_rng(0)
    perm = rng.permutation(len(p["keys"]))
    start = np.cumsum(p["count"].reshape(-1)) - p["count"].reshape(-1)
    st = start.reshape(p["count"].shape)[perm].reshape(-1)
    cn = p["count"][perm].reshape(-1)
    idx = np.concatenate([np.arange(s, s + c) for s, c in zip(st, cn)])
    parts = []
    for sl in np.array_split(np.arange(len(perm)), 3):
        lo = int(p["count"][perm[:sl[0]]].sum()) if len(sl) else 0
        hi = lo + int(p["count"][perm[sl]].sum())
        parts.append((p["keys"][perm[sl]], dict(count=p["count"][perm[sl]], obj=p["obj"][idx[lo:hi]],
                                                cls=p["cls"][idx[lo:hi]], logp=p["logp"][idx[lo:hi]])))
    got = M.sorted_labels(parts)
    for k in p:
        assert np.array_equal(got[k], p[k]), k


def test_many_pair_and_churn_scenes_hold_chains():
    for name in ("pairs9", "pairs17", "pairs40", "churn"):
        _, snaps = M.played(name)
        assert max(G.max_pairs() for _, G in snaps) > 8, name


# ---- point-average streams -----------------------------------------------------------------------------------------

def test_point_view_at_8_is_the_oracle_dump():
    for name, batches in M.point_scenes().items():
        G = O.numpy_grid_of(batches)
        d, r = BS.grid_dump(G, 8), G.dump()
        for f in ("keys", "count", "pos_sum", "col_sum"):
            assert np.array_equal(d[f], r[f]), (name, f)


def _streams():
    out = dict(M.point_scenes())
    out["frames"] = list(O.frame_points())
    return out


@pytest.mark.parametrize("name", ["stress_calls12", "stress_u8", "float64", "subnormal", "frames"])
def test_input_order_runs_at_high_local_indices_and_in_the_last_cta(name):
    """Runs longer than 1 (an order to keep) in voxels at local index >= 512 of B = 16 blocks (CTAs 2..8 of a
    block), and at B = 1 and 2 in more blocks than can stay out of the last, partial CTA of the pool, whatever its
    order."""
    batches = _streams()[name]
    runs = M.runs_by_block(batches, 16)
    assert any((l >= 512).any() for _, l, _ in runs)
    assert max(int(n.max()) for _, _, n in runs) > 1
    G = O.numpy_grid_of(batches)
    for B in (1, 2):
        blocks = np.unique(BS.block_keys_of(G.keys, B), axis=0)
        with_runs = np.unique(np.concatenate([b for b, _, _ in M.runs_by_block(batches, B)]), axis=0)
        quiet = len(blocks) - len(with_runs)
        assert quiet < M.last_cta_blocks(len(blocks), B), (name, B, quiet, len(blocks))


def test_exact_batches_serve_the_mode_switch():
    """The switched-mode test's scenes are exact in any order: both modes must give numpy_grid."""
    from tests import _grid_prep_scenes as E
    G = oracle.numpy_grid(E.VS_EXACT)
    for _, p, c in E.exact_batches():
        G.integrate(p, c)
    R = O.reversed_dump([(p, c) for _, p, c in E.exact_batches()], E.VS_EXACT)
    for f in ("count", "pos", "col"):
        assert np.array_equal(getattr(G, f), getattr(R, f)), f
    assert SC.VS == E.VS_EXACT and SL.chunks_of(9) == 1
