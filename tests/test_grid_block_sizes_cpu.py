"""CPU: the block-size rules the grids use at B in (1, 2, 16), and the re-keying the GPU block-size tests rely on.

Without the compiled reference (oracle/_ref), B != 8 is tied to the reference only by its key rules as written in
terms of B: block key floor_div(v, B) (voxel_hashing.h:139-151), local key v - B b (:154-161) and voxel index
lx + B ly + B^2 lz (voxel_block.h:67-70).  A voxel's state does not depend on B, so the B = 8 goldens pin the values;
the tests below check that laying the golden-stream state out at another B and back is the identity, voxel for
voxel, and that the keys are Python's integer floor division.  With oracle/_ref built, the layouts are also checked
live against `RefGrid(voxel, B)` after every step."""

import os

import numpy as np
import pytest

import oracle
from pyslam_b200 import integrator_semantic
from tests import _block_sizes as BS
from tests import _grid_prep_scenes as E
from tests._util import GOLDEN, ROOT

SIZES = (1, 2, 16)


def _edge_voxel_keys():
    """Keys at +-2^20, around zero and on negative block edges of every B, and the far-key scene's voxels."""
    v = [0, -1, 1, 2 ** 20, -2 ** 20, 2 ** 20 - 1, -2 ** 20 - 1, 2 ** 31 - 1, -2 ** 31]
    for B in BS.RULE_SIZES:
        v += [-B, -B - 1, -B + 1, B - 1, B, 3 * B - 1, -3 * B]
    g = np.array(sorted(set(v)), np.int64)
    k = np.stack(np.meshgrid(g, g[::3], g[::5], indexing="ij"), -1).reshape(-1, 3)
    far = np.floor(E.far_points() * (np.float32(1) / np.float32(E.VS_EXACT))).astype(np.int64)
    return np.concatenate([k, far])


@pytest.mark.parametrize("B", BS.RULE_SIZES)
def test_block_and_local_keys_are_integer_floor_division(B):
    vk = _edge_voxel_keys()
    bk = BS.block_keys_of(vk, B)
    lx = BS.local_index_of(vk, B)
    for v, b, l in zip(vk.tolist(), bk.tolist(), lx.tolist()):
        want_b = [BS.floor_div(x, B) for x in v]
        loc = [x - B * y for x, y in zip(v, want_b)]
        assert b == want_b and all(0 <= q < B for q in loc)
        assert l == loc[0] + B * loc[1] + B * B * loc[2]
    # the shift / mask of the kernels, on int32
    v32 = vk[(vk >= -2 ** 31) & (vk < 2 ** 31)].astype(np.int32)
    s = B.bit_length() - 1
    assert np.array_equal((v32 >> s).astype(np.int64), np.floor_divide(v32.astype(np.int64), B))
    assert np.array_equal((v32 & (B - 1)).astype(np.int64), v32.astype(np.int64) - B * np.floor_divide(v32, B))


@pytest.mark.parametrize("B", SIZES)
def test_hashes_are_block_key_hash(B):
    k = np.unique(BS.block_keys_of(_edge_voxel_keys(), B), axis=0)
    h = BS.block_key_hash(k)
    for kk, hh in zip(k.tolist()[:200], h.tolist()[:200]):
        m = (1 << 64) - 1
        x, y, z = (q & m for q in kk)
        assert hh == (x ^ ((y << 1) & m) ^ ((z << 2) & m))


@pytest.mark.parametrize("B", SIZES)
def test_point_oracle_layouts_hold_the_b8_state_voxel_for_voxel(B):
    """The exact-sum scene through `oracle.numpy_grid`: its dump at B, re-keyed by voxel, is its dump at 8."""
    G = oracle.numpy_grid(E.VS_EXACT)
    for _, p, c in E.exact_batches():
        G.integrate(p, c)
        d8, dB = BS.grid_dump(G, 8), BS.grid_dump(G, B)
        r8 = G.dump()
        for f in ("keys", "count", "pos_sum", "col_sum"):
            assert np.array_equal(d8[f], r8[f]), f
        k8, v8 = BS.voxels(d8, 8, ("count", "pos_sum", "col_sum"))
        kB, vB = BS.voxels(dB, B, ("count", "pos_sum", "col_sum"))
        seen8 = v8["count"] > 0
        seenB = vB["count"] > 0
        assert np.array_equal(k8[seen8], kB[seenB])
        for f in v8:
            assert np.array_equal(v8[f][seen8], vB[f][seenB]), f
        assert np.array_equal(dB["keys"], np.unique(BS.block_keys_of(G.keys, B), axis=0).astype(np.int32))


@pytest.mark.parametrize("B", SIZES)
def test_golden_streams_relaid_at_b_and_back(B):
    """The point-average golden stream (refgrid_T0: the oracle's B = 8 dump equals the golden dump) and the first
    semantic golden frame through the voting oracle: each state laid out at B and re-keyed back is the same state,
    voxel for voxel, and its blocks are floor_div of the voxels' keys."""
    z = np.load(os.path.join(GOLDEN, "refgrid_T0.npz"))
    G = oracle.numpy_grid(float(z["voxel_size"]))
    G.integrate(z["points"], z["colors"])
    d8 = G.dump()
    assert np.array_equal(d8["keys"], z["keys"]) and np.array_equal(d8["count"], z["count"])
    states = [(d8, ("count", "pos_sum", "col_sum"), dict(count=0, pos_sum=0.0, col_sum=0.0))]
    s = np.load(os.path.join(GOLDEN, "semantic_T0.npz"))
    S = oracle.numpy_semantic_grid(float(s["voxel_size"]), "voting")
    S.integrate(s["vote_points_0"], s["vote_colors_0"], s["vote_cls_0"], s["vote_inst_0"], s["vote_depths_0"])
    states.append((S.dump(), ("count", "pos_sum", "col_sum", "object_id", "class_id", "aux"),
                   dict(count=0, pos_sum=0.0, col_sum=0.0, object_id=-1, class_id=-1, aux=0)))
    for d, fields, cleared in states:
        vk, vals = BS.voxels(d, 8, fields)
        seen = vals["count"] > 0
        dB = BS.layout(vk[seen], {f: v[seen] for f, v in vals.items()}, B, cleared)
        assert np.array_equal(dB["keys"], np.unique(BS.block_keys_of(vk[seen], B), axis=0).astype(np.int32))
        kB, back = BS.voxels(dB, B, fields)
        hit = back["count"] > 0
        assert np.array_equal(kB[hit], vk[seen])
        for f in fields:
            assert np.array_equal(back[f][hit], vals[f][seen]), f
            assert np.all(back[f][~hit] == cleared[f]), f


def test_plugin_capacity_defaults_keep_the_voxel_budget():
    p = dict(integrator_semantic.DEFAULT_PARAMETERS)
    base = p["kVolumetricIntegrationB200CapacityBlocks"]
    for B in BS.BLOCK_SIZES:
        q = dict(p, kVolumetricIntegrationBlockSize=B, kVolumetricIntegrationB200MaxCapacityBlocks=1 << 16)
        a = integrator_semantic._grid_args(q)
        assert a["block_size"] == B
        assert a["capacity_blocks"] == -(-base * 512 // B ** 3)
        assert a["max_capacity_blocks"] == -(-(1 << 16) * 512 // B ** 3)
        given = integrator_semantic._grid_args(q, {"kVolumetricIntegrationB200CapacityBlocks",
                                                   "kVolumetricIntegrationB200MaxCapacityBlocks"})
        assert given["capacity_blocks"] == base and given["max_capacity_blocks"] == 1 << 16
    assert integrator_semantic._grid_args(dict(p, kVolumetricIntegrationBlockSize=8))["capacity_blocks"] == base
    assert integrator_semantic._grid_args(p)["max_capacity_blocks"] is None


_HAVE_REF = os.path.isdir(os.path.join(ROOT, "oracle", "_ref")) and any(
    f.endswith(".so") for f in os.listdir(os.path.join(ROOT, "oracle", "_ref")))


@pytest.mark.skipif(not _HAVE_REF, reason="the compiled reference (oracle/_ref) is not built")
@pytest.mark.parametrize("B", SIZES)
def test_point_layout_equals_the_reference_live(B):
    ref = oracle.RefGrid(E.VS_EXACT, B)
    G = oracle.numpy_grid(E.VS_EXACT)
    for _, p, c in E.exact_batches():
        ref.integrate(p, c)
        G.integrate(p, c)
        d = ref.dump_blocks()
        k = np.asarray(d["keys"])
        o = np.lexsort((k[:, 2], k[:, 1], k[:, 0]))
        mine = BS.grid_dump(G, B)
        assert np.array_equal(k[o], mine["keys"])
        assert np.array_equal(np.asarray(d["count"])[o], mine["count"])
