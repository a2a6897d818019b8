"""CPU: pin the oracle's key / block / hash arithmetic against the reference's own code and
worked examples (SURVEY.md §8c).  No GPU needed."""

import os

import numpy as np
import pytest

import oracle
from oracle import oracle as O
from tests._util import GOLDEN

needs_ref = pytest.mark.skipif(not oracle.have_ref(), reason="compiled reference (oracle/_ref) not built")


def _tsdf_lib():
    return O._tsdf()


# Worked example of pySLAM's cpp/volumetric/voxel_hashing.h:126-142 (B = 4, v in [-9, 9]).
# The comment rows printed in that header are misaligned for negative voxels (they list -8 -> -3);
# the authority is the compiled `floor_div` itself, which test_floor_div_header_table_reference
# checks against the mathematically exact table below.
FLOOR_DIV_TABLE_V = list(range(-9, 10))
FLOOR_DIV_TABLE_B = [-3, -2, -2, -2, -2, -1, -1, -1, -1, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2]
FLOOR_DIV_TABLE_L = [3, 0, 1, 2, 3, 0, 1, 2, 3, 0, 1, 2, 3, 0, 1, 2, 3, 0, 1]


def test_floor_div_header_table_oracle():
    L = _tsdf_lib()
    for v, b, l in zip(FLOOR_DIV_TABLE_V, FLOOR_DIV_TABLE_B, FLOOR_DIV_TABLE_L):
        assert L.tsdf_oracle_floor_div(v, 4) == b
        assert v - b * 4 == l


@needs_ref
def test_floor_div_header_table_reference():
    for v, b in zip(FLOOR_DIV_TABLE_V, FLOOR_DIV_TABLE_B):
        assert oracle.ref_floor_div(v, 4) == b


def test_floor_div_equals_arithmetic_shift_for_block_8():
    """The CUDA kernels use v >> 3; it must equal floor_div(v, 8) over the whole int32 range."""
    L = _tsdf_lib()
    rng = np.random.default_rng(0)
    vals = np.concatenate([rng.integers(-2 ** 31, 2 ** 31, 2000), np.arange(-70, 70),
                           [2 ** 31 - 1, -2 ** 31, -2 ** 31 + 7]]).astype(np.int64)
    for v in vals:
        assert L.tsdf_oracle_floor_div(int(v), 8) == int(v) >> 3
        assert int(v) - (int(v) >> 3) * 8 == int(v) & 7


@needs_ref
def test_known_answer_point_and_hash():
    """SURVEY.md §8c KAT (probe of the compiled reference): (x,y,z)=(-0.0123,0.5,1.234) @5 mm."""
    vk, bk, lk = oracle.ref_keys((-0.0123, 0.5, 1.234), 0.005)
    assert vk.tolist() == [-3, 100, 246]
    assert bk.tolist() == [-1, 12, 30]
    assert lk.tolist() == [5, 4, 6]
    assert oracle.ref_block_key_hash(-1, 12, 30) == 2 ** 64 - 97
    assert O._ref().ref_sizeof_voxel_data() == 28  # voxel_data.h:118-133


def test_oracle_hash_known_answer():
    assert _tsdf_lib().tsdf_oracle_block_key_hash(-1, 12, 30) == 2 ** 64 - 97


def test_oracle_keys_and_hashes_match_the_reference_golden():
    """The oracle's key arithmetic on the float32 points the UNMODIFIED reference grid was fed (tests/golden/
    refgrid_T0.npz, written by tests/golden/make_golden.py from the compiled reference): the same block keys, the
    reference's BlockKeyHash of every block and the reference's point count in every voxel."""
    L = _tsdf_lib()
    g = np.load(os.path.join(GOLDEN, "refgrid_T0.npz"))
    inv = float(np.float32(1.0) / np.float32(float(g["voxel_size"])))
    vk = np.array([[L.tsdf_oracle_voxel_coord(float(c), inv) for c in p] for p in g["points"]], np.int64)
    uniq, inverse = np.unique(vk, axis=0, return_inverse=True)
    ub = np.array([[L.tsdf_oracle_floor_div(int(v), 8) for v in k] for k in uniq], np.int64)
    bk, lk = ub[inverse.reshape(-1)], vk - 8 * ub[inverse.reshape(-1)]
    keys = g["keys"].astype(np.int64)
    mine = np.unique(bk, axis=0)
    assert np.array_equal(mine[np.lexsort(mine.T[::-1])], keys[np.lexsort(keys.T[::-1])])
    for k, h in zip(g["keys"], g["hashes"]):
        assert L.tsdf_oracle_block_key_hash(*map(int, k)) == int(h)
    row = {tuple(k): i for i, k in enumerate(keys.tolist())}
    count = np.zeros_like(g["count"])
    np.add.at(count, (np.array([row[tuple(k)] for k in bk.tolist()]), lk[:, 0] + 8 * lk[:, 1] + 64 * lk[:, 2]), 1)
    assert np.array_equal(count, g["count"])


@needs_ref
def test_oracle_keys_match_reference_on_random_points():
    L = _tsdf_lib()
    rng = np.random.default_rng(42)
    for vs in (0.005, 0.004, 0.01, 0.015, 0.1):
        inv = np.float32(1.0) / np.float32(vs)
        pts = np.concatenate([rng.uniform(-30, 30, (400, 3)), rng.uniform(-0.05, 0.05, (200, 3)),
                              # points sitting (almost) on voxel boundaries
                              np.round(rng.uniform(-3, 3, (300, 3)) / vs) * vs]).astype(np.float32)
        for p in pts:
            vk, bk, lk = oracle.ref_keys(p, vs)
            mine = [L.tsdf_oracle_voxel_coord(float(c), float(inv)) for c in p]
            assert mine == vk.tolist()
            mb = [L.tsdf_oracle_floor_div(v, 8) for v in mine]
            assert mb == bk.tolist()
            assert [v - 8 * b for v, b in zip(mine, mb)] == lk.tolist()
            assert L.tsdf_oracle_block_key_hash(*mb) == oracle.ref_block_key_hash(*mb)


@needs_ref
def test_reference_grid_block_keys_equal_oracle_allocation_lattice():
    """Block-key set of the TSDF oracle's allocation == blocks the UNMODIFIED reference grid creates
    when fed the (p + {-tau,0,tau}^3) lattice of the same samples (valid while 2*tau <= 2 blocks)."""
    from pyslam_b200 import synthetic as S
    cfg = S.CONFIGS["T0"]
    d, c, T = S.render_frame(cfg, 1)
    o = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, unit_resolution=8)  # decision D1
    o.integrate(d, c, cfg.K, T)
    dump = o.dump_blocks()
    # rebuild the lattice points exactly as the oracle does (float64 -> float32)
    stride = 4
    dd = d[::stride, ::stride]
    jj, ii = np.meshgrid(np.arange(dd.shape[1]) * stride, np.arange(dd.shape[0]) * stride)
    ok = (dd > 0) & (dd < np.float32(cfg.depth_trunc))
    z = dd[ok].astype(np.float64)
    x = (jj[ok] - cfg.cx) * z / cfg.fx
    y = (ii[ok] - cfg.cy) * z / cfg.fy
    Twc = S.inv_T(T)
    R = T[:3, :3].T
    t = -np.stack([(R[a, 0] * T[0, 3] + R[a, 1] * T[1, 3]) + R[a, 2] * T[2, 3] for a in range(3)])
    pw = np.stack([((R[a, 0] * x + R[a, 1] * y) + R[a, 2] * z) + t[a] for a in range(3)], axis=1)
    assert np.allclose(pw, (np.c_[x, y, z] @ Twc[:3, :3].T) + Twc[:3, 3], atol=1e-9)
    tau = float(np.float32(cfg.sdf_trunc))
    offs = np.array([[a, b, c_] for a in (-tau, 0, tau) for b in (-tau, 0, tau) for c_ in (-tau, 0, tau)])
    lattice = (pw[:, None, :] + offs[None, :, :]).reshape(-1, 3).astype(np.float32)
    g = oracle.RefGrid(cfg.voxel_size, 8)
    g.integrate(lattice)
    ref = g.dump_blocks()
    ref_set = {tuple(k) for k in ref["keys"]}
    mine_set = {tuple(k) for k in dump["keys"]}
    assert ref_set == mine_set
    ref_hash = {tuple(k): int(h) for k, h in zip(ref["keys"], ref["hashes"])}
    for k, h in zip(dump["keys"], dump["hashes"]):
        assert ref_hash[tuple(k)] == int(h)
