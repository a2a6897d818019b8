"""GPU: the fused allocation's group unit set (allocate_group_kernel -> allocate_group_expand_kernel) where it runs
out of entries, against the CPU twin bit for bit.  Units that find no entry touch their blocks directly; the set's size
is forced down with B2V_GROUP_UNIT_SET, and one scene's group has more units than the default set holds.  Per group:
the union of touched blocks, the last frame's touched count and the group's new blocks; over the run: the (block,
frame) update count and the final volume (keys, hashes, all five planes)."""

import numpy as np
import pytest

import oracle
from pyslam_b200 import B200TsdfVolume
from pyslam_b200 import synthetic as S
from pyslam_b200.sharding import owner_of
from tests._util import sort_dump, sorted_keys

pytestmark = pytest.mark.gpu

SMALL_SET = 16   # entries per group buffer: every group below has more units than that


def _same(a, b):
    a, b = sort_dump(a), sort_dump(b)
    for name in ("keys", "hashes", "vox"):
        assert np.array_equal(a[name], b[name]), name


_frames_cache = {}


def _frames(name, n):
    if name not in _frames_cache:
        cfg = S.CONFIGS[name]
        fr = [S.render_frame(cfg, i) for i in range(cfg.n_frames)]
        _frames_cache[name] = tuple(np.stack([f[k] for f in fr]) for k in range(3))
    return tuple(a[:n] for a in _frames_cache[name])


def _twin_groups(vs, tau, trunc, unit, D, C, K, T, group):
    """Per group of `group` frames: (sorted union of the frames' touched blocks, last frame's touched count, blocks new
    in the group); the total of touched counts; the final dump."""
    tw = oracle.TsdfOracle(vs, tau, trunc, unit_resolution=unit)
    groups, seen, updates = [], set(), 0
    for g0 in range(0, len(D), group):
        union = set()
        for i in range(g0, min(g0 + group, len(D))):
            n = tw.integrate(D[i], C[i], K, T[i], nthreads=8)
            updates += n
            union |= {tuple(k) for k in tw.last_touched()}
        keys = sorted_keys(np.array(sorted(union), np.int32).reshape(-1, 3))
        groups.append((keys, n, len(union - seen)))
        seen |= union
    return groups, updates, tw.dump_blocks()


def _units(keys, unit):
    return len(np.unique(np.asarray(keys) >> (1 if unit == 16 else 0), axis=0))


def _run_groups(vol, D, C, K, T, group, want_groups, owner=None):
    """One integrate_batch call per group: each group's union, last touched count and new blocks."""
    vol.set_group_size(group)
    for gi, g0 in enumerate(range(0, len(D), group)):
        sl = slice(g0, g0 + group)
        vol.integrate_batch(D[sl], C[sl], K, T[sl])
        keys, last_n, new = want_groups[gi]
        if owner is not None:  # (rank, world): this rank's share of the twin's union
            keys = keys[owner_of(keys, owner[1]) == owner[0]]
        got = sorted_keys(vol.last_touched_keys())
        assert np.array_equal(got, keys), gi
        if owner is None:
            assert vol.last_frame_stats() == (last_n, new), gi


@pytest.mark.parametrize("unit", [16, 8])
@pytest.mark.parametrize("group", [2, 17, 32])
def test_unit_set_overflow_equals_the_twin(group, unit, monkeypatch):
    monkeypatch.setenv("B2V_GROUP_UNIT_SET", str(SMALL_SET))
    cfg = S.CONFIGS["C1"]
    D, C, T = _frames("C1", 68)
    groups, updates, ref = _twin_groups(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, unit, D, C, cfg.K, T, group)
    assert min(_units(g[0], unit) for g in groups) > SMALL_SET
    vol = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 16,
                         volume_unit_resolution=unit)
    _run_groups(vol, D, C, cfg.K, T, group, groups)
    assert vol.counters()[0] == updates
    _same(vol.dump_blocks(), ref)
    vol.close()


@pytest.mark.parametrize("world", [2, 3])
def test_unit_set_overflow_in_hash_shards(world, monkeypatch):
    monkeypatch.setenv("B2V_GROUP_UNIT_SET", str(SMALL_SET))
    cfg = S.CONFIGS["C1"]
    D, C, T = _frames("C1", 64)
    groups, _, ref = _twin_groups(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, 16, D, C, cfg.K, T, 32)
    parts = []
    for r in range(world):
        vol = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 16,
                             shard_rank=r, shard_count=world)
        _run_groups(vol, D, C, cfg.K, T, 32, groups, owner=(r, world))
        parts.append(vol.dump_blocks())
        vol.close()
    _same({k: np.concatenate([p[k] for p in parts]) for k in ("keys", "hashes", "vox")}, ref)


def test_unit_set_overflow_in_a_volume_that_grows_mid_batch(monkeypatch):
    """One call of 100 frames in groups of 32 into a pool of 64 blocks: groups are skipped, the pool grows and they
    are replayed, while their units take the overflow path."""
    monkeypatch.setenv("B2V_GROUP_UNIT_SET", str(SMALL_SET))
    cfg = S.CONFIGS["C1"]
    D, C, T = _frames("C1", 100)
    groups, updates, ref = _twin_groups(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, 16, D, C, cfg.K, T, 32)
    vol = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=64,
                         max_capacity_blocks=1 << 16)
    vol.set_group_size(32)
    vol.integrate_batch(D, C, cfg.K, T)
    assert vol.capacity()[1] >= 1
    assert np.array_equal(sorted_keys(vol.last_touched_keys()), groups[-1][0])
    assert vol.last_frame_stats() == groups[-1][1:]
    assert vol.counters()[0] == updates
    _same(vol.dump_blocks(), ref)
    vol.close()


def _scattered_frames(n, H=120, W=160, seed=7):
    """Frames whose depth samples scatter over far-apart 8^3 blocks: random depths in [0.5, 6) m, cameras 50 m apart
    (no two frames share a block), 2 % invalid pixels."""
    rng = np.random.default_rng(seed)
    D = rng.uniform(0.5, 6.0, (n, H, W)).astype(np.float32)
    D[rng.random((n, H, W)) < 0.02] = 0.0
    C = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    T = np.tile(np.eye(4), (n, 1, 1))
    T[:, 0, 3] = -50.0 * np.arange(n)   # Tcw: camera i at x = 50 i
    K = (131.25, 131.25, 79.5, 59.5)
    return D, C, K, T


def test_group_union_beyond_the_default_unit_set():
    """One 32-frame group of decision-D1 units (the block is the unit) whose union has more units than the default
    set's 2^16 entries."""
    vs, tau, trunc = 0.005, 0.01, 8.0
    D, C, K, T = _scattered_frames(32)
    groups, updates, ref = _twin_groups(vs, tau, trunc, 8, D, C, K, T, 32)
    assert _units(groups[0][0], 8) > 1 << 16
    vol = B200TsdfVolume(vs, tau, trunc, capacity_blocks=1 << 18, volume_unit_resolution=8)
    _run_groups(vol, D, C, K, T, 32, groups)
    assert vol.counters()[0] == updates
    _same(vol.dump_blocks(), ref)
    vol.close()
