"""Scenes of the point-average grid's input-order sums (VoxelBlockGrid(input_order_sums=True)), where the order of a
voxel's float32 adds decides its bits: non-dyadic coordinates at the reference's voxel size 0.015, runs of thousands
of points, float64 points, sub-normal addends, and real frames.  `oracle.numpy_grid` sums in input order
(np.add.at), so it is the truth for these scenes; `reversed_dump` sums the same points in the opposite order, to show
that an equality with it would not hold by chance."""

from functools import lru_cache

import numpy as np

import oracle
from pyslam_b200 import synthetic as S
from tests import _grid_prep_scenes as E

f32 = np.float32
VS = 0.015                 # the reference's default voxel size: float32(1 / 0.015) rounds, coordinates are not dyadic
N_FRAMES = 10              # real frames per stream
FRAME_CFG = "C2"


def _voxel_points(rng, keys, which, dtype=f32):
    """One point per entry of `which` inside voxel keys[which], at least 5% of a voxel from every face."""
    u = rng.uniform(0.05, 0.95, (len(which), 3))
    return ((keys[which] + u) * VS).astype(dtype)


def stress_scene(seed=11, n=120_000, voxels=300):
    """(points float32 [n,3], uint8 colours, float colours): n points in `voxels` voxels around the origin, with
    Zipf-like voxel weights (the busiest voxel takes about 19 000 points) and the voxels' points interleaved in
    random input order."""
    rng = np.random.default_rng(seed)
    keys = np.unique(rng.integers(-24, 24, (voxels * 2, 3)), axis=0)[:voxels]
    rng.shuffle(keys)
    w = 1.0 / np.arange(1, len(keys) + 1)
    which = rng.choice(len(keys), n, p=w / w.sum())
    pts = _voxel_points(rng, keys, which)
    return pts, rng.integers(0, 256, (n, 3), dtype=np.uint8), rng.random((n, 3)).astype(f32)


def float64_scene(seed=12, n=100_000, voxels=200):
    """(points float64, float colours): as stress_scene, in float64 (keys from the float64 coordinates)."""
    rng = np.random.default_rng(seed)
    keys = np.unique(rng.integers(-30, 30, (voxels * 2, 3)), axis=0)[:voxels]
    w = 1.0 / np.sqrt(np.arange(1, len(keys) + 1))
    which = rng.choice(len(keys), n, p=w / w.sum())
    return _voxel_points(rng, keys, which, np.float64), rng.random((n, 3)).astype(f32)


def subnormal_scene(seed=13, n=40_000):
    """(points, float colours) in the voxels around the origin, mixing sub-normal float32 coordinates and colours
    (|x| < 2^-126) with normal ones in the same voxels, so a flush to zero or another order changes the sums.  An
    eighth of the points lies in voxels x = 0 or -1 of a far row (y, z about 0.5) with x below 1e-41 only, so
    those voxels' x sums stay sub-normal."""
    rng = np.random.default_rng(seed)
    tiny = rng.uniform(1e-45, 1e-38, (n, 3)) * rng.choice([-1.0, 1.0], (n, 3))
    normal = rng.uniform(-0.0149, 0.0149, (n, 3))
    pts = np.where(rng.random((n, 3)) < 0.6, tiny, normal)
    row = rng.random(n) < 0.125
    pts[row, 0] = tiny[row, 0] * 1e-4
    pts[row, 1:] = 0.5 + normal[row, 1:]
    pts = pts.astype(f32)
    cols = np.where(rng.random((n, 3)) < 0.5, rng.uniform(1e-45, 1e-38, (n, 3)), rng.random((n, 3))).astype(f32)
    return pts, cols


def is_subnormal(a):
    a = np.abs(np.asarray(a, f32))
    return (a > 0) & (a < np.finfo(f32).tiny)


@lru_cache(maxsize=1)
def frames():
    """N_FRAMES frames of the C2 sequence: [(depth, rgb, Twc)]."""
    cfg = S.CONFIGS[FRAME_CFG]
    out = []
    for i in range(N_FRAMES):
        d, c, Tcw = S.render_frame(cfg, i)
        out.append((d, c, S.inv_T(Tcw)))
    return tuple(out)


def frame_K():
    return S.CONFIGS[FRAME_CFG].K


def frame_max_depth():
    return float(S.CONFIGS[FRAME_CFG].depth_trunc)


@lru_cache(maxsize=1)
def frame_points():
    """The front-end points of frames(): [(points float32, colours float32)] in row-major pixel order."""
    return tuple(E.rgbd_points(d, c, frame_K(), Twc, max_depth=frame_max_depth()) for d, c, Twc in frames())


def numpy_grid_of(batches, vs=VS):
    G = oracle.numpy_grid(vs)
    for b in batches:
        G.integrate(*b)
    return G


def longest_runs(batches, vs=VS):
    """(longest, p99) of the points per voxel and call: the run one thread of the input-order pass walks."""
    G = oracle.numpy_grid(vs)
    runs = []
    for b in batches:
        runs.append(np.unique(G.voxel_keys(b[0]), axis=0, return_counts=True)[1])
    r = np.concatenate(runs)
    return int(r.max()), float(np.percentile(r, 99))


def reversed_dump(batches, vs=VS):
    """numpy_grid's state when each call's points are summed in reverse order."""
    return numpy_grid_of([tuple(None if a is None else a[::-1] for a in b) for b in batches], vs)
