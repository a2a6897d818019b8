"""Scenes of the bench's configurations C3 (Replica shape), C4 (ScanNet shape) and C5 (KITTI shape) for the parity
tests of tests/test_gpu_bench_configs.py and tests/test_bench_configs_cpu.py.

Bench frames come from `bench.load_frames(name, 300, 0, 1)`: the 300 frames `bench.py` integrates, spread over the whole
sequence (C5: every 15th frame of the 4541-frame street, the camera up to 1973 m along z), cached in the temp
directory.  Runs of consecutive frames are rendered directly; C5's far end (frames 4488..4503, z ~ 1975 m) is where
float32 voxel centres and pose translations are ~2000 m and one float32 ulp is 1.2e-4 m, so `p = E h + t` cancels
most of its digits and the order of float operations decides more results than near the origin."""

import os

import numpy as np

import oracle
from pyslam_b200 import synthetic as S
from tests._util import sort_dump

NT = max(1, min(len(os.sched_getaffinity(0)), 64))   # host threads for the CPU oracles
BENCH_FRAMES = 300
PASSES = 2                                           # every observed voxel reaches weight >= 2

# runs of consecutive frames: (config, first frame, frames)
FAR_C5 = ("C5", 4488, 16)
RUN_C4 = ("C4", 600, 16)

_frames = {}


def bench_frames(name):
    """(cfg, depth [300,H,W], colour [300,H,W,3], Tcw [300,4,4]): the frames bench.py integrates."""
    if name not in _frames:
        import bench
        _frames[name] = bench.load_frames(name, BENCH_FRAMES, 0, 1)
    return _frames[name]


def release_frames(name=None):
    """drop the cached bench frames of one config (all if None)"""
    if name is None:
        _frames.clear()
    else:
        _frames.pop(name, None)


def consecutive(name, start, n):
    """(cfg, depth, colour, Tcw) of frames start .. start + n - 1, stacked."""
    cfg = S.CONFIGS[name]
    fr = [S.render_frame(cfg, i) for i in range(start, start + n)]
    return (cfg,) + tuple(np.stack([f[k] for f in fr]) for k in range(3))


def twin(cfg, D, C, T, passes=1):
    """The CPU twin (oracle/tsdf_oracle.c) after `passes` passes over the frames."""
    tw = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    for _ in range(passes):
        for i in range(len(D)):
            tw.integrate(D[i], C[i], cfg.K, T[i], nthreads=NT)
    return tw


def open3d_order(cfg, D, C, T):
    """The Open3D-order restatement (oracle/open3d_order.c) over the frames, with each frame's touched units."""
    o3 = oracle.Open3DOrderVolume(cfg.voxel_size, cfg.sdf_trunc, 16, 4)
    units = []
    for i in range(len(D)):
        o3.integrate(D[i], C[i], cfg.K, T[i], cfg.depth_trunc, nthreads=NT)
        units.append(o3.last_touched_units())
    return o3, units


def unit_blocks(units):
    """The 8^3 blocks of Open3D's 16^3 units, sorted."""
    sub = np.stack(np.meshgrid(*[np.arange(2)] * 3, indexing="ij"), -1).reshape(-1, 3)
    k = (np.asarray(units)[:, None, :] * 2 + sub[None]).reshape(-1, 3)
    return k[np.lexsort(k.T[::-1])].astype(np.int32)


def canon(m):
    """canonical_mesh of a TriangleMesh or of an oracle mesh dict"""
    if isinstance(m, dict):
        return oracle.canonical_mesh(m["vertices"], m["colors"], m["edges"], m["triangles"])
    return oracle.canonical_mesh(m.vertices, m.vertex_colors, m.edge_ids, m.triangles)


def same_topology_and_vertices(ca, cb):
    """Canonical meshes with the same edges, triangles and float64 vertices, bit for bit."""
    assert len(ca["triangles"]) == len(cb["triangles"])
    for k in ("edges", "triangles"):
        assert np.array_equal(ca[k], cb[k]), k
    assert np.array_equal(ca["vertices"].view(np.uint64), cb["vertices"].view(np.uint64)), "vertices"


def equal_to_open3d_order(dump, o3dump, colour_tol=1e-3):
    """A float32-colour dump against the Open3D-order dump: keys, weights and tsdf exact, colour within colour_tol on
    the 0..255 scale.  Returns (observed voxels, max weight)."""
    a, b = sort_dump(dump), sort_dump(o3dump)
    assert np.array_equal(a["keys"], b["keys"])
    assert np.array_equal(a["vox"][:, 1].astype(np.float64), b["vox"][:, 1]), "weights"
    assert np.array_equal(a["vox"][:, 0].astype(np.float64), b["vox"][:, 0]), "tsdf"
    assert np.abs(a["vox"][:, 2:].astype(np.float64) - b["vox"][:, 2:]).max() < colour_tol
    w = b["vox"][:, 1]
    return int((w > 0).sum()), float(w.max())


def centre_ulp(keys, voxel_size):
    """The largest float32 ulp of a voxel-centre coordinate in blocks `keys` (the centre of the block's far voxel)."""
    c = (np.abs(np.asarray(keys, np.float64)) * 8 + 8) * voxel_size
    return float(np.spacing(c.astype(np.float32)).max())
