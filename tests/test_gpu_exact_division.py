"""GPU: the exact-division fallback of the per-voxel TSDF update.

The update divides (tsdf * w + t) / (w + 1) with a shared reciprocal and two residual corrections, which is exact
only for a numerator of at least 2^-100 in magnitude (or zero).  A smaller numerator takes __fdiv_rn.  Integrated
frames never produce one: it needs a stored tsdf below 2^-100 and a voxel whose sdf is exactly 0.  Here blocks with a
tiny tsdf are uploaded and a flat depth image is placed exactly on a plane of voxel centres."""

import numpy as np
import pytest

import oracle
from pyslam_b200 import B200TsdfVolume
from pyslam_b200 import synthetic as S
from tests._util import sort_dump

TINY = np.float32(1e-35)   # tsdf * 1 + 0 < 2^-100
PLANE_Z = 15               # global voxel z of the plane; < 16, so it lies in the volume unit at z = 0


def _scene():
    cfg = S.CONFIGS["T0"]
    vs = np.float32(cfg.voxel_size)
    # camera z of voxel z = PLANE_Z under the identity pose, as the update computes it: the unit's first voxel centre
    # (vs / 2, float32), then one float32 step of vs per voxel
    z = np.float32(vs * np.float32(0.5))
    for _ in range(PLANE_Z):
        z = np.float32(z + vs)
    depth = np.full((cfg.height, cfg.width), z, np.float32)
    color = np.full((cfg.height, cfg.width, 3), 120, np.uint8)
    keys = np.array([(bx, by, PLANE_Z // 8) for bx in range(-3, 3) for by in range(-3, 3)], np.int32)
    vox = np.zeros((len(keys), 5, 512), np.float32)
    vox[:, 0] = TINY
    vox[:, 1] = 1.0
    vox[:, 2:] = 50.0
    return cfg, depth, color, keys, vox


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [False, True])
def test_tiny_numerator_takes_the_exact_division_path(fused):
    cfg, depth, color, keys, vox = _scene()
    n = 3
    vol = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=4096)
    orc = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    vol.upload_blocks(keys, vox)
    for k, v in zip(keys, vox):
        orc.set_block(k, v)
    T = np.eye(4)
    if fused:
        vol.integrate_batch(np.stack([depth] * n), np.stack([color] * n), cfg.K, np.stack([T] * n))
    else:
        for _ in range(n):
            vol.integrate(depth, color, cfg.K, T)
    for _ in range(n):
        orc.integrate(depth, color, cfg.K, T)
    a, b = sort_dump(vol.dump_blocks()), sort_dump(orc.dump_blocks())
    assert np.array_equal(a["keys"], b["keys"])
    assert np.array_equal(a["vox"], b["vox"])
    assert np.sum(a["vox"][:, 0] == _plane_tsdf(n)) >= 64   # the plane's voxels took the fallback n times


def _plane_tsdf(n):
    """tsdf of a plane voxel after n frames with t = 0: (tsdf * w + 0) / (w + 1), each step rounded to float32 (the
    float64 division is correctly rounded and the quotients stay normal, so rounding it to float32 is too)"""
    ts, w = TINY, np.float32(1.0)
    for _ in range(n):
        num = np.float32(np.float64(ts) * np.float64(w))
        assert 0 < abs(num) < 2.0 ** -100
        ts, w = np.float32(np.float64(num) / np.float64(w + 1)), np.float32(w + 1)
    return ts


def test_plane_scene_reaches_the_fallback_in_the_oracle():
    """The scene above, on the CPU twin alone: the plane voxels hold the chained exact quotients."""
    cfg, depth, color, keys, vox = _scene()
    orc = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    for k, v in zip(keys, vox):
        orc.set_block(k, v)
    for _ in range(3):
        orc.integrate(depth, color, cfg.K, np.eye(4))
    d = orc.dump_blocks()
    assert np.sum(d["vox"][:, 0] == _plane_tsdf(3)) >= 64
