"""CPU: the update-edge scenes of tests/test_gpu_tsdf_update_edges.py reach the boundaries they are built for, and the
twin (oracle/tsdf_oracle.c) stays the right truth on them.

- Every scene's emulated value equals its boundary constant, and the twin's weight planes show exactly the predicted
  voxels updated or skipped.
- The twin equals the Open3D-order restatement (oracle/open3d_order.c) in tsdf and weight on every scene with a
  rigid pose.  The exact-division scenes are not compared: Open3D allocates with the full inverse of the extrinsic,
  the twin and the kernels with its rigid inverse, which differ for their non-rigid poses.
- The straddling exact-division row mixes fast and exact voxels within a run and within a warp.
- A census over these scenes and 32 C2 frames reaches every group-mask popcount from 1 to 32."""

import numpy as np
import pytest

import oracle
from pyslam_b200 import synthetic as S
from tests import _update_edges as U
from tests._util import sort_dump, sorted_keys

f32 = np.float32


def _twin(sc):
    return oracle.TsdfOracle(sc.voxel_size, sc.sdf_trunc, sc.depth_trunc, stride=sc.stride, unit_resolution=sc.unit)


def _weight(tw, key, l):
    d = tw.dump_blocks()
    i = np.flatnonzero(np.all(d["keys"] == np.asarray(key), axis=1))
    assert len(i) == 1, key
    return d["vox"][i[0], 1, l[0] + 8 * l[1] + 64 * l[2]]


def _check_frames_alone(sc):
    """Each frame alone in a fresh twin: its target voxel took it exactly when predicted, and the emulated live set
    over the twin's touched blocks is the set of voxels whose weight the twin raised."""
    for f, (key, l, inside) in zip(sc.frames, sc.targets):
        tw = _twin(sc)
        tw.integrate(f[0], f[1], np.array(sc.K), f[2])
        assert _weight(tw, key, l) == (1.0 if inside else 0.0)
        d = tw.dump_blocks()
        want = U.live_voxels(f, sc.K, sc.voxel_size, sc.sdf_trunc, sc.depth_trunc, sc.unit, d["keys"])
        got = {tuple(int(x) for x in k): np.flatnonzero(v[1] > 0) for k, v in zip(d["keys"], d["vox"])}
        got = {k: v for k, v in got.items() if len(v)}
        assert got.keys() == want.keys()
        for k in got:
            assert np.array_equal(got[k], want[k]), k


def test_u_f_never_equals_the_margin_constant():
    """u_f = A + 0.5 (float32).  Every result in [2^-14, 2^-13) comes from an A in (-0.5, -0.25), where the sum is
    exact: u_f is then a multiple of 2^-25, and 0.0001f is not.  So `u_f >= 0.0001f` and `u_f > 0.0001f` decide
    alike for every input; the margin scenes take the reachable neighbours of 0.0001 instead."""
    lo = np.array(-0.5, f32).view(np.int32)
    hi = np.array(-0.25, f32).view(np.int32)
    A = np.arange(hi, lo + 1, dtype=np.int32).view(f32)        # every float32 in [-0.5, -0.25]
    assert not np.any((A + f32(0.5)) == U.MARGIN)
    assert np.array(U.MARGIN).view(np.int32) % (1 << 12) != 0   # its significand is not a multiple of 2^-25 / 2^-37


@pytest.mark.parametrize("W,H", [(96, 72), (2208, 1242)])
def test_margin_scenes_hit_their_boundaries(W, H):
    sc = U.margin_scene(W, H)
    safe_w, safe_h = f32(W) - U.MARGIN, f32(H) - U.MARGIN
    if W > 2048:
        assert safe_w == f32(W)                                  # the right margin collapses
    vals = {name: v for name, v, _ in sc.values}
    for a, safe in (("u", safe_w), ("v", safe_h)):
        assert vals[f"{a}_hi_out"] == safe and vals[f"{a}_hi_in"] == np.nextafter(safe, f32(0))
        assert vals[f"{a}_lo_out"] < U.MARGIN <= vals[f"{a}_lo_in"]
        assert vals[f"{a}_lo_in"] - vals[f"{a}_lo_out"] <= f32(2 ** -12)
    for f, (key, l, _), (name, v, _) in zip(sc.frames, sc.targets, sc.values):
        p = U.project(U.pose_E(f[2]), sc.K, W, H, sc.voxel_size, 16, key, *l)
        assert p[3 if name[0] == "u" else 4] == v


@pytest.mark.parametrize("unit", [16, 8])
def test_margin_scene_updates_the_predicted_voxels(unit):
    _check_frames_alone(U.margin_scene(96, 72, unit))


def test_margin_scene_hd_updates_the_predicted_voxels():
    _check_frames_alone(U.margin_scene(2208, 1242))


@pytest.mark.parametrize("unit", [16, 8])
def test_truncation_scene(unit):
    sc = U.truncation_scene(unit)
    tau = f32(sc.sdf_trunc)
    vals = {name: v for name, v, _ in sc.values}
    assert vals["sdf=-tau"] == -tau and vals["sdf=next(-tau)"] == np.nextafter(-tau, f32(1))
    assert vals["t=1"] == f32(1) and f32(0.999999) < vals["t<1"] < f32(1)
    for f, (key, l, _) in zip(sc.frames, sc.targets):
        assert U.lam(sc.K, int(sc.K[2]), int(sc.K[3])) == f32(1)
        live, sdf, t = U.block_update(f, sc.K, sc.voxel_size, sc.sdf_trunc, sc.depth_trunc, unit, key)
        i = (l[2], l[1], l[0])
        assert sdf[i] * (f32(1) / tau) == t[i] or t[i] == f32(1)
    _check_frames_alone(sc)


@pytest.mark.parametrize("unit", [8, 16])
def test_single_voxel_scene(unit):
    """Live frames: exactly one voxel of the volume takes the frame; the targets cover every run position and every
    warp.  The frame after each: the same pose with the target one ulp past the truncation bound, no voxel takes it
    and its block is touched."""
    sc = U.single_voxel_scene(unit)
    seen = set()
    for f, (key, l, inside), (_, sdf, bound) in zip(sc.frames, sc.targets, sc.values):
        assert (sdf > bound) == inside
        if not inside:
            assert sdf == np.nextafter(bound, f32(-1)) or sdf < bound
        tw = _twin(sc)
        tw.integrate(f[0], f[1], np.array(sc.K), f[2])
        assert tuple(key) in set(map(tuple, tw.last_touched().tolist()))
        w = tw.dump_blocks()["vox"][:, 1]
        assert int((w > 0).sum()) == (1 if inside else 0)
        seen.add(U.warp_and_run(l))
    assert seen == {(w, k) for w in range(4) for k in range(4)}
    _check_frames_alone(sc)


def test_division_scenes_take_the_exact_path():
    """'tiny': every in-image voxel of the touched blocks is on the exact path.  'straddle': a thread's 4-voxel run
    (and so a warp) holds in-image voxels of both paths.  Both update voxels (through the twin)."""
    for kind in ("tiny", "straddle"):
        frame = U.division_frames(kind, n=1)[0]
        tw = oracle.TsdfOracle(**U.DIV_PARAMS, unit_resolution=16)
        tw.integrate(frame[0], frame[1], np.array(U.DIV_K), frame[2])
        keys = tw.last_touched()
        split = U.division_split(frame, 16, keys)
        rare = sum(int(r.sum()) for r, _ in split.values())
        fast = sum(int(f.sum()) for _, f in split.values())
        assert rare > 1000
        assert (fast == 0) == (kind == "tiny")
        if kind == "straddle":
            mixed_run = mixed_warp = False
            for r, f in split.values():
                for z0 in (0, 4):   # a thread's run: lz = z0..z0+3 of one (lx, ly)
                    rr, ff = r[z0:z0 + 4], f[z0:z0 + 4]
                    mixed_run |= bool(np.any(rr.any(0) & ff.any(0)))
                    for wy in (0, 4):   # a warp: lx 0..7 x ly wy..wy+3 of one z half
                        mixed_warp |= bool(rr[:, wy:wy + 4].any() and ff[:, wy:wy + 4].any())
            assert mixed_run and mixed_warp
        assert (tw.dump_blocks()["vox"][:, 1] > 0).sum() > 1000


# ---------------------------------------------------------------------------------------------------------------------
# the twin against the Open3D-order restatement
# ---------------------------------------------------------------------------------------------------------------------

def _twin_vs_open3d(voxel_size, sdf_trunc, depth_trunc, K, frames, stride, unit=16):
    o3 = oracle.Open3DOrderVolume(voxel_size, sdf_trunc, unit, stride)
    tw = oracle.TsdfOracle(voxel_size, sdf_trunc, depth_trunc, stride=stride, unit_resolution=unit)
    for d, c, T in frames:
        o3.integrate(d, c, np.array(K), T, depth_trunc, nthreads=4)
        tw.integrate(d, c, np.array(K), T, nthreads=4)
    a, b = sort_dump(o3.dump_blocks()), sort_dump(tw.dump_blocks())
    assert np.array_equal(a["keys"], b["keys"])
    assert np.array_equal(a["vox"][:, 1], b["vox"][:, 1].astype(np.float64)), "weights differ"
    assert np.array_equal(a["vox"][:, 0], b["vox"][:, 0].astype(np.float64)), "tsdf differs"
    return int((b["vox"][:, 1] > 0).sum())


@pytest.mark.parametrize("name", ["margins-96", "margins-2208", "truncation", "single-voxel"])
def test_twin_equals_open3d_order(name):
    sc = {"margins-96": lambda: U.margin_scene(96, 72), "margins-2208": lambda: U.margin_scene(2208, 1242),
          "truncation": U.truncation_scene, "single-voxel": lambda: U.single_voxel_scene(16)}[name]()
    assert _twin_vs_open3d(sc.voxel_size, sc.sdf_trunc, sc.depth_trunc, sc.K, sc.frames, sc.stride) >= 16


# ---------------------------------------------------------------------------------------------------------------------
# group-mask census
# ---------------------------------------------------------------------------------------------------------------------

def _popcounts(voxel_size, sdf_trunc, depth_trunc, K, frames, stride, unit=16):
    """Popcounts of the group masks of a 32-frame group: per touched block, the number of frames touching it."""
    tw = oracle.TsdfOracle(voxel_size, sdf_trunc, depth_trunc, stride=stride, unit_resolution=unit)
    count = {}
    for d, c, T in frames:
        tw.integrate(d, c, np.array(K), T, nthreads=8)
        for k in map(tuple, tw.last_touched().tolist()):
            count[k] = count.get(k, 0) + 1
    return set(count.values())


def test_group_mask_census_reaches_every_popcount():
    """The parity of a block's popcount decides whether its last frame is applied from the first or the second
    gather buffer: the scenes of this file and 32 C2 frames reach every popcount 1..32."""
    cfg = S.CONFIGS["C2"]
    seen = _popcounts(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, cfg.K,
                      [S.render_frame(cfg, i) for i in range(32)], 4)
    for sc in (U.margin_scene(96, 72), U.truncation_scene(), U.single_voxel_scene(16)):
        seen |= _popcounts(sc.voxel_size, sc.sdf_trunc, sc.depth_trunc, sc.K, sc.frames, sc.stride)
    for kind in ("tiny", "straddle"):
        seen |= _popcounts(**U.DIV_PARAMS, K=U.DIV_K, frames=U.division_sequence(kind, (0, 1, 2, 30, 31)), stride=4)
    assert set(range(1, 33)) <= seen, sorted(set(range(1, 33)) - seen)
