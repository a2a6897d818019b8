"""GPU: the TSDF update at its per-voxel decision boundaries, against the CPU twin (oracle/tsdf_oracle.c) bit for bit:
keys, hashes, all five planes, the per-frame touched sets frame by frame, and counters()[0] (the (block, frame)
updates) equal to the twin's in every mode.  Every scene of tests/_update_edges.py runs frame by frame, fused in
groups of 32, 3 and 2, and un-fused; tests/test_update_edges_cpu.py proves each scene reaches its boundary.

- margins: u_f / v_f just inside and outside the image margins, at W = 96 and at W = 2208 (right margin collapsed);
- truncation: sdf == -tau against the float above, t == 1 against just below;
- single live voxel: blocks in which exactly one voxel (at each run position and in each warp) takes a frame, and
  the same frames one ulp past the truncation bound;
- exact division inside fused groups: the frame of interest at group positions 0, 1, 2, 30 and 31, as two
  consecutive frames and as every frame of a group, with every voxel or one run's voxels on the exact path;
- uploaded weights: [0, 2^24] integrates like the twin, anything else is refused by upload, import and state load
  with the volume unchanged;
- HD frames: 128 frames at 2208 x 1242 and 4096 x 2160 in fused groups of 32, so that every staging and texel slot
  0..127 is used and the texel offsets pass 2^31 (2208) and 2^32 (4096)."""

import numpy as np
import pytest

import oracle
from pyslam_b200 import B200TsdfVolume
from pyslam_b200 import synthetic as S
from tests import _update_edges as U
from tests._util import sort_dump, sorted_keys

pytestmark = pytest.mark.gpu

MODES = ("frames", "group32", "group3", "group2", "unfused")


def _volume(p, unit, stride, capacity=1 << 15):
    return B200TsdfVolume(p["voxel_size"], p["sdf_trunc"], p["depth_trunc"], capacity_blocks=capacity,
                          depth_sampling_stride=stride, volume_unit_resolution=unit)


def _same(a, b):
    a, b = sort_dump(a), sort_dump(b)
    for name in ("keys", "hashes", "vox"):
        assert np.array_equal(a[name], b[name]), name


def _run_modes(p, K, frames, unit, stride, uploads=None):
    """The frames in every mode against the twin (uploaded blocks first, when given).  Returns the twin's dump."""
    K = np.array(K, np.float64)
    tw = oracle.TsdfOracle(p["voxel_size"], p["sdf_trunc"], p["depth_trunc"], stride=stride, unit_resolution=unit)
    if uploads is not None:
        for k, v in zip(*uploads):
            tw.set_block(k, v)
    touched, updates = [], 0
    for d, c, T in frames:
        updates += tw.integrate(d, c, K, T, nthreads=8)
        touched.append(sorted_keys(tw.last_touched()))
    ref = tw.dump_blocks()
    D, C, T = (np.stack([f[k] for f in frames]) for k in range(3))
    for mode in MODES:
        vol = _volume(p, unit, stride)
        if uploads is not None:
            vol.upload_blocks(*uploads)
        if mode == "frames":
            for (d, c, t), want in zip(frames, touched):
                vol.integrate(d, c, K, t)
                assert np.array_equal(sorted_keys(vol.last_touched_keys()), want)
        else:
            if mode == "unfused":
                vol.set_fusion(False)
            else:
                vol.set_group_size(int(mode[5:]))
            vol.integrate_batch(D, C, K, T)
        assert vol.counters()[0] == updates, mode
        _same(vol.dump_blocks(), ref)
        vol.close()
    return ref


def _scene_params(sc):
    return dict(voxel_size=sc.voxel_size, sdf_trunc=sc.sdf_trunc, depth_trunc=sc.depth_trunc)


def _target_weights(ref, targets):
    """The final weight of each target voxel."""
    idx = {tuple(k): i for i, k in enumerate(ref["keys"].tolist())}
    return [ref["vox"][idx[tuple(key)], 1, l[0] + 8 * l[1] + 64 * l[2]] for key, l, _ in targets]


# ---------------------------------------------------------------------------------------------------------------------
# margins, truncation, single live voxels
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("W,H,unit", [(96, 72, 16), (96, 72, 8), (2208, 1242, 16)])
def test_image_margins(W, H, unit):
    sc = U.margin_scene(W, H, unit)
    ref = _run_modes(_scene_params(sc), sc.K, sc.frames, unit, sc.stride)
    assert all(w > 0 for w in _target_weights(ref, sc.targets))


@pytest.mark.parametrize("unit", [16, 8])
def test_truncation_bounds(unit):
    sc = U.truncation_scene(unit)
    _run_modes(_scene_params(sc), sc.K, sc.frames, unit, sc.stride)
    # each frame alone: its target took it exactly when the CPU scene test predicts
    for f, (key, l, inside) in zip(sc.frames, sc.targets):
        vol = _volume(_scene_params(sc), unit, sc.stride)
        vol.integrate(f[0], f[1], np.array(sc.K), f[2])
        assert _target_weights(vol.dump_blocks(), [(key, l, inside)])[0] == float(inside)
        vol.close()


@pytest.mark.parametrize("unit", [8, 16])
def test_single_live_voxel_per_block(unit):
    """32 frames on one block: 16 in which exactly one of its voxels takes the frame (every run position, every
    warp), each followed by the same frame with that voxel one ulp past the truncation bound."""
    sc = U.single_voxel_scene(unit)
    ref = _run_modes(_scene_params(sc), sc.K, sc.frames, unit, sc.stride)
    assert int((ref["vox"][:, 1] > 0).sum()) == 16
    assert all(w == 1.0 for w in _target_weights(ref, sc.targets))
    # the live frames alone, and the ulp-past frames alone (touch, no update, no stored block)
    for sel in (slice(0, None, 2), slice(1, None, 2)):
        _run_modes(_scene_params(sc), sc.K, sc.frames[sel], unit, sc.stride)


# ---------------------------------------------------------------------------------------------------------------------
# exact division inside fused groups
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["tiny", "straddle"])
@pytest.mark.parametrize("positions", [(0,), (1,), (2,), (30,), (31,), (5, 6), "all"])
def test_exact_division_in_fused_groups(kind, positions):
    frames = U.division_sequence(kind, positions)
    ref = _run_modes(U.DIV_PARAMS, U.DIV_K, frames, 16, 4)
    assert (ref["vox"][:, 1] > 0).sum() > 1000


# ---------------------------------------------------------------------------------------------------------------------
# uploaded weights
# ---------------------------------------------------------------------------------------------------------------------

def _weight_keys():
    cfg = S.CONFIGS["T0"]
    tw = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    d, c, T = S.render_frame(cfg, 0)
    tw.integrate(d, c, cfg.K, T)
    return sorted_keys(tw.last_touched())[::3]


@pytest.mark.parametrize("w", U.ACCEPTED_WEIGHTS)
def test_uploaded_weights_in_range_integrate_like_the_twin(w):
    cfg = S.CONFIGS["T0"]
    up = U.weight_blocks(_weight_keys(), w)
    frames = [S.render_frame(cfg, i) for i in range(4)]
    ref = _run_modes(dict(voxel_size=cfg.voxel_size, sdf_trunc=cfg.sdf_trunc, depth_trunc=cfg.depth_trunc), cfg.K,
                     frames, 16, 4, uploads=up)
    if w == 2.0 ** 24:
        assert (ref["vox"][:, 1] == np.float32(2.0 ** 24)).sum() > 1000      # w + 1 rounds back to w


@pytest.mark.parametrize("w", U.REJECTED_WEIGHTS)
def test_uploaded_weights_out_of_range_are_refused(w, tmp_path):
    """upload_blocks, import_blocks_torch and load_state refuse a block with one such weight; the volume keeps its
    blocks, capacity and values."""
    import torch
    cfg = S.CONFIGS["T0"]
    keys = _weight_keys()
    good = U.weight_blocks(keys[:8], 3.0, seed=1)
    vol = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=64,
                         max_capacity_blocks=4096)
    vol.upload_blocks(*good)
    d, c, T = S.render_frame(cfg, 0)
    vol.integrate(d, c, cfg.K, T)
    before, cap = vol.dump_blocks(), vol.capacity()
    bk, bv = U.weight_blocks(keys, 1.0, seed=2)
    bv[len(keys) // 2, 1, 300] = np.float32(w)                              # one voxel of one block
    with pytest.raises(RuntimeError, match="weights outside"):
        vol.upload_blocks(bk, bv)
    k4 = torch.from_numpy(np.concatenate([bk, np.zeros((len(bk), 1), np.int32)], 1)).cuda()
    with pytest.raises(RuntimeError, match="weights outside"):
        vol.import_blocks_torch(k4, torch.from_numpy(bv).cuda())
    src = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=4096)
    src.upload_blocks(bk, np.where(np.arange(5)[None, :, None] == 1, 1.0, bv).astype(np.float32))
    path = str(tmp_path / "state.npz")
    src.save_state(path)
    z = dict(np.load(path))
    z["blocks_vox"][len(keys) // 2, 1, 300] = np.float32(w)
    np.savez(path, **z)
    with pytest.raises(ValueError, match="weights outside"):
        vol.load_state(path)
    assert vol.capacity() == cap
    _same(vol.dump_blocks(), before)
    src.close()
    vol.close()


# ---------------------------------------------------------------------------------------------------------------------
# HD frames: every slot of four group buffers, texel offsets past 2^31 and 2^32
# ---------------------------------------------------------------------------------------------------------------------

HD = {
    (2208, 1242): S.SequenceConfig("HD2K", 2208, 1242, 1050.0, 1050.0, 1103.5, 620.5, 0.02, 0.08, 4.0, 4, 11),
    (4096, 2160): S.SequenceConfig("HD4K", 4096, 2160, 1950.0, 1950.0, 2047.5, 1079.5, 0.02, 0.08, 4.0, 4, 12),
}
N_HD = 128


def _hd_frames(cfg):
    """4 rendered poses cycled over 128 frames; frame i's colour is its pose's plus i (mod 256), so a frame read
    from another slot shows in the colour planes."""
    base = [S.render_frame(cfg, i) for i in range(4)]
    return base, [(i % 4, np.uint8(i)) for i in range(N_HD)]


@pytest.mark.parametrize("W,H,kind", [(2208, 1242, "f32_host"), (4096, 2160, "u16_host"), (4096, 2160, "u16_cuda")])
def test_hd_frames_in_every_slot(W, H, kind):
    cfg = HD[(W, H)]
    px = W * H
    texel_pitch = (px + 32) & ~31
    assert 127 * texel_pitch * 8 > 2 ** 31 and (W < 4096 or 61 * texel_pitch * 8 > 2 ** 32)
    base, order = _hd_frames(cfg)
    scale = np.float32(1.0 / 5000.0)
    raw = [np.round(b[0] * 5000.0).astype(np.uint16) for b in base]
    depth_f = [r.astype(np.float32) * scale for r in raw] if kind != "f32_host" else [b[0] for b in base]
    C = np.empty((N_HD, H, W, 3), np.uint8)
    for i, (j, add) in enumerate(order):
        np.add(base[j][1], add, out=C[i], casting="unsafe")
    T = np.stack([base[j][2] for j, _ in order])
    p = dict(voxel_size=cfg.voxel_size, sdf_trunc=cfg.sdf_trunc, depth_trunc=cfg.depth_trunc)

    tw = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    updates = 0
    for i, (j, _) in enumerate(order):
        updates += tw.integrate(depth_f[j], C[i], cfg.K, T[i], nthreads=oracle.TsdfOracle.max_threads())
    ref = tw.dump_blocks()

    fused = _volume(p, 16, 4, capacity=1 << 17)
    fused.set_group_size(32)
    if kind == "f32_host":
        D = np.stack([depth_f[j] for j, _ in order])
        fused.integrate_batch(D, C, cfg.K, T)
    elif kind == "u16_host":
        D = np.stack([raw[j] for j, _ in order])
        fused.integrate_batch(D, C, cfg.K, T, depth_scale=scale)
    else:
        import torch
        D = torch.from_numpy(np.stack([raw[j] for j, _ in order]).view(np.int16)).cuda()
        Cd = torch.from_numpy(C).cuda()
        fused.integrate_batch(D, Cd, cfg.K, T, depth_scale=scale)
        fused.synchronize()
        del D, Cd
    assert fused.counters()[0] == updates
    got = fused.dump_blocks()
    _same(got, ref)

    single = _volume(p, 16, 4, capacity=1 << 17)
    for i, (j, _) in enumerate(order):
        if kind == "f32_host":
            single.integrate(depth_f[j], C[i], cfg.K, T[i])
        else:
            single.integrate(raw[j], C[i], cfg.K, T[i], depth_scale=scale)
    _same(single.dump_blocks(), got)
    single.close()

    if kind != "u16_cuda":
        m = fused.extract_mesh()
        want = tw.extract_mesh()
        a = oracle.canonical_mesh(m.vertices, m.vertex_colors, m.edge_ids, m.triangles)
        b = oracle.canonical_mesh(want["vertices"], want["colors"], want["edges"], want["triangles"])
        for name in ("edges", "triangles", "vertices", "colors"):
            assert np.array_equal(a[name], b[name]), name
        assert len(a["triangles"]) > 10000
        pc = fused.extract_point_cloud()
        wp = oracle.numpy_point_cloud(got, cfg.voxel_size, 16)
        o1 = np.lexsort(pc.points.T[::-1])
        o2 = np.lexsort(wp["points"].T[::-1])
        assert np.array_equal(pc.points[o1], wp["points"][o2]) and np.array_equal(pc.colors[o1], wp["colors"][o2])
    fused.close()
