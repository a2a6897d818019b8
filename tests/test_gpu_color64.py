"""GPU: the float64-colour volume (B200TsdfVolume(color_float64=True), b2v_config.color_f64) against the float64-colour
restatement of tests/_color64.py, bit for bit: keys, tsdf, weights and rgb64, the mesh and the point cloud.  The
restatement equals the Open3D-order one (tests/test_color64_cpu.py), and T0 is checked against the golden directly.  Also: every input path and fusion setting, growth, reset, saturating uploaded weights, hash shards
with the face-halo exchange, state files, the TSDF plugin, and that tsdf and weights equal a default volume's."""

import os

import numpy as np
import pytest
import torch

import oracle
from pyslam_b200 import B200TsdfVolume, sharding
from pyslam_b200 import synthetic as S
from tests import _color64 as C64
from tests._util import GOLDEN, sort_dump

pytestmark = pytest.mark.gpu

N_C2 = 40


def _vol(cfg, cap=1 << 15, **kw):
    return B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=cap, color_float64=True,
                          **kw)


def _twin(cfg):
    return C64.Color64Twin(cfg)


def _stack(frames):
    return [np.stack([f[k] for f in frames]) for k in range(3)]


def _canon(m):
    return oracle.canonical_mesh(m.vertices, m.vertex_colors, m.edge_ids, m.triangles)


def _rows(*cols):
    a = np.concatenate([np.asarray(c, np.float64).reshape(len(c), -1) for c in cols], axis=1)
    return a[np.lexsort(a.T[::-1])] if len(a) else a


def _same_blocks(a, b):
    a, b = sort_dump(a), sort_dump(b)
    assert np.array_equal(a["keys"], b["keys"])
    assert np.array_equal(a["vox"].view(np.uint32), b["vox"].view(np.uint32))
    assert np.array_equal(a["rgb64"].view(np.uint64), b["rgb64"].view(np.uint64))


def _same_mesh(m, ref):
    ca = _canon(m)
    cb = oracle.canonical_mesh(ref["vertices"], ref["colors"], ref["edges"], ref["triangles"])
    assert len(ca["triangles"]) > 100
    for k in ("edges", "triangles", "vertices", "colors"):
        assert np.array_equal(ca[k], cb[k]), k


def _same_points(p, ref):
    assert len(p.points) > 100
    assert np.array_equal(_rows(p.edge_ids, p.points, p.colors), _rows(ref["edges"], ref["points"], ref["colors"]))


@pytest.fixture(scope="module")
def c2():
    cfg = S.CONFIGS["C2"]
    frames = [S.render_frame(cfg, i) for i in range(N_C2)]
    tw = _twin(cfg)
    for d, c, T in frames:
        tw.integrate(d, c, cfg.K, T, nthreads=8)
    dump = tw.dump_blocks()
    return cfg, frames, dump, C64.mesh(tw.tw.extract_mesh(), dump), C64.point_cloud(dump, cfg.voxel_size)


def test_T0_equals_the_golden():
    z = np.load(os.path.join(GOLDEN, "tsdf_T0.npz"))
    cfg = S.CONFIGS["T0"]
    v = _vol(cfg)
    for i in range(int(z["n_frames"])):
        v.integrate(z["depth"][i], z["color"][i], z["K"], z["Tcw"][i])
    d = sort_dump(v.dump_blocks())
    assert np.array_equal(d["keys"], z["keys"])
    assert np.array_equal(d["vox"][:, :2], z["vox"][:, :2])
    assert np.array_equal(d["rgb64"], z["o3d_rgb64"])
    assert np.array_equal(d["vox"][:, 2:], z["o3d_rgb64"].astype(np.float32))
    cm = _canon(v.extract_mesh())
    assert np.array_equal(cm["edges"], z["mesh_edges"]) and np.array_equal(cm["triangles"], z["mesh_triangles"])
    assert np.array_equal(cm["vertices"], z["mesh_vertices"])
    assert np.array_equal(cm["colors"], z["o3d_mesh_colors"])


@pytest.mark.parametrize("mode", ["g32", "g16", "g3", "g2", "nofuse", "nooverlap"])
def test_C2_fused_and_unfused_equal_the_twin(c2, mode):
    cfg, frames, dump, mesh, pts = c2
    v = _vol(cfg)
    if mode.startswith("g"):
        v.set_group_size(int(mode[1:]))
    elif mode == "nofuse":
        v.set_fusion(False)
    else:
        v.set_overlap(False)
    d, c, T = _stack(frames)
    v.integrate_batch(d, c, cfg.K, T)
    _same_blocks(v.dump_blocks(), dump)
    _same_mesh(v.extract_mesh(), mesh)
    _same_points(v.extract_point_cloud(), pts)


def test_C2_frame_by_frame_equals_the_twin_after_every_frame():
    cfg = S.CONFIGS["C2"]
    v, tw = _vol(cfg), _twin(cfg)
    for i in range(8):
        d, c, T = S.render_frame(cfg, i)
        v.integrate(d, c, cfg.K, T)
        tw.integrate(d, c, cfg.K, T, nthreads=8)
        _same_blocks(v.dump_blocks(), tw.dump_blocks())


def test_raw_u16_device_frames_on_a_caller_stream_and_gpu_rectification(c2):
    cfg, frames, _, _, _ = c2
    n = 12
    d16 = [np.round(f[0] * 5000.0).astype(np.uint16) for f in frames[:n]]
    scale = np.float32(1.0 / 5000.0)
    tw = _twin(cfg)
    for (_, c, T), q in zip(frames[:n], d16):
        tw.integrate(q.astype(np.float32) * scale, c, cfg.K, T, nthreads=8)
    want = tw.dump_blocks()
    # raw 16-bit depth, host
    a = _vol(cfg)
    a.integrate_batch(np.stack(d16), np.stack([f[1] for f in frames[:n]]), cfg.K,
                      np.stack([f[2] for f in frames[:n]]), depth_scale=float(scale))
    _same_blocks(a.dump_blocks(), want)
    # float depth as CUDA tensors on a caller stream
    b = _vol(cfg)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for (_, c, T), q in zip(frames[:n], d16):
            dd = torch.from_numpy(q.astype(np.float32) * scale).cuda()
            cc = torch.from_numpy(c).cuda()
            b.integrate(dd, cc, cfg.K, T, stream=s.cuda_stream)
    s.synchronize()
    _same_blocks(b.dump_blocks(), want)
    # identity rectification maps on the GPU (bilinear colour at integer coordinates is the pixel itself)
    r = _vol(cfg)
    y, x = np.mgrid[:cfg.height, :cfg.width].astype(np.float32)
    r.set_rectification(x, y)
    r.integrate_batch(np.stack(d16), np.stack([f[1] for f in frames[:n]]), cfg.K,
                      np.stack([f[2] for f in frames[:n]]), depth_scale=float(scale))
    _same_blocks(r.dump_blocks(), want)


def test_growth_from_64_blocks_equals_a_fixed_volume(c2):
    cfg, frames, dump, mesh, _ = c2
    g = _vol(cfg, cap=64, max_capacity_blocks=1 << 15)
    d, c, T = _stack(frames)
    g.integrate_batch(d, c, cfg.K, T)
    cap, growths = g.capacity()
    assert growths >= 1
    _same_blocks(g.dump_blocks(), dump)
    _same_mesh(g.extract_mesh(), mesh)


def test_reset_then_integrate_equals_a_fresh_volume():
    cfg = S.CONFIGS["T0"]
    frames = [S.render_frame(cfg, i) for i in range(4)]
    v, fresh = _vol(cfg), _vol(cfg)
    for d, c, T in frames:
        v.integrate(d, c, cfg.K, T)
    v.reset()
    assert v.num_blocks() == 0
    for d, c, T in frames[2:]:
        v.integrate(d, c, cfg.K, T)
        fresh.integrate(d, c, cfg.K, T)
    _same_blocks(v.dump_blocks(), fresh.dump_blocks())


@pytest.mark.parametrize("w", [16777215.0, 16777216.0])
def test_uploaded_weights_saturate_as_the_twin_does(w):
    cfg = S.CONFIGS["T0"]
    frames = [S.render_frame(cfg, i) for i in range(3)]
    tw = _twin(cfg)
    tw.integrate(*frames[0][:2], cfg.K, frames[0][2])
    seed = sort_dump(tw.dump_blocks())
    vox = seed["vox"].copy()
    vox[:, 1] = np.where(vox[:, 1] > 0, np.float32(w), 0.0)
    rgb = seed["rgb64"] + 1.0 / 3.0
    v, t2 = _vol(cfg), _twin(cfg)
    v.upload_blocks(seed["keys"], vox, rgb64=rgb)
    t2.upload(seed["keys"], vox, rgb)
    for d, c, T in frames[1:]:
        v.integrate(d, c, cfg.K, T)
        t2.integrate(d, c, cfg.K, T)
    got, want = sort_dump(v.dump_blocks()), sort_dump(t2.dump_blocks())
    _same_blocks(got, want)
    assert got["vox"][:, 1].max() == 16777216.0


def test_upload_arguments_and_weight_check():
    cfg = S.CONFIGS["T0"]
    v = _vol(cfg)
    keys = np.array([[0, 0, 0]], np.int32)
    vox = np.zeros((1, 5, 512), np.float32)
    with pytest.raises(ValueError):
        v.upload_blocks(keys, vox)                   # rgb64 required
    bad = vox.copy()
    bad[0, 1, 7] = 2.0 ** 25
    with pytest.raises(RuntimeError):
        v.upload_blocks(keys, bad, rgb64=np.zeros((1, 3, 512)))
    assert v.num_blocks() == 0
    d = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=64)
    with pytest.raises(ValueError):
        d.upload_blocks(keys, vox, rgb64=np.zeros((1, 3, 512)))   # a float32 volume refuses rgb64


def test_tsdf_and_weights_equal_a_default_volume(c2):
    cfg, frames, _, _, _ = c2
    d, c, T = _stack(frames)
    a, b = _vol(cfg), B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 15)
    a.integrate_batch(d, c, cfg.K, T)
    b.integrate_batch(d, c, cfg.K, T)
    da, db = sort_dump(a.dump_blocks()), sort_dump(b.dump_blocks())
    assert "rgb64" not in db
    assert np.array_equal(da["keys"], db["keys"])
    assert np.array_equal(da["vox"][:, :2].view(np.uint32), db["vox"][:, :2].view(np.uint32))
    ma, mb = _canon(a.extract_mesh()), _canon(b.extract_mesh())
    assert np.array_equal(ma["vertices"], mb["vertices"]) and np.array_equal(ma["triangles"], mb["triangles"])


@pytest.mark.parametrize("world", [2, 3])
def test_hash_shards_halo_mesh_and_points_equal_the_unsharded_volume(c2, world):
    cfg, frames, dump, mesh, pts = c2
    d, c, T = _stack(frames)
    single = _vol(cfg)
    single.integrate_batch(d, c, cfg.K, T)
    shards = [_vol(cfg, shard_rank=r, shard_count=world) for r in range(world)]
    for s in shards:
        s.integrate_batch(d, c, cfg.K, T)
    recs = [sharding.halo_records(v, world) for v in shards]
    assert all(int(h[:, 3].min()) >= 256 for rr in recs for h, _ in rr if len(h))   # the float64 flag on every record
    mp = [sharding.mesh_piece(v, [recs[s][r] for s in range(world)]) for r, v in enumerate(shards)]
    pp = [sharding.point_piece(v, [recs[s][r] for s in range(world)]) for r, v in enumerate(shards)]
    welded = sharding.weld(mp, device=0)
    _same_mesh(welded, mesh)
    ps = dict(points=np.concatenate([p.points for p in pp]), colors=np.concatenate([p.colors for p in pp]),
              edges=np.concatenate([p.edge_ids for p in pp]))
    _same_points(single.extract_point_cloud(), ps)
    _same_points(single.extract_point_cloud(), pts)
    # a float32 shard's records are refused by a float64 one
    f32 = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 15, shard_rank=1,
                         shard_count=world)
    f32.integrate_batch(d, c, cfg.K, T)
    h32, x32 = sharding.halo_records(f32, world)[0]
    with pytest.raises(RuntimeError, match="mask"):
        shards[0].extract_mesh_with_halo(h32, x32.reshape(-1)[: (x32.numel() // 8) * 8].reshape(-1, 8))


def test_state_round_trip_into_1_and_3_shards_and_cross_mode_refused(c2, tmp_path):
    cfg, frames, dump, mesh, _ = c2
    d, c, T = _stack(frames)
    v = _vol(cfg)
    v.integrate_batch(d, c, cfg.K, T)
    path = str(tmp_path / "map.npz")
    v.save_state(path)
    one = _vol(cfg)
    one.load_state(path)
    _same_blocks(one.dump_blocks(), dump)
    _same_mesh(one.extract_mesh(), mesh)
    parts = [_vol(cfg, shard_rank=r, shard_count=3) for r in range(3)]
    for p in parts:
        p.load_state(path)
    got = {k: np.concatenate([p.dump_blocks()[k] for p in parts]) for k in ("keys", "vox", "rgb64")}
    _same_blocks(got, dump)
    # a float32 volume refuses the float64 file, and a float64 volume a float32 file; both are left unchanged
    f32 = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 15)
    f32.integrate(*frames[0][:2], cfg.K, frames[0][2])
    before = sort_dump(f32.dump_blocks())
    with pytest.raises(ValueError):
        f32.load_state(path)
    after = sort_dump(f32.dump_blocks())
    assert np.array_equal(before["vox"], after["vox"])
    p32 = str(tmp_path / "map32.npz")
    f32.save_state(p32)
    with pytest.raises(ValueError):
        one.load_state(p32)
    _same_blocks(one.dump_blocks(), dump)


def test_tsdf_plugin_with_float64_colour():
    from tests import test_gpu_shard_plugin as SP
    cfg = S.CONFIGS["T0"]
    make = SP._tsdf(cfg, kVolumetricIntegrationB200ColorFloat64=True)
    one, many = make(), make(kVolumetricIntegrationB200Devices=[0, 0])
    outs = []
    for integ in (one, many):
        for i in range(12):
            integ.add_keyframe_data(SP._tsdf_kd(cfg, i, False))
        integ.run_pending()
        outs.append(SP._snap(integ, True))
    assert one.volume.color_float64
    ca, cb = _canon(outs[0]), _canon(outs[1])
    for k in ("vertices", "triangles", "edges", "colors"):
        assert np.array_equal(ca[k], cb[k]), k
    d = one.volume.dump_blocks()
    assert d["rgb64"].shape == (len(d["keys"]), 3, 512)
    assert np.any(d["rgb64"] != d["rgb64"].astype(np.float32))   # colours the float32 planes cannot hold
    one.quit()
    many.quit()
