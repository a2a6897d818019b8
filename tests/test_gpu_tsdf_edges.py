"""GPU: the TSDF kernels against the CPU twin (oracle/tsdf_oracle.c) at their edges, bit for bit: keys, hashes,
per-frame touched sets, all five planes, the mesh (edges, triangles, float64 vertices and colours) and the point
cloud's values.

- §1 allocation fallbacks: scenes that overflow the allocate kernel's per-tile shared-memory sets (key set, key list,
  new / first-touched lists), put units beyond rel_key's reach or boxes beyond the box offsets, or boxes wider than 15
  units (tests/test_tsdf_edges_cpu.py proves each scene reaches its path).
- §2 boundary inputs: special depths, voxels behind / on the camera plane, a principal point off the image, images
  smaller than one allocation tile at every stride, sparse group masks, the pool capacity boundary, fused groups of
  frames smaller than an earlier frame.
- §3 extraction on uploaded adversarial blocks: every marching-cubes case, a block at the emit kernels' maximum
  output, and the point cloud's positions and colours against oracle.numpy_point_cloud."""

import numpy as np
import pytest

import oracle
from pyslam_b200 import B200TsdfVolume
from pyslam_b200 import synthetic as S
from tests import _edge_scenes as E
from tests._util import sort_dump, sorted_keys

pytestmark = pytest.mark.gpu


def _volume(vs, tau, trunc, unit, stride=4, capacity=1 << 16, **kw):
    return B200TsdfVolume(vs, tau, trunc, capacity_blocks=capacity, depth_sampling_stride=stride,
                          volume_unit_resolution=unit, **kw)


def _same(a, b):
    """Two dumps (either side may be the twin's) hold the same blocks bit for bit."""
    a, b = sort_dump(a), sort_dump(b)
    for name in ("keys", "hashes", "vox"):
        assert np.array_equal(a[name], b[name]), name


def _same_mesh(m, ref):
    a = oracle.canonical_mesh(m.vertices, m.vertex_colors, m.edge_ids, m.triangles)
    b = oracle.canonical_mesh(ref["vertices"], ref["colors"], ref["edges"], ref["triangles"])
    for name in ("edges", "triangles", "vertices", "colors"):
        assert np.array_equal(a[name], b[name]), name
    return a


# ---------------------------------------------------------------------------------------------------------------------
# §1 allocation fallbacks
# ---------------------------------------------------------------------------------------------------------------------

_twin_cache = {}


def _twin(name):
    """Per-frame touched sets and the final dump of the twin over the scene's frames (computed once per scene)."""
    if name not in _twin_cache:
        sc = E.SCENES[name]
        tw = oracle.TsdfOracle(sc.voxel_size, sc.sdf_trunc, sc.depth_trunc, stride=sc.stride, unit_resolution=sc.unit)
        touched = []
        for s in E.SEEDS:
            d, c, T = sc.frame(s)
            tw.integrate(d, c, np.array(sc.K), T, nthreads=8)
            touched.append(sorted_keys(tw.last_touched()))
        _twin_cache[name] = (touched, tw.dump_blocks())
    return _twin_cache[name]


def _batch(sc):
    fr = [sc.frame(s) for s in E.SEEDS]
    return tuple(np.stack([f[k] for f in fr]) for k in range(3))


@pytest.mark.parametrize("name", list(E.SCENES))
@pytest.mark.parametrize("tma", [True, False])
def test_allocation_fallback_scenes_single_frames(name, tma, monkeypatch):
    """Frame by frame from an empty volume (the first frame takes the new-block overflow), with the TMA tile staging
    and with plain loads: every frame's touched set and the final volume equal the twin's."""
    sc = E.SCENES[name]
    if not tma:
        monkeypatch.setenv("B2V_TMA", "0")
    touched, ref = _twin(name)
    vol = _volume(sc.voxel_size, sc.sdf_trunc, sc.depth_trunc, sc.unit, sc.stride)
    total_new = 0
    for s, want in zip(E.SEEDS, touched):
        d, c, T = sc.frame(s)
        vol.integrate(d, c, np.array(sc.K), T)
        assert np.array_equal(sorted_keys(vol.last_touched_keys()), want), s
        t, new = vol.last_frame_stats()
        assert t == len(want)
        total_new += new
    assert total_new == vol.num_blocks() == len(ref["keys"])
    _same(vol.dump_blocks(), ref)
    vol.close()


@pytest.mark.parametrize("name", list(E.SCENES))
def test_allocation_fallback_scenes_batches(name):
    """The scene's frames as one fused group of up to 32, as groups of 3, and un-fused: the twin's volume each time."""
    sc = E.SCENES[name]
    touched, ref = _twin(name)
    D, C, T = _batch(sc)
    for mode in ("group32", "group3", "unfused"):
        vol = _volume(sc.voxel_size, sc.sdf_trunc, sc.depth_trunc, sc.unit, sc.stride)
        if mode == "unfused":
            vol.set_fusion(False)
        else:
            vol.set_group_size(32 if mode == "group32" else 3)
        vol.integrate_batch(D, C, np.array(sc.K), T)
        assert vol.last_frame_stats()[0] == len(touched[-1]), mode
        assert vol.num_blocks() == len(ref["keys"]), mode
        _same(vol.dump_blocks(), ref)
        vol.close()


def test_noisy_d1_shards_partition_the_volume():
    """3 hash shards (the 64-bit modulo owner test) of the noisy-D1 batch: their union is the twin's volume."""
    sc = E.SCENES["noisy-D1"]
    _, ref = _twin("noisy-D1")
    D, C, T = _batch(sc)
    parts = []
    for r in range(3):
        s = _volume(sc.voxel_size, sc.sdf_trunc, sc.depth_trunc, sc.unit, sc.stride, shard_rank=r, shard_count=3)
        s.integrate_batch(D, C, np.array(sc.K), T)
        p = s.dump_blocks()
        assert np.all(p["hashes"] % np.uint64(3) == r)
        parts.append(p)
        s.close()
    _same({k: np.concatenate([p[k] for p in parts]) for k in ("keys", "hashes", "vox")}, ref)


# ---------------------------------------------------------------------------------------------------------------------
# §2 boundary inputs
# ---------------------------------------------------------------------------------------------------------------------

def _run_both(cfg, frames, unit=16, stride=4, capacity=1 << 15, batch=True):
    """frames [(depth, colour, K, Tcw)] sharing one K: frame by frame (touched sets checked) and, if `batch`, as one
    fused batch; both against the twin."""
    tw = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, stride=stride, unit_resolution=unit)
    vol = _volume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, unit, stride, capacity)
    for d, c, K, T in frames:
        vol.integrate(d, c, K, T)
        n = tw.integrate(d, c, K, T)
        assert np.array_equal(sorted_keys(vol.last_touched_keys()), sorted_keys(tw.last_touched()))
        assert vol.last_frame_stats()[0] == n
    ref = tw.dump_blocks()
    _same(vol.dump_blocks(), ref)
    vol.close()
    if batch:
        fused = _volume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, unit, stride, capacity)
        fused.integrate_batch(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]), frames[0][2],
                              np.stack([f[3] for f in frames]))
        assert fused.last_frame_stats()[0] == len(tw.last_touched())
        _same(fused.dump_blocks(), ref)
        fused.close()
    return ref


@pytest.mark.parametrize("unit", [16, 8])
def test_special_depths(unit):
    cfg = S.CONFIGS["T0"]
    d, c, T = E.specials_frame()
    d1, c1, T1 = S.render_frame(cfg, 1)
    ref = _run_both(cfg, [(d, c, cfg.K, T), (d1, c1, cfg.K, T1), (d, c, cfg.K, T1)], unit=unit)
    assert (ref["vox"][:, 1] > 0).sum() > 10000


@pytest.mark.parametrize("unit", [16, 8])
def test_camera_inside_the_band(unit):
    """Voxels behind the camera, then a layer of voxel centres exactly on the camera plane (p.z = +0.0)."""
    cfg = S.CONFIGS["T0"]
    ref = _run_both(cfg, E.band_frames(cfg), unit=unit)
    assert (ref["vox"][:, 1] > 0).sum() > 500


@pytest.mark.parametrize("K", [(80.0, 95.0, -20.25, 72 + 10.5), (80.0, 80.0, 0.0, 0.0)])
def test_principal_point_off_the_image(K):
    cfg = S.CONFIGS["T0"]
    frames = []
    for i in range(3):
        d, c, T = S.render_frame(cfg, i)
        frames.append((d, c, np.array(K), T))
    _run_both(cfg, frames)


@pytest.mark.parametrize("shape", [(1, 1), (3, 5), (31, 33), (32, 32), (8, 16), (40, 48)])
def test_small_images_every_stride_and_unit(shape):
    """Images smaller than one allocation tile, at strides whose tiles take the plain loads (1, 2, 3, 5, 8) and the
    TMA staging (4; (8, 16) and (40, 48) are TMA-eligible widths narrower than / not a multiple of the 32-pixel box)."""
    cfg = S.CONFIGS["T0"]
    H, W = shape
    for stride in (1, 2, 3, 4, 5, 8):
        for unit in (8, 16):
            frames = []
            for i in range(3):
                d, c, K, T = E.crop(cfg, i, H, W)
                frames.append((d, c, K, T))
            _run_both(cfg, frames, unit=unit, stride=stride, capacity=4096)


def _sparse_check(cfg, D, C, T, group):
    tw = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    for i in range(len(D)):
        tw.integrate(D[i], C[i], cfg.K, T[i])
    ref = tw.dump_blocks()
    fused = _volume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, 16, capacity=1 << 14)
    fused.set_group_size(group)
    plain = _volume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, 16, capacity=1 << 14)
    plain.set_fusion(False)
    for v in (fused, plain):
        v.integrate_batch(D, C, cfg.K, T)
        assert v.last_frame_stats()[0] == len(tw.last_touched())
        _same(v.dump_blocks(), ref)
    assert fused.counters()[0] == plain.counters()[0]      # the same (block, frame) updates
    return fused, plain, tw


def test_sparse_group_masks():
    cfg = S.CONFIGS["T0"]
    fr = [S.render_frame(cfg, i % cfg.n_frames) for i in range(32)]
    D, C, T = (np.stack([f[k] for f in fr]) for k in range(3))
    # frames 1..30 of a 32-frame group see nothing: only bits 0 and 31 of the masks are set
    D1 = D.copy()
    for i in range(1, 31):
        D1[i] = E.invalid_depth(D1[i].shape, i)
    fused, plain, tw = _sparse_check(cfg, D1, C, T, 32)
    # a batch that touches nothing leaves the volume unchanged and reports (0, 0)
    before = fused.dump_blocks()
    bad = np.stack([E.invalid_depth(D[0].shape, 100 + i) for i in range(5)])
    for v in (fused, plain):
        v.integrate_batch(bad, C[:5], cfg.K, T[:5])
        assert v.last_frame_stats() == (0, 0)
        _same(v.dump_blocks(), before)
        v.close()
    # only the last frame of a group sees the right half of the image
    D2 = D[:9].copy()
    D2[:8, :, cfg.width // 2:] = 0.0
    fused, plain, tw = _sparse_check(cfg, D2, C[:9], T[:9], 9)
    fused.close()
    plain.close()


def test_pool_capacity_boundary():
    """capacity_blocks equal to the twin's block count: no error, the twin's volume.  One block less: the pool-full
    error, raised at the next synchronisation."""
    cfg = S.CONFIGS["C1"]
    fr = [S.render_frame(cfg, i) for i in (0, 1, 2)]
    tw = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    for d, c, T in fr:
        tw.integrate(d, c, cfg.K, T)
    n = tw.num_blocks()
    D, C, T = (np.stack([f[k] for f in fr]) for k in range(3))
    exact = _volume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, 16, capacity=n)
    for d, c, t in fr:
        exact.integrate(d, c, cfg.K, t)
    exact.synchronize()
    assert exact.num_blocks() == n
    _same(exact.dump_blocks(), tw.dump_blocks())
    exact.close()
    fused = _volume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, 16, capacity=n)
    fused.integrate_batch(D, C, cfg.K, T)
    fused.synchronize()
    _same(fused.dump_blocks(), tw.dump_blocks())
    fused.close()
    for batch in (False, True):
        short = _volume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, 16, capacity=n - 1)
        with pytest.raises(RuntimeError, match="block pool full"):
            if batch:
                short.integrate_batch(D, C, cfg.K, T)
            else:
                for d, c, t in fr:
                    short.integrate(d, c, cfg.K, t)
            short.synchronize()
        short.close()


@pytest.mark.parametrize("group", [8, 3])
@pytest.mark.parametrize("depth_kind", ["f32_host", "u16_host", "u16_cuda"])
def test_smaller_frames_after_larger_ones(depth_kind, group):
    """Fused groups of frames smaller than an earlier frame of the volume: the staging slots of a group follow the
    current frame size, so every frame of a group reads its own upload (or widened uint16 depth)."""
    cfg, big = S.CONFIGS["T0"], S.CONFIGS["C1"]
    scale = np.float32(1.0 / 5000.0)
    vol = _volume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, 16)
    vol.set_group_size(group)
    tw = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
    for c, n in ((big, 4), (cfg, 8)):
        fr = [S.render_frame(c, i) for i in range(n)]
        D, Cc, T = (np.stack([f[k] for f in fr]) for k in range(3))
        if depth_kind == "f32_host":
            vol.integrate_batch(D, Cc, c.K, T)
        else:
            raw = np.round(D * 5000.0).astype(np.uint16)
            D = raw.astype(np.float32) * scale
            if depth_kind == "u16_cuda":
                import torch
                vol.integrate_batch(torch.from_numpy(raw).cuda(), torch.from_numpy(Cc).cuda(), c.K, T,
                                    depth_scale=scale)
                vol.synchronize()   # before the tensors are released
            else:
                vol.integrate_batch(raw, Cc, c.K, T, depth_scale=scale)
        for i in range(n):
            tw.integrate(D[i], Cc[i], c.K, T[i])
    _same(vol.dump_blocks(), tw.dump_blocks())
    vol.close()


# ---------------------------------------------------------------------------------------------------------------------
# §3 extraction on uploaded adversarial blocks
# ---------------------------------------------------------------------------------------------------------------------

def _uploaded(keys, vox, vs=0.02, tau=0.08, unit=16):
    vol = _volume(vs, tau, 4.0, unit, capacity=4096)
    vol.upload_blocks(keys, vox)
    tw = oracle.TsdfOracle(vs, tau, 4.0, unit_resolution=unit)
    for k, v in zip(keys, vox):
        tw.set_block(k, v)
    return vol, tw


def _sorted_points(p, c):
    o = np.lexsort((c[:, 2], c[:, 1], c[:, 0], p[:, 2], p[:, 1], p[:, 0]))
    return p[o], c[o]


def _check_points(vol, vs, unit, mesh=None):
    """extract_point_cloud == oracle.numpy_point_cloud bit for bit.  Where an edge carries both a point and a mesh
    vertex, the two independent formulas agree: off the edge's axis to 1e-12 m (both float64); along it to
    |p| 2^-23 + 1e-12, because the point divides the whole coordinate by the float32 sum rs = r0 + r1, whose rounding
    (<= 2^-24 relative) scales the absolute position; colours to 1e-6."""
    dump = vol.dump_blocks()
    want = oracle.numpy_point_cloud(dump, vs, unit)
    pc = vol.extract_point_cloud()
    assert pc.points.dtype == np.float64 and pc.colors.dtype == np.float64
    gp, gc = _sorted_points(pc.points, pc.colors)
    wp, wc = _sorted_points(want["points"], want["colors"])
    assert gp.shape == wp.shape
    assert np.array_equal(gp, wp) and np.array_equal(gc, wc)
    if mesh is not None:
        vid = {tuple(e): i for i, e in enumerate(mesh.edge_ids.tolist())}
        pairs = [(i, vid[tuple(e)]) for i, e in enumerate(want["edges"].tolist()) if tuple(e) in vid]
        assert len(pairs) > 1000
        pi, mi = np.array(pairs).T
        p, v = want["points"][pi], mesh.vertices[mi]
        on_axis = np.arange(3)[None, :] == want["edges"][pi, 3:4]
        err = np.abs(p - v)
        assert err[~on_axis].max() < 1e-12
        assert np.all(err[on_axis] <= np.abs(p[on_axis]) * 2.0 ** -23 + 1e-12)
        assert np.abs(want["colors"][pi] - mesh.vertex_colors[mi]).max() < 1e-6
    return len(gp)


@pytest.mark.parametrize("unit", [16, 8])
def test_random_blocks_mesh_and_point_cloud(unit):
    keys, vox = E.random_blocks()
    vol, tw = _uploaded(keys, vox, unit=unit)
    dump = vol.dump_blocks()
    assert set(np.unique(E.cube_cases(dump["keys"], dump["vox"])).tolist()) >= set(range(1, 255))
    m = vol.extract_mesh()
    a = _same_mesh(m, tw.extract_mesh())
    assert len(a["triangles"]) > 10000
    assert _check_points(vol, 0.02, unit, m) > 10000
    vol.close()


def test_maximum_output_block():
    """A checkerboard block with its 7 forward neighbours observed: 1536 vertices in one block (the emit kernels'
    shared vertex list is full) and 4 triangles per cube."""
    keys, vox = E.max_output_blocks()
    vol, tw = _uploaded(keys, vox)
    m = vol.extract_mesh()
    a = _same_mesh(m, tw.extract_mesh())
    own = np.all((a["edges"][:, :3] >= 0) & (a["edges"][:, :3] < 8), axis=1)
    assert own.sum() == 3 * 512
    assert len(a["triangles"]) >= 4 * 512
    _check_points(vol, 0.02, 16, m)
    vol.close()


def test_point_cloud_values_of_an_integrated_volume():
    cfg = S.CONFIGS["C1"]
    vol = _volume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, 16, capacity=1 << 15)
    for i in range(4):
        d, c, T = S.render_frame(cfg, i)
        vol.integrate(d, c, cfg.K, T)
    assert _check_points(vol, cfg.voxel_size, 16, vol.extract_mesh()) > 1000
    vol.close()
