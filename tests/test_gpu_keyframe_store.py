"""GPU: the TSDF volume's frame store.  Frames integrated with the store on, then reset() and integrated again from the
store with other poses (integrate_stored), give the map a fresh volume gives when it integrates the same frames'
images with those poses: the same blocks bit for bit, the same mesh and the same point cloud.  Through the plugins, a
loop-closure rebuild sends only light tasks and gives the store-off plugin's mesh, sharded or not."""

import os
from types import SimpleNamespace

import numpy as np
import pytest

import oracle
from pyslam_b200 import B200TsdfVolume, keyframe_store, shard_plugin
from pyslam_b200 import synthetic as S
from tests import plugin_standins as P
from tests._edge_scenes import crop, specials_frame
from tests._util import GOLDEN, sort_dump

pytestmark = pytest.mark.gpu

_frames_cache = {}


def _frames(name, n):
    if (name, n) not in _frames_cache:
        cfg = S.CONFIGS[name]
        fr = [S.render_frame(cfg, i % cfg.n_frames) for i in range(n)]
        _frames_cache[name, n] = tuple(np.stack([f[k] for f in fr]) for k in range(3))
    return _frames_cache[name, n]


def _moved(T, shift=0.0):
    """The poses after a 'loop closure': each rotated by a small angle and moved a little (frame i also by
    i * shift metres along x)."""
    out = []
    for i, t in enumerate(T):
        a = 0.01 * (1 + i % 3)
        D = np.eye(4)
        D[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
        D[:3, 3] = [0.01 + i * shift, -0.005, 0.007]
        out.append(t @ D)
    return np.stack(out)


def _volume(cfg, **kw):
    kw.setdefault("capacity_blocks", 1 << 15)
    return B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, **kw)


def _same(a, b):
    da, db = sort_dump(a.dump_blocks()), sort_dump(b.dump_blocks())
    assert len(da["keys"]) > 50
    assert set(da) == set(db)
    for name in da:
        assert np.array_equal(da[name], db[name]), name
    ma, mb = a.extract_mesh(), b.extract_mesh()
    ca = oracle.canonical_mesh(ma.vertices, ma.vertex_colors, ma.edge_ids, ma.triangles)
    cb = oracle.canonical_mesh(mb.vertices, mb.vertex_colors, mb.edge_ids, mb.triangles)
    assert len(ma.triangles) > 100
    for name in ("edges", "triangles", "vertices", "colors"):
        assert np.array_equal(ca[name], cb[name]), name
    pa, pb = a.extract_point_cloud(), b.extract_point_cloud()
    assert len(pa.points) > 100
    rows = lambda p: (lambda r: r[np.lexsort(r.T[::-1])])(  # noqa: E731
        np.concatenate([p.edge_ids.astype(np.float64), p.points, p.colors], axis=1))
    assert np.array_equal(rows(pa), rows(pb))


def _integrate(vol, mode, D, C, K, T, scale=None):
    """The frames in `mode` ("frames": one call per frame; "groupN": one batch call in groups of N); the store slot of
    each frame."""
    if mode == "frames":
        slots = []
        for i in range(len(D)):
            vol.integrate(D[i], C[i], K, T[i], depth_scale=scale)
            slots += list(vol.last_stored_slots())
        return np.array(slots, np.int32)
    vol.set_group_size(int(mode[5:]))
    vol.integrate_batch(D, C, K, T, depth_scale=scale)
    return vol.last_stored_slots()


def _replay(vol, mode, slots, K, T):
    vol.reset()
    if mode == "frames":
        for s, t in zip(slots, T):
            vol.integrate_stored([s], K, t[None])
    else:
        vol.integrate_stored(slots, K, T)
    assert (vol.last_stored_slots() == -1).all()


CASES = {
    "group32": dict(cfg="C1", n=64, mode="group32"),
    "group16_f64": dict(cfg="T0", n=24, mode="group16", color_float64=True),
    "frames": dict(cfg="T0", n=12, mode="frames"),
    "frames_f64": dict(cfg="T0", n=8, mode="frames", color_float64=True),
    "u16": dict(cfg="T0", n=24, mode="group16", u16=True),
    "u16_frames": dict(cfg="T0", n=6, mode="frames", u16=True),
    "rectify": dict(cfg="T0", n=24, mode="group8", rectify=True),
    "specials": dict(cfg="T0", n=16, mode="group16", specials=True),
    "specials_frames": dict(cfg="T0", n=4, mode="frames", specials=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_replay_equals_integrating_the_images(case):
    c = dict(CASES[case])
    cfg = S.CONFIGS[c.pop("cfg")]
    n, mode = c.pop("n"), c.pop("mode")
    u16, rectify, specials = c.pop("u16", False), c.pop("rectify", False), c.pop("specials", False)
    D, C, T = _frames(cfg.name, n)
    if specials:
        D = np.stack([specials_frame(i, seed=11 + i)[0] for i in range(n)])
    scale = None
    if u16:
        D, scale = np.round(D * 5000.0).astype(np.uint16), np.float32(1.0 / 5000.0)
    T2 = _moved(T)

    def make(store):
        v = _volume(cfg, **c)
        if rectify:
            g = np.load(os.path.join(GOLDEN, "remap_T0.npz"))
            v.set_rectification(g["map1"], g["map2"], swap_rb=True)
        if store:
            v.set_frame_store(n)
        return v

    vol, off, ref = make(True), make(False), make(False)
    slots = _integrate(vol, mode, D, C, cfg.K, T, scale)
    assert np.array_equal(slots, np.arange(n))
    frames, nbytes = vol.frame_store_stats()
    assert frames == n and nbytes >= n * D[0].size * 8
    _integrate(off, mode, D, C, cfg.K, T, scale)
    _same(vol, off)   # the first pass does not depend on the store
    _replay(vol, mode, slots, cfg.K, T2)
    _integrate(ref, mode, D, C, cfg.K, T2, scale)
    _same(vol, ref)
    # a second rebuild from the same store, at the first poses, gives the first map again
    _replay(vol, mode, slots, cfg.K, T)
    _same(vol, off)


def test_replay_grows_the_pool():
    """A growable volume whose replay needs more blocks than the first pass took: the pool overflows and grows during
    the replay, and the map equals a fixed pool's."""
    cfg = S.CONFIGS["T0"]
    D, C, T = _frames("T0", 24)
    T2 = _moved(T, shift=0.6)   # the frames no longer overlap: many more blocks
    vol = _volume(cfg, capacity_blocks=64, max_capacity_blocks=1 << 16)
    vol.set_frame_store(24)
    vol.set_group_size(8)
    vol.integrate_batch(D, C, cfg.K, T)
    slots = vol.last_stored_slots()
    growths0 = vol.capacity()[1]
    vol.reset()
    vol.integrate_stored(slots, cfg.K, T2)
    ref = _volume(cfg, capacity_blocks=1 << 16)
    ref.set_group_size(8)
    ref.integrate_batch(D, C, cfg.K, T2)
    assert vol.capacity()[1] > growths0
    _same(vol, ref)


def test_store_fills_in_the_middle_of_a_call_and_keeps_one_frame_size():
    cfg = S.CONFIGS["T0"]
    D, C, T = _frames("T0", 12)
    vol = _volume(cfg)
    vol.set_frame_store(5)
    vol.set_group_size(4)
    vol.integrate_batch(D[:3], C[:3], cfg.K, T[:3])
    assert list(vol.last_stored_slots()) == [0, 1, 2]
    vol.integrate_batch(D[3:8], C[3:8], cfg.K, T[3:8])
    assert list(vol.last_stored_slots()) == [3, 4, -1, -1, -1]
    frames, nbytes = vol.frame_store_stats()
    assert frames == 5 and nbytes >= 5 * D[0].size * 8
    vol.clear_frame_store()
    assert vol.frame_store_stats() == (0, 0)
    # a frame of another size than the first stored one is not stored
    vol.set_frame_store(3)
    d, c, K, t = crop(cfg, 0, 40, 56)
    vol.integrate(D[0], C[0], cfg.K, T[0])
    vol.integrate(d, c, K, t)
    assert list(vol.last_stored_slots()) == [-1]
    vol.integrate_batch(D[1:3], C[1:3], cfg.K, T[1:3])
    assert list(vol.last_stored_slots()) == [1, 2] and vol.frame_store_stats()[0] == 3
    with pytest.raises(RuntimeError, match="holds no frame"):
        vol.integrate_stored([3], cfg.K, T[:1])
    # the stored frames of both calls, replayed after a reset, against the images at new poses
    T2 = _moved(T[:3])
    vol.reset()
    vol.integrate_stored([0, 1, 2], cfg.K, T2)
    ref = _volume(cfg)
    ref.integrate_batch(D[:3], C[:3], cfg.K, T2)
    _same(vol, ref)
    # reset keeps the store
    assert vol.frame_store_stats()[0] == 3


@pytest.mark.parametrize("limit", [1, 2 << 20])
def test_store_that_cannot_map_stops_and_integration_goes_on(monkeypatch, limit):
    """The store may map at most `limit` bytes (B2V_FRAME_STORE_MAX_BYTES, read at create), as when the device runs
    out of memory: the frames that fit are stored, the others get -1, the store stops, and every call integrates as
    without the store."""
    cfg = S.CONFIGS["T0"]
    D, C, T = _frames("T0", 48)
    monkeypatch.setenv("B2V_FRAME_STORE_MAX_BYTES", str(limit))
    vol = _volume(cfg)
    monkeypatch.delenv("B2V_FRAME_STORE_MAX_BYTES")
    off = _volume(cfg)
    vol.set_frame_store(64)
    slots = []
    for v in (vol, off):
        v.set_group_size(16)
        for a, b in ((0, 8), (8, 48), (0, 4)):
            v.integrate_batch(D[a:b], C[a:b], cfg.K, T[a:b])
            if v is vol:
                slots += list(vol.last_stored_slots())
    frames, nbytes = vol.frame_store_stats()
    pitch = D[0].size * 8
    assert nbytes <= limit and frames == min(48, nbytes // pitch)
    assert slots == list(range(frames)) + [-1] * (52 - frames)
    if limit > 1:
        assert 8 <= frames < 48   # the second call filled the mapped storage and stopped there
    _same(vol, off)
    if frames:
        T2 = _moved(T[:frames])
        vol.reset()
        vol.integrate_stored(np.arange(frames), cfg.K, T2)
        ref = _volume(cfg)
        ref.integrate_batch(D[:frames], C[:frames], cfg.K, T2)
        _same(vol, ref)


def test_failing_call_stores_no_frame():
    """A call that fails after its frames were given slots (here: rectification maps of another size) stores none of
    them; the next call's frames take those slots."""
    cfg = S.CONFIGS["T0"]
    D, C, T = _frames("T0", 4)
    vol = _volume(cfg)
    vol.set_frame_store(8)
    y, x = np.mgrid[:40, :56].astype(np.float32)
    vol.set_rectification(x, y)
    with pytest.raises(RuntimeError, match="different image size"):
        vol.integrate_batch(D[:2], C[:2], cfg.K, T[:2])
    assert list(vol.last_stored_slots()) == [-1, -1] and vol.frame_store_stats()[0] == 0
    vol.set_rectification(None, None)
    vol.integrate_batch(D[:3], C[:3], cfg.K, T[:3])
    assert list(vol.last_stored_slots()) == [0, 1, 2]
    T2 = _moved(T[:3])
    vol.reset()
    vol.integrate_stored([0, 1, 2], cfg.K, T2)
    ref = _volume(cfg)
    ref.integrate_batch(D[:3], C[:3], cfg.K, T2)
    _same(vol, ref)


# ---- plugins ---------------------------------------------------------------------------------------------------------

def _plugin(cfg, store, **kw):
    Cls = P.standalone_integrator_class()
    cam = SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)
    y, x = np.mgrid[:cfg.height, :cfg.width].astype(np.float32)
    return Cls(cam, P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF", calib_maps=(x, y),
               kVolumetricIntegrationVoxelLength=cfg.voxel_size, kVolumetricIntegrationTSdfTrunc=cfg.sdf_trunc,
               kVolumetricIntegrationB200CapacityBlocks=1 << 15, kVolumetricIntegrationB200MaxBatch=16,
               kVolumetricIntegrationB200KeyframeStoreFrames=store, **kw)


def _kd(cfg, i, T):
    d, c, _ = S.render_frame(cfg, i % cfg.n_frames)
    return P.VolumetricIntegrationKeyframeData(id=i, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=d,
                                               timestamp=0.5 * i)


def _rebuild_mesh(integ, cfg, n):
    """Keyframes 0..n-1, then a loop-closure rebuild: RESET and every keyframe again with its corrected pose.  The
    tasks the rebuild sent, and the mesh after it."""
    _, _, T = _frames(cfg.name, n)
    T2 = _moved(T)
    for i in range(n):
        integ.add_keyframe_data(_kd(cfg, i, T[i]))
    integ.run_pending()
    integ.reset()
    for i in range(n):
        integ.add_keyframe_data(_kd(cfg, i, T2[i]))
    sent = list(integ.q_in.queue)
    integ.run_pending()
    m = integ._map_call("mesh")
    return sent, oracle.canonical_mesh(m.vertices, m.vertex_colors, m.edge_ids, m.triangles)


def _same_canon(a, b):
    assert len(a["triangles"]) > 100
    for name in ("edges", "triangles", "vertices", "colors"):
        assert np.array_equal(a[name], b[name]), name


def test_plugin_rebuild_sends_only_poses():
    cfg = S.CONFIGS["T0"]
    results = []
    for store in (0, 64):
        integ = _plugin(cfg, store)
        try:
            results.append(_rebuild_mesh(integ, cfg, 20))
        finally:
            integ.quit()
    (sent_off, mesh_off), (sent_on, mesh_on) = results
    assert not any(keyframe_store.is_stored(t) for t in sent_off)
    assert len(sent_on) == 20 and all(keyframe_store.is_stored(t) for t in sent_on)
    assert all(t.keyframe_data.img is None and t.keyframe_data.depth is None for t in sent_on)
    _same_canon(mesh_on, mesh_off)


@pytest.fixture
def _close_groups(monkeypatch):
    groups = []
    init = shard_plugin.ShardGroup.__init__

    def recorded(self, *a, **k):
        groups.append(self)
        init(self, *a, **k)

    monkeypatch.setattr(shard_plugin.ShardGroup, "__init__", recorded)
    yield
    for g in groups:
        if hasattr(g, "_closed"):
            g.close()


def test_sharded_plugin_rebuild_equals_unsharded(_close_groups):
    """Two ranks sharing device 0 over gloo: each fills its own store with the same slots; the rebuild's stored run
    is one shard op with slots and poses only."""
    cfg = S.CONFIGS["T0"]
    one = _plugin(cfg, 64)
    try:
        sent_one, mesh_one = _rebuild_mesh(one, cfg, 20)
    finally:
        one.quit()
    many = _plugin(cfg, 64, kVolumetricIntegrationB200Devices=[0, 0])
    ops = []
    run = many._shards.run

    def recording(op, meta=None, arrays=None):
        ops.append((op, sorted((arrays or {}).keys())))
        return run(op, meta, arrays)

    many._shards.run = recording
    try:
        sent_many, mesh_many = _rebuild_mesh(many, cfg, 20)
    finally:
        many.quit()
    assert all(keyframe_store.is_stored(t) for t in sent_many + sent_one)
    stored_ops = [o for o in ops if o[0] == "integrate_stored"]
    assert stored_ops and all(arrays == [] for _, arrays in stored_ops)
    _same_canon(mesh_many, mesh_one)
