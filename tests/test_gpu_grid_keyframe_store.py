"""GPU: loop-closure rebuild of the point-average and semantic grids from keyframes held on the GPU (the grids' frame
store: `set_frame_store` / `stage_stored`, b2v_grid.cu, b2v_prep.cu; the grid plugins'
kVolumetricIntegrationB200KeyframeStoreFrames).

A stored frame must stage again bit for bit as `set_frame` staged it, and a rebuild from stored frames must give the
same map as a rebuild from the images: the same staged images through the same association, carve, remap and
integrate calls in the same order."""

import os
from types import SimpleNamespace

import numpy as np
import pytest

from pyslam_b200 import CameraFrustrum, VoxelBlockGrid, VoxelBlockSemanticGrid, VoxelBlockSemanticProbabilisticGrid
from pyslam_b200 import keyframe_store as KS
from pyslam_b200 import shard_plugin
from pyslam_b200 import synthetic as S
from tests import plugin_standins as P
from tests._util import GOLDEN, sort_dump

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
f32 = np.float32
TUM1_D = np.array([0.262383, -0.953104, -0.005358, 0.002628, 1.163314])
SEM_KEYS = ("keys", "count", "pos_sum", "col_sum", "object_id", "class_id", "confidence", "aux", "lab_obj", "lab_cls",
            "lab_logp")
PT_KEYS = ("keys", "count", "pos_sum", "col_sum")


def tum_maps(cfg):
    K = np.array([[cfg.fx, 0, cfg.cx], [0, cfg.fy, cfg.cy], [0, 0, 1]])
    return cv2.initUndistortRectifyMap(K, TUM1_D, None, K, (cfg.width, cfg.height), cv2.CV_32FC1)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == f32 else a


def labels(cfg, i, d):
    cls = S.render_class_ids(cfg, i)
    inst = np.where(cls % 3 == 0, -1, cls * 7 + (np.arange(cls.shape[1])[None, :] // 400)).astype(np.int32)
    inst[d == 0] = 0
    return cls, inst


def _images(fr):
    out = {n: bits(getattr(fr, n).numpy()) for n in ("depth", "filtered_depth", "color")}
    for n in ("class_image", "instance_image"):
        img = getattr(fr, n)
        out[n] = None if img is None else img.numpy()
    out["same_filtered"] = fr.filtered_depth is fr.depth
    return out


def _same_images(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if a[k] is None or isinstance(a[k], bool):
            assert a[k] is b[k] or a[k] == b[k], k
        else:
            assert np.array_equal(a[k], b[k]), k


# ---- round trip ------------------------------------------------------------------------------------------------------

def _edge_depths(d):
    """NaN, +-Inf, -0, 0 and negative depths in the frame (a few pixels of each, and a band for the filter)."""
    d = d.copy()
    flat = d.reshape(-1)
    n = flat.size
    for k, v in enumerate((np.nan, np.inf, -np.inf, -0.0, 0.0, -1.0, -3.5)):
        flat[(k * 97 + 11) % n::max(n // 50, 1)][:7] = v
    flat[n // 2] = np.float32(np.frombuffer(np.uint32(0x7FC12345).tobytes(), f32)[0])   # a NaN payload
    return d


@pytest.mark.parametrize("case", ["T0", "C3", "T0_nomaps", "odd"])
@pytest.mark.parametrize("u16", [False, True])
def test_stored_frames_stage_as_set_frame_staged_them(case, u16):
    rng = np.random.default_rng(3)
    if case == "odd":   # a pixel count that is not a multiple of 4 (the kernels' last partial group)
        H, W = 37, 53
        d = rng.uniform(0.3, 3.0, (H, W)).astype(f32)
        mx = my = None
    else:
        cfg = S.CONFIGS["C3" if case == "C3" else "T0"]
        d = S.render_frame(cfg, 5)[0]
        mx, my = tum_maps(cfg) if case != "T0_nomaps" else (None, None)
    H, W = d.shape
    if not u16:
        d = _edge_depths(d)
    depth = np.round(np.nan_to_num(d, nan=0, posinf=0, neginf=0).clip(0) * 5000).astype(np.uint16) if u16 else d
    scale = f32(1 / 5000) if u16 else None
    bgr = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    cls = rng.integers(-2, 20, (H, W)).astype(np.int32)
    inst = rng.integers(-3, 2 ** 31 - 1, (H, W)).astype(np.int32)
    sem = VoxelBlockSemanticGrid(0.05, 8, capacity_blocks=64)
    pt = VoxelBlockGrid(0.05, 8, capacity_blocks=64)
    for g in (sem, pt):
        g.set_frame_store(16)
        if mx is not None:
            g.set_rectification(mx, my, swap_rb=True)
    staged = {}
    for flt in (True, False):
        for lab in ("none", "class", "both"):
            cl = cls if lab != "none" else None
            ins = inst if lab == "both" else None
            fr = sem.set_frame(depth, bgr, cl, ins, depth_scale=scale, filter_shadow_points=flt)
            staged[("sem", sem.last_stored_slot())] = _images(fr)
        fr = pt.set_frame(depth, bgr, depth_scale=scale, filter_shadow_points=flt)
        staged[("pt", pt.last_stored_slot())] = _images(fr)
    assert sem.frame_store_stats()[0] == 6 and pt.frame_store_stats()[0] == 2
    assert sorted(s for k, s in staged if k == "sem") == list(range(6))
    if not u16:
        filtered = staged[("pt", 0)]["filtered_depth"]
        assert (filtered == np.float32(-1).view(np.uint32)).any()   # the filter set pixels
    for (kind, slot), want in staged.items():
        g = sem if kind == "sem" else pt
        _same_images(_images(g.stage_stored(slot)), want)
    # per-frame store sizes: 8 / 16 bytes per pixel
    pitch = lambda b: -(-H * W // 4) * 4 * b
    assert pt.frame_store_stats()[1] >= 2 * pitch(8) and sem.frame_store_stats()[1] >= 6 * pitch(16)
    sem.close()
    pt.close()


# ---- replay == images ------------------------------------------------------------------------------------------------

def _c3_frames(n=4, stride=12):
    cfg = S.CONFIGS["C3"]
    out = []
    for i in range(0, n * stride, stride):
        d, c, T = S.render_frame(cfg, i)
        cls, inst = labels(cfg, i, d)
        out.append((np.round(d * 5000).astype(np.uint16), np.ascontiguousarray(c[..., ::-1]), cls, inst, T))
    return cfg, out


def _moved(T, k):
    """A loop-closure correction: the pose shifted by a few centimetres."""
    M = np.eye(4)
    M[:3, 3] = [0.01 * (k % 3), -0.02, 0.015 * (k % 2)]
    return np.asarray(T) @ M


def _semantic_body(grid, cfg, fr, T, assoc, carve):
    """One keyframe of the semantic plugin's loop body on a staged frame; (instance map, object image) or None."""
    cf = CameraFrustrum(cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.width, cfg.height, T, depth_max=8.0, depth_min=1e-2)
    m, obj = None, None
    if assoc and fr.instance_image is not None:
        m = grid.assign_object_ids_to_instance_ids(cf, fr.class_image, fr.instance_image, fr.filtered_depth,
                                                   depth_threshold=0.05, do_carving=carve, min_vote_ratio=0.5,
                                                   min_votes=3)
        obj = grid.remap_instance_ids()
    elif carve:
        grid.carve(cf, fr.filtered_depth, 0.05)
    grid.integrate_rgbd(fr.filtered_depth, fr.color, cfg.K, np.linalg.inv(T), fr.class_image, obj,
                        max_depth=cfg.depth_trunc, filter_shadow_points=False)
    return m, None if obj is None else obj.numpy()


def _sem_state(grid, per_frame):
    return (sort_dump(grid.dump_blocks(8)), grid.label_overflows(), grid.get_next_object_id(), per_frame)


@pytest.mark.parametrize("tag,overflow", [("vote", 0), ("prob", 0), ("prob", 1 << 16)])
@pytest.mark.parametrize("assoc,carve", [(True, True), (True, False), (False, True)])
def test_semantic_rebuild_from_store_equals_rebuild_from_images(tag, overflow, assoc, carve):
    cfg, frames = _c3_frames()
    mx, my = tum_maps(cfg)
    grid_t = VoxelBlockSemanticGrid if tag == "vote" else VoxelBlockSemanticProbabilisticGrid
    kw = dict(max_label_overflow_pairs=overflow) if tag == "prob" else {}
    # capacity 4 blocks: both rebuilds grow their storage during the replay
    grids = [grid_t(0.015, 8, capacity_blocks=4, max_capacity_blocks=1 << 15, **kw) for _ in range(2)]
    for g in grids:
        g.set_depth_threshold(1.5)
        g.set_rectification(mx, my, swap_rb=True)
    stored, img = grids
    stored.set_frame_store(len(frames))
    slots = []
    for k, (d16, bgr, cls, inst, T) in enumerate(frames):   # first integration, both grids from images
        for g in grids:
            fr = g.set_frame(d16, bgr, cls, inst if k % 2 == 0 else None, depth_scale=f32(1 / 5000),
                             filter_shadow_points=True)
            _semantic_body(g, cfg, fr, T, assoc, carve)
        slots.append(stored.last_stored_slot())
    assert slots == list(range(len(frames)))
    for g in grids:
        g.clear()
    for k, (d16, bgr, cls, inst, T) in enumerate(frames):   # rebuild with corrected poses
        Tm = _moved(T, k)
        fa = stored.stage_stored(slots[k])
        fb = img.set_frame(d16, bgr, cls, inst if k % 2 == 0 else None, depth_scale=f32(1 / 5000),
                           filter_shadow_points=True)
        a = _semantic_body(stored, cfg, fa, Tm, assoc, carve)
        b = _semantic_body(img, cfg, fb, Tm, assoc, carve)
        sa, sb = _sem_state(stored, a), _sem_state(img, b)
        for key in SEM_KEYS:
            assert np.array_equal(sa[0][key], sb[0][key]), (k, key)
        assert sa[1:3] == sb[1:3]
        assert sa[3][0] == sb[3][0] and (sa[3][1] is None) == (sb[3][1] is None)
        if sa[3][1] is not None:
            assert np.array_equal(sa[3][1], sb[3][1])
    assert len(sa[0]["keys"]) > 500 and stored.capacity()[1] >= 2
    for g in grids:
        g.close()


@pytest.mark.parametrize("input_order", [True, False])
@pytest.mark.parametrize("shards", [1, 2, 3])
def test_point_grid_rebuild_from_store_equals_rebuild_from_images(input_order, shards):
    """Carve with the unfiltered depth, integrate the filtered one; input-order sums bit for bit, the default mode's
    float atomics keys and counts exactly.  Every shard rank stages the same frames into the same slots."""
    cfg = S.CONFIGS["C2"]
    mx, my = tum_maps(cfg)
    frames = [S.render_frame(cfg, i) for i in (0, 10, 20, 30)]

    def make():
        out = []
        for r in range(shards):
            g = VoxelBlockGrid(0.03, 8, capacity_blocks=4, max_capacity_blocks=1 << 14, input_order_sums=input_order,
                               shard_rank=r, shard_count=shards)
            g.set_rectification(mx, my, swap_rb=True)
            out.append(g)
        return out

    def body(g, fr, T):
        cf = CameraFrustrum(cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.width, cfg.height, T, depth_max=8.0, depth_min=1e-2)
        g.carve(cf, fr.depth, 3e-2)
        g.integrate_rgbd(fr.filtered_depth, fr.color, cfg.K, np.linalg.inv(T), max_depth=4.0)

    stored, img = make(), make()
    for g in stored:
        g.set_frame_store(8)
    slots = []
    for d, c, T in frames:
        bgr = np.ascontiguousarray(c[..., ::-1])
        for g in stored + img:
            body(g, g.set_frame(d, bgr, filter_shadow_points=True), T)
        ranks = {g.last_stored_slot() for g in stored}
        assert len(ranks) == 1
        slots.append(ranks.pop())
    for g in stored + img:
        g.clear()
    for k, (d, c, T) in enumerate(frames):
        Tm = _moved(T, k)
        bgr = np.ascontiguousarray(c[..., ::-1])
        for a, b in zip(stored, img):
            body(a, a.stage_stored(slots[k]), Tm)
            body(b, b.set_frame(d, bgr, filter_shadow_points=True), Tm)
            da, db = sort_dump(a.dump_blocks()), sort_dump(b.dump_blocks())
            for key in (PT_KEYS if input_order else ("keys", "count")):
                assert np.array_equal(da[key], db[key]), (k, key)
            if not input_order:
                assert np.allclose(da["pos_sum"], db["pos_sum"], rtol=1e-5, atol=1e-6)
    assert sum(g.num_blocks() for g in stored) > 100
    for g in stored + img:
        g.close()


# ---- store edge cases ------------------------------------------------------------------------------------------------

def test_store_edge_cases(tmp_path):
    cfg = S.CONFIGS["T0"]
    frames = [S.render_frame(cfg, i) for i in range(3)]
    g = VoxelBlockSemanticGrid(0.02, 8, capacity_blocks=1024)
    assert g.last_stored_slot() == -1 and g.frame_store_stats() == (0, 0)
    d, c, T = frames[0]
    g.set_frame(d, c)
    assert g.last_stored_slot() == -1   # store off
    g.set_frame_store(8)
    cls = np.ones(d.shape, np.int32)
    g.set_frame(d, c, cls)
    assert g.last_stored_slot() == 0
    g.set_frame(np.zeros((10, 12), f32), np.zeros((10, 12, 3), np.uint8))
    assert g.last_stored_slot() == -1   # another size
    g.set_frame(frames[1][0], frames[1][1])
    assert g.last_stored_slot() == 1
    # a failing set_frame stores nothing
    g.set_rectification(*np.mgrid[:5, :5].astype(f32)[::-1])
    with pytest.raises(RuntimeError):
        g.set_frame(d, c)
    assert g.last_stored_slot() == -1 and g.frame_store_stats()[0] == 2
    g.set_rectification(None, None)
    # clear() and load_state keep the store
    g.integrate_rgbd(d, c, cfg.K, np.linalg.inv(T), cls)
    g.save_state(str(tmp_path / "s.npz"))
    g.clear()
    g.load_state(str(tmp_path / "s.npz"))
    assert g.frame_store_stats()[0] == 2
    fr = g.stage_stored(0)
    assert np.array_equal(fr.class_image.numpy(), cls) and np.array_equal(fr.depth.numpy(), d)
    # a bad slot leaves the staged frame as it was
    before = _images(fr)
    for bad in (-1, 2, 99):
        with pytest.raises(RuntimeError, match="holds no frame"):
            g.stage_stored(bad)
    _same_images(_images(fr), before)
    g.clear_frame_store()
    assert g.frame_store_stats() == (0, 0)
    g.close()


@pytest.mark.parametrize("limit", [1, 2 << 20])
def test_store_that_cannot_map_stops_and_set_frame_goes_on(monkeypatch, limit):
    monkeypatch.setenv("B2V_FRAME_STORE_MAX_BYTES", str(limit))
    cfg = S.CONFIGS["C1"]
    d, c, T = S.render_frame(cfg, 0)
    g = VoxelBlockGrid(0.02, 8, capacity_blocks=1 << 12)
    g.set_frame_store(100)
    fit = limit // (cfg.width * cfg.height * 8)   # 614 KB per 320x240 frame
    got = []
    for k in range(fit + 2):
        fr = g.set_frame(d, c, filter_shadow_points=True)
        got.append(g.last_stored_slot())
        g.integrate_rgbd(fr.filtered_depth, fr.color, cfg.K, np.linalg.inv(T), max_depth=4.0)
    assert got == list(range(fit)) + [-1, -1]
    assert g.frame_store_stats()[0] == fit and g.num_blocks() > 0
    g.close()


# ---- plugins ---------------------------------------------------------------------------------------------------------

class RectifyingBase(P.StandaloneIntegratorBase):
    """The base class's host preparation in full (base.py:1007-1054), including the label images."""

    def estimate_depth_if_needed_and_rectify(self, kd):
        depth = kd.depth.astype(f32) if kd.depth.dtype != f32 else kd.depth
        color, cls, inst = kd.img, kd.semantic_img, kd.semantic_instances_img
        if self.calib_map1 is not None:
            m1, m2 = self.calib_map1, self.calib_map2
            color = cv2.remap(color, m1, m2, interpolation=cv2.INTER_LINEAR)
            depth = cv2.remap(depth, m1, m2, interpolation=cv2.INTER_NEAREST)
            cls = None if cls is None else cv2.remap(cls, m1, m2, interpolation=cv2.INTER_NEAREST)
            inst = None if inst is None else cv2.remap(inst, m1, m2, interpolation=cv2.INTER_NEAREST)
        return np.ascontiguousarray(color[..., ::-1]), depth, None, cls, inst


def _plugin(kind, gpu, store, **kw):
    from pyslam_b200 import integrator_semantic as IS
    make = IS.make_semantic_integrator_class if kind != "voxel" else IS.make_voxel_grid_integrator_class
    g = np.load(os.path.join(GOLDEN, "remap_T0.npz"))
    cfg = S.CONFIGS["T0"]
    cam = SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)
    if kind == "prob":
        kw["use_semantic_probabilistic"] = True
    return make(RectifyingBase, P.API)(
        cam, P.DatasetEnvironmentType.INDOOR, None, "B200", calib_maps=(g["map1"], g["map2"]),
        kVolumetricIntegrationB200GpuRectify=gpu, kVolumetricIntegrationB200KeyframeStoreFrames=store,
        kVolumetricIntegrationVoxelLength=0.02, kVolumetricIntegrationVoxelGridUseCarving=True,
        kVolumetricIntegrationVoxelGridCarvingDepthThreshold=0.08, kVolumetricIntegrationB200CapacityBlocks=1024,
        kVolumetricIntegrationVoxelGridMinCount=1, **kw)


def _keyframes(moved):
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    out = []
    for i in range(int(g["n_frames"])):
        T = _moved(g[f"Tcw_{i}"], i) if moved else g[f"Tcw_{i}"]
        out.append(P.VolumetricIntegrationKeyframeData(
            id=i, pose=T, img=np.ascontiguousarray(g[f"color_{i}"][..., ::-1]), depth=g[f"depth_{i}"],
            semantic_img=g[f"class_image_{i}"], semantic_instances_img=g[f"instance_image_{i}"],
            timestamp=0.1 * i))
    return out


def _output(integ):
    integ.add_update_output_task()
    integ.step()
    out = None
    while (o := integ.pop_output()) is not None:
        out = o
    return out


def _rebuild(integ, light_expected):
    """Integrate the keyframes, then rebuild(map): RESET and every keyframe again with a corrected pose.  Returns the
    output after the rebuild."""
    for kd in _keyframes(False):
        integ.add_keyframe_data(kd)
        integ.step()
    integ.reset()
    for kd in _keyframes(True):
        integ.add_keyframe_data(kd)
    sent = []
    while not integ.q_in.empty():
        sent.append(integ.q_in.get())
    assert all(KS.is_stored(t) == light_expected for t in sent)
    if light_expected:
        assert all(getattr(t.keyframe_data, n) is None for t in sent for n in KS.IMAGE_FIELDS)
    for t in sent:
        integ.q_in.put(t)
        integ.step()
    return _output(integ)


def _same_plugin_output(kind, a, b):
    if kind == "voxel":
        pa, pb = a.point_cloud, b.point_cloud
        assert len(pa.points) > 100
        rows = [np.concatenate([p.points, p.colors], 1) for p in (pa, pb)]
        assert np.array_equal(*(r[np.lexsort(r.T[::-1])] for r in rows))
        return
    la, lb = a.objects.object_list, b.objects.object_list
    assert len(la) == len(lb) > 0
    for x, y in zip(la, lb):
        assert (x.object_id, x.class_id) == (y.object_id, y.class_id)
        rows = [np.concatenate([o.points, o.colors], 1) for o in (x, y)]
        assert np.array_equal(*(q[np.lexsort(q.T[::-1])] for q in rows))


@pytest.mark.parametrize("kind", ["voxel", "vote", "prob"])
@pytest.mark.parametrize("gpu", [True, False])
def test_plugins_rebuild_from_light_tasks_equal_store_off(kind, gpu):
    """Raw path (maps on the device) and host path (the base class prepares the frames): with the store on, the
    rebuild sends only light tasks and its output equals the store-off plugin's."""
    kw = dict(kVolumetricIntegrationB200InputOrderSums=True) if kind == "voxel" else {}
    on, off = _plugin(kind, gpu, 16, **kw), _plugin(kind, gpu, 0, **kw)
    assert on._gpu_rectify == gpu
    a, b = _rebuild(on, True), _rebuild(off, False)
    _same_plugin_output(kind, a, b)
    if kind != "voxel":
        assert on.last_instance_map == off.last_instance_map
    assert on.volume.frame_store_stats()[0] == len(_keyframes(False))
    on.quit()
    off.quit()


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


@pytest.mark.parametrize("kind", ["voxel", "prob"])
def test_sharded_plugin_rebuild_from_store_equals_unsharded(kind, _close_groups):
    kw = dict(kVolumetricIntegrationB200InputOrderSums=True) if kind == "voxel" else {}
    sharded = _plugin(kind, True, 16, kVolumetricIntegrationB200Devices=[0, 0], **kw)
    single = _plugin(kind, True, 0, **kw)
    a, b = _rebuild(sharded, True), _rebuild(single, False)
    _same_plugin_output(kind, a, b)
    sharded.quit()
    single.quit()


def _workers_capped(monkeypatch, limit):
    """The shard workers' frame stores may map at most `limit` bytes (B2V_FRAME_STORE_MAX_BYTES in their environment);
    rank 0's is not capped."""
    init = shard_plugin.ShardGroup.__init__

    def capped(self, *a, **k):
        os.environ["B2V_FRAME_STORE_MAX_BYTES"] = str(limit)
        try:
            init(self, *a, **k)
        finally:
            del os.environ["B2V_FRAME_STORE_MAX_BYTES"]

    monkeypatch.setattr(shard_plugin.ShardGroup, "__init__", capped)


@pytest.mark.parametrize("kind", ["voxel", "prob"])
def test_sharded_plugin_publishes_only_slots_every_rank_stored(kind, _close_groups, monkeypatch):
    """A worker's store stops (it cannot map) while rank 0's keeps storing: no slot is published, the rebuild sends
    every keyframe with its images, and its output equals the unsharded store-off plugin's."""
    _workers_capped(monkeypatch, 1)
    kw = dict(kVolumetricIntegrationB200InputOrderSums=True) if kind == "voxel" else {}
    sharded = _plugin(kind, True, 16, kVolumetricIntegrationB200Devices=[0, 0], **kw)
    single = _plugin(kind, True, 0, **kw)
    a, b = _rebuild(sharded, False), _rebuild(single, False)
    _same_plugin_output(kind, a, b)
    assert sharded.volume.frame_store_stats()[0] >= len(_keyframes(False)) and sharded._stored_slots == {}
    sharded.quit()
    single.quit()


def test_sharded_tsdf_plugin_publishes_only_slots_every_rank_stored(_close_groups, monkeypatch):
    from tests import test_gpu_keyframe_store as TK
    _workers_capped(monkeypatch, 1)
    cfg = S.CONFIGS["T0"]
    many = TK._plugin(cfg, 64, kVolumetricIntegrationB200Devices=[0, 0])
    try:
        sent_many, mesh_many = TK._rebuild_mesh(many, cfg, 20)
        assert many.volume.frame_store_stats()[0] == 40 and many._stored_slots == {}
    finally:
        many.quit()
    one = TK._plugin(cfg, 0)
    try:
        sent_one, mesh_one = TK._rebuild_mesh(one, cfg, 20)
    finally:
        one.quit()
    assert not any(KS.is_stored(t) for t in sent_many + sent_one)
    TK._same_canon(mesh_many, mesh_one)
