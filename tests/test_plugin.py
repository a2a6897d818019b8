"""Host logic of the plugin adapter (CPU, with a fake volume) and the same flow on the GPU."""

import os
from types import SimpleNamespace

import numpy as np
import pytest

from pyslam_b200 import integrator as I
from tests import plugin_standins as P
from pyslam_b200 import synthetic as S


class _FakeVolume:
    """Records calls; stands in for B200TsdfVolume so the queue / task logic runs on CPU."""

    def __init__(self, **kw):
        self.kw = kw
        self.calls = []
        self.closed = False

    def integrate_batch(self, depths, colors, K, poses, depth_scale=None):
        assert colors.dtype == np.uint8 and depths.shape[0] == colors.shape[0] == poses.shape[0]
        assert depths.dtype == np.float32 or (depth_scale and depths.dtype == np.uint16)
        self.calls.append(("integrate_batch", tuple(K), np.asarray(poses).copy(), int(depths.shape[0]),
                           colors[0, 0, 0].copy()))
        self.last_depth, self.last_scale = depths, depth_scale

    def reset(self):
        self.calls.append(("reset",))

    def extract_triangle_mesh(self):
        self.calls.append(("mesh",))
        return SimpleNamespace(vertices=np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float64),
                               triangles=np.array([[0, 1, 2]], np.int32),
                               vertex_colors=np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float64),
                               vertex_normals=np.zeros((0, 3)))

    def extract_point_cloud(self):
        self.calls.append(("points",))
        return SimpleNamespace(points=np.zeros((2, 3)), colors=np.ones((2, 3)))

    def close(self):
        self.closed = True


def _camera(cfg):
    return SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width,
                           height=cfg.height, D=None)


def test_adapter_task_flow_with_fake_volume_one_frame_batches(monkeypatch, tmp_path):
    monkeypatch.setattr(I, "B200TsdfVolume", _FakeVolume)
    Cls = P.standalone_integrator_class()
    cfg = S.CONFIGS["T0"]
    integ = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF",
                kVolumetricIntegrationVoxelLength=0.02)
    assert integ.volume.kw["voxel_length"] == 0.02 and integ.volume.kw["depth_trunc"] == 4.0
    d, c, T = S.render_frame(cfg, 0)
    bgr = np.ascontiguousarray(c[..., ::-1])
    kd = P.VolumetricIntegrationKeyframeData(id=7, pose=T, img=bgr, depth=(d * 1000).astype(np.uint16))
    integ.add_keyframe_data(kd)
    integ.step()
    name, K, poses, n, px = integ.volume.calls[0]
    assert name == "integrate_batch" and n == 1 and K == (cfg.fx, cfg.fy, cfg.cx, cfg.cy)
    assert np.array_equal(poses[0], T)
    assert np.array_equal(px, c[0, 0])  # BGR -> RGB before the volume sees it (base.py:1054)
    out = integ.pop_output()             # first integrate always produces an output
    assert out.id == 7 and out.mesh.triangles.shape == (1, 3) and out.point_cloud is None
    # a second frame inside the output interval integrates but does not extract
    integ.add_keyframe_data(kd)
    integ.step()
    assert integ.pop_output() is None and integ.volume.calls[-1][0] == "integrate_batch"
    assert integ.volume.calls[-1][3] == 1
    # UPDATE_OUTPUT forces an extraction
    integ.add_update_output_task()
    integ.step()
    assert integ.pop_output().task_type == P.VolumetricIntegrationTaskType.UPDATE_OUTPUT
    # SAVE writes dense_map.ply and signals completion
    integ.save(str(tmp_path))
    integ.step()
    assert integ.save_request_completed.value == 1
    ply = open(os.path.join(tmp_path, "dense_map.ply"), "rb").read()
    assert ply.startswith(b"ply\nformat binary_little_endian 1.0\nelement vertex 3\n")
    assert b"element face 1\n" in ply and len(ply.split(b"end_header\n", 1)[1]) == 3 * 15 + 13
    # RESET arrives on the management queue and is honoured before the next task
    integ.reset()
    integ.add_update_output_task()
    integ.step()
    assert ("reset",) in integ.volume.calls
    # exceptions inside a task are logged and do not kill the loop (tsdf.py:303-307)
    integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(id=9, pose=T, img=bgr[:3], depth=d))
    monkeypatch.setattr(_FakeVolume, "integrate_batch", lambda *a, **k: (_ for _ in ()).throw(RuntimeError("x")))
    integ.step()
    assert integ.is_running.value == 1
    integ.add_task(None)
    integ.step()
    assert integ.is_running.value == 0
    integ.quit()
    assert integ.volume.closed


def test_backlog_is_drained_into_one_fused_batch_lone_frames_into_one_frame_batches(monkeypatch):
    """rebuild(map) re-enqueues every keyframe (base.py:1242-1318): consecutive INTEGRATE tasks already in the queue
    go to ONE integrate_batch call (bounded); a task of another type met while draining is handled by the next
    call, in order; output cadence and RESET semantics are unchanged."""
    monkeypatch.setattr(I, "B200TsdfVolume", _FakeVolume)
    Cls = P.standalone_integrator_class()
    cfg = S.CONFIGS["T0"]
    integ = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF",
                kVolumetricIntegrationB200MaxBatch=4)
    d, c, T = S.render_frame(cfg, 0)
    bgr = np.ascontiguousarray(c[..., ::-1])
    poses = []
    for i in range(6):
        Ti = T.copy()
        Ti[0, 3] += 0.01 * i
        poses.append(Ti)
        integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(id=i, pose=Ti, img=bgr, depth=d))
    integ.add_update_output_task()
    integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(id=6, pose=T, img=bgr, depth=d))
    integ.step()                                   # frames 0..3 (bounded by MaxBatch) in one call
    name, K, P4, n, _ = integ.volume.calls[0]
    assert name == "integrate_batch" and n == 4 and np.array_equal(P4, np.stack(poses[:4]))
    assert integ.pop_output().id == 3              # the first output carries the last integrated id
    integ.step()                                   # frames 4, 5; the UPDATE_OUTPUT task is met and deferred
    assert integ.volume.calls[-1][0] == "integrate_batch" and integ.volume.calls[-1][3] == 2
    assert integ.pop_output() is None              # inside the output interval
    integ.step()                                   # the deferred UPDATE_OUTPUT, before frame 6
    assert integ.pop_output().task_type == P.VolumetricIntegrationTaskType.UPDATE_OUTPUT
    assert [cl[0] for cl in integ.volume.calls if cl[0].startswith("integrate")] == ["integrate_batch"] * 2
    integ.step()                                   # frame 6 alone: the single-frame call
    assert integ.volume.calls[-1][0] == "integrate_batch" and integ.volume.calls[-1][3] == 1
    assert integ.integrated_frames == 7
    # MaxBatch = 1 restores one task per call
    integ2 = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF", kVolumetricIntegrationB200MaxBatch=1)
    for i in range(3):
        integ2.add_keyframe_data(P.VolumetricIntegrationKeyframeData(id=i, pose=T, img=bgr, depth=d))
    integ2.run_pending()
    assert [(cl[0], cl[3]) for cl in integ2.volume.calls
            if cl[0].startswith("integrate")] == [("integrate_batch", 1)] * 3


def test_outdoor_depth_trunc_and_point_cloud_mode(monkeypatch):
    monkeypatch.setattr(I, "B200TsdfVolume", _FakeVolume)
    Cls = P.standalone_integrator_class()
    cfg = S.CONFIGS["T0"]
    integ = Cls(_camera(cfg), P.DatasetEnvironmentType.OUTDOOR, None, "B200_TSDF",
                kVolumetricIntegrationTsdfExtractMesh=False)
    assert integ.volume.kw["depth_trunc"] == 10.0
    integ.add_update_output_task()
    integ.step()
    out = integ.pop_output()
    assert out.mesh is None and out.point_cloud.points.shape == (2, 3)


@pytest.mark.gpu
def test_adapter_end_to_end_on_gpu(tmp_path):
    import oracle
    Cls = P.standalone_integrator_class()
    cfg = S.CONFIGS["T0"]
    integ = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF",
                kVolumetricIntegrationVoxelLength=cfg.voxel_size,
                kVolumetricIntegrationTSdfTrunc=cfg.sdf_trunc,
                kVolumetricIntegrationB200CapacityBlocks=4096)
    orc = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, 4.0)
    for i in range(3):
        d, c, T = S.render_frame(cfg, i)
        integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(
            id=i, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=d))
        orc.integrate(d, c, cfg.K, T)
    integ.run_pending()
    integ.add_update_output_task()
    integ.step()
    out = None
    while True:
        o = integ.pop_output()
        if o is None:
            break
        out = o
    ref = orc.extract_mesh()
    assert out.mesh.vertices.shape == ref["vertices"].shape
    assert out.mesh.triangles.shape == ref["triangles"].shape
    integ.save(str(tmp_path))
    integ.step()
    assert os.path.getsize(os.path.join(tmp_path, "dense_map.ply")) > 15 * len(ref["vertices"])
    integ.quit()


def test_adapter_gpu_rectification_hands_raw_frames_to_the_volume_as_one_frame_batches(monkeypatch):
    """With calibration maps the adapter installs them on the volume (swap_rb=True) and passes the RAW BGR
    image and float32 depth; with the option off it goes through the base class's CPU remap."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "remap_T0.npz"))

    class _RectVolume(_FakeVolume):
        def set_rectification(self, m1, m2, swap_rb=False):
            self.calls.append(("rect", m1.shape, bool(swap_rb)))

    monkeypatch.setattr(I, "B200TsdfVolume", _RectVolume)
    Cls = P.standalone_integrator_class()
    cfg = S.CONFIGS["T0"]
    integ = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF",
                calib_maps=(g["map1"], g["map2"]))
    assert integ.volume.calls[0] == ("rect", g["map1"].shape, True)
    kd = P.VolumetricIntegrationKeyframeData(id=1, pose=g["Tcw"], img=g["bgr"], depth=g["depth"])
    integ.add_keyframe_data(kd)
    integ.step()
    call = [c for c in integ.volume.calls if c[0] == "integrate_batch" and c[3] == 1][-1]
    assert np.array_equal(call[4], g["bgr"][0, 0])   # raw BGR, untouched
    # raw uint16 depth: python core -> depth.astype(float32) on the host; C++ core (USE_CPP) -> the uint16 image goes
    # to the GPU with depth_scale = camera.depth_factor (base.py:1007-1015 multiplies by self.camera.depth_factor)
    raw16 = np.round(g["depth"] * 5000.0).astype(np.uint16)
    integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(id=2, pose=g["Tcw"], img=g["bgr"], depth=raw16))
    integ.step()
    assert integ.volume.last_depth[0].dtype == np.float32 and integ.volume.last_scale is None
    assert np.array_equal(integ.volume.last_depth[0], raw16.astype(np.float32))
    api_cpp = SimpleNamespace(**{**vars(P.API), "USE_CPP": True})
    ClsCpp = I.make_integrator_class(P.StandaloneIntegratorBase, api_cpp)
    cam = _camera(cfg)
    cam.depth_factor = 1.0 / 5000.0
    integ_cpp = ClsCpp(cam, P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF", calib_maps=(g["map1"], g["map2"]))
    integ_cpp.add_keyframe_data(P.VolumetricIntegrationKeyframeData(id=3, pose=g["Tcw"], img=g["bgr"], depth=raw16))
    integ_cpp.step()
    assert integ_cpp.volume.last_depth[0].dtype == np.uint16 and integ_cpp.volume.last_scale == np.float32(1.0 / 5000.0)
    cv2 = pytest.importorskip("cv2")
    del cv2
    integ2 = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF",
                 calib_maps=(g["map1"], g["map2"]), kVolumetricIntegrationB200GpuRectify=False)
    assert not any(c[0] == "rect" for c in integ2.volume.calls)
    integ2.add_keyframe_data(kd)
    integ2.step()
    call = [c for c in integ2.volume.calls if c[0] == "integrate_batch" and c[3] == 1][-1]
    assert np.array_equal(call[4], g["rgb_u"][0, 0])  # CPU-rectified RGB


@pytest.mark.gpu
def test_adapter_gpu_rectification_equals_cpu_rectification():
    pytest.importorskip("cv2")
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "remap_T0.npz"))
    Cls = P.standalone_integrator_class()
    cfg = S.CONFIGS["T0"]
    nk = g["new_K"]
    cam = SimpleNamespace(fx=float(nk[0, 0]), fy=float(nk[1, 1]), cx=float(nk[0, 2]), cy=float(nk[1, 2]),
                          width=cfg.width, height=cfg.height, D=None)
    dumps = []
    for gpu_rect in (True, False):
        integ = Cls(cam, P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF",
                    calib_maps=(g["map1"], g["map2"]), kVolumetricIntegrationB200GpuRectify=gpu_rect,
                    kVolumetricIntegrationVoxelLength=cfg.voxel_size,
                    kVolumetricIntegrationTSdfTrunc=cfg.sdf_trunc,
                    kVolumetricIntegrationB200CapacityBlocks=4096)
        for i in range(4):
            d, c, T = S.render_frame(cfg, i)
            integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(
                id=i, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=d))
        integ.run_pending()
        from tests._util import sort_dump
        dumps.append(sort_dump(integ.volume.dump_blocks()))
        integ.quit()
    assert len(dumps[0]["keys"]) > 20
    assert np.array_equal(dumps[0]["keys"], dumps[1]["keys"])
    assert np.array_equal(dumps[0]["vox"], dumps[1]["vox"])


# ---- semantic backend ------------------------------------------------------------------------------------------
class _FakeSemanticGrid:
    def __init__(self, **kw):
        self.kw = kw
        self.calls = []

    def set_depth_threshold(self, v):
        self.calls.append(("thr", v))

    def set_depth_decay_rate(self, v):
        self.calls.append(("rate", v))

    def assign_object_ids_to_instance_ids(self, fr, cls, inst, depth, **kw):
        self.calls.append(("assign", np.asarray(fr.T_cw).copy(), kw))
        return {0: 0, 7: 3, 9: -1}

    def carve(self, fr, depth, thr):
        self.calls.append(("carve", thr))

    def integrate_rgbd(self, depth, color, K, Twc, class_image=None, object_image=None, **kw):
        self.calls.append(("rgbd", tuple(K), np.asarray(Twc).copy(), None if object_image is None else
                           object_image.copy(), kw))

    def get_voxels(self, min_count=1, min_confidence=0.0):
        self.calls.append(("voxels", min_count, min_confidence))
        return SimpleNamespace(points=np.zeros((2, 3)), colors=np.ones((2, 3), np.float32),
                               class_ids=np.array([1, 2], np.int32), object_ids=np.array([3, -1], np.int32),
                               confidences=np.ones(2, np.float32))

    def get_object_segments(self, min_count=1, min_confidence=0.0):
        from pyslam_b200.volume import ObjectData, ObjectDataGroup
        self.calls.append(("objects", min_count, min_confidence))
        pts = np.array([[0.0, 0, 0], [1.0, 0, 0], [0, 2.0, 0], [0, 0, 3.0]])
        return ObjectDataGroup([ObjectData(3, 1, pts, np.ones((4, 3), np.float32), 0.7, 0.9)])

    def reset(self):
        self.calls.append(("reset",))

    def close(self):
        self.calls.append(("close",))


def test_semantic_adapter_flow_with_fake_grid(monkeypatch, tmp_path):
    from pyslam_b200 import integrator_semantic as IS
    monkeypatch.setattr(IS, "VoxelBlockSemanticGrid", _FakeSemanticGrid)
    monkeypatch.setattr(IS, "VoxelBlockSemanticProbabilisticGrid", _FakeSemanticGrid)
    monkeypatch.setattr(IS, "filter_shadow_points", lambda d: d)
    Cls = P.standalone_semantic_integrator_class()
    cfg = S.CONFIGS["T0"]
    integ = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_SEMANTIC",
                use_semantic_probabilistic=True, kVolumetricIntegrationVoxelGridUseCarving=True)
    assert integ.volume.calls[:2] == [("thr", 5.0), ("rate", 0.1)]          # indoor defaults (config :370-375)
    d, c, T = S.render_frame(cfg, 0)
    inst = np.full(d.shape, 7, np.int32)
    inst[:, :10] = 9
    inst[:, 10:20] = 0
    kd = P.VolumetricIntegrationKeyframeData(id=3, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=d,
                                             semantic_img=np.ones(d.shape, np.int32), semantic_instances_img=inst)
    integ.add_keyframe_data(kd)
    integ.step()
    names = [x[0] for x in integ.volume.calls]
    assert "assign" in names and "carve" not in names                        # carving rides on the association
    rgbd = [x for x in integ.volume.calls if x[0] == "rgbd"][0]
    assert np.allclose(rgbd[2] @ T, np.eye(4), atol=1e-9)                    # Twc = inv(Tcw)
    assert set(np.unique(rgbd[3])) == {-1, 0, 3}                             # instance ids remapped to object ids
    assert rgbd[4]["filter_shadow_points"] is True and rgbd[4]["use_depths"] is True
    # instance ids were integrated -> the reference's OBJECTS representation (semantic_grid.py:523-587)
    out = integ.pop_output()
    assert out.point_cloud is None and out.objects.num_objects == 1 and ("objects", 3, 0.6) in integ.volume.calls
    o = out.objects.object_list[0]
    assert (o.object_id, o.class_id) == (3, 1) and o.points.shape == (4, 3) and o.box_size.shape == (3,)
    assert o.box_matrix.shape == (4, 4) and np.all(np.sort(o.box_size) > 0)
    # ... and with objects switched off the single point cloud with labels
    integ1 = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_SEMANTIC",
                 use_semantic_probabilistic=True, kVolumetricIntegrationB200GenerateObjects=False)
    integ1.add_keyframe_data(kd)
    integ1.step()
    out = integ1.pop_output()
    assert out.point_cloud.semantics.tolist() == [1, 2] and out.point_cloud.object_ids.tolist() == [3, -1]
    assert ("voxels", 3, 0.6) in integ1.volume.calls
    # no instance image: plain carve + integrate without object ids
    integ2 = Cls(_camera(cfg), P.DatasetEnvironmentType.OUTDOOR, None, "B200_SEMANTIC",
                 kVolumetricIntegrationVoxelGridUseCarving=True)
    assert integ2.volume.calls[:2] == [("thr", 10.0), ("rate", 0.05)]
    integ2.add_keyframe_data(P.VolumetricIntegrationKeyframeData(
        id=4, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=d, semantic_img=np.ones(d.shape, np.int32)))
    integ2.step()
    names = [x[0] for x in integ2.volume.calls]
    assert "carve" in names and "assign" not in names
    assert [x for x in integ2.volume.calls if x[0] == "rgbd"][0][3] is None
    integ2.save(str(tmp_path))
    integ2.step()
    assert os.path.exists(os.path.join(tmp_path, "dense_map.ply"))
    integ2.reset()
    integ2.add_update_output_task()
    integ2.step()
    assert ("reset",) in integ2.volume.calls


@pytest.mark.gpu
def test_semantic_adapter_end_to_end_on_gpu():
    """The plugin class driving the real GPU grid == the same calls made by hand."""
    from pyslam_b200 import CameraFrustrum, VoxelBlockSemanticProbabilisticGrid, remap_instance_ids
    from tests._util import GOLDEN, sort_dump
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    cfg = S.CONFIGS["T0"]
    kw = dict(kVolumetricIntegrationVoxelLength=float(g["voxel_size"]), kVolumetricIntegrationVoxelGridUseCarving=True,
              kVolumetricIntegrationVoxelGridShadowPointsFilter=False,
              kVolumetricIntegrationVoxelGridCarvingDepthThreshold=0.08,
              kVolumetricIntegrationB200CapacityBlocks=1024, use_semantic_probabilistic=True)
    Cls = P.standalone_semantic_integrator_class()
    integ = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_SEMANTIC", **kw)
    manual = VoxelBlockSemanticProbabilisticGrid(float(g["voxel_size"]), 8, capacity_blocks=1024)
    manual.set_depth_threshold(5.0)
    manual.set_depth_decay_rate(0.1)
    K = g["K"]
    for i in range(int(g["n_frames"])):
        d, c, T = g[f"depth_{i}"], g[f"color_{i}"], g[f"Tcw_{i}"]
        cls_img, inst_img = g[f"class_image_{i}"], g[f"instance_image_{i}"]
        integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(
            id=i, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=d, semantic_img=cls_img,
            semantic_instances_img=inst_img))
        integ.step()
        fr = CameraFrustrum(K[0], K[1], K[2], K[3], d.shape[1], d.shape[0], T, depth_max=8.0, depth_min=1e-2)
        m = manual.assign_object_ids_to_instance_ids(fr, cls_img, inst_img, d, depth_threshold=0.08, do_carving=True,
                                                     min_vote_ratio=0.5, min_votes=3)
        assert m == integ.last_instance_map
        manual.integrate_rgbd(d, c, K, np.linalg.inv(T), cls_img, remap_instance_ids(inst_img, m), max_depth=4.0,
                              use_depths=True, filter_shadow_points=False)
    a, b = sort_dump(integ.volume.dump_blocks(8)), sort_dump(manual.dump_blocks(8))
    for k in ("keys", "count", "pos_sum", "col_sum", "object_id", "class_id", "confidence", "lab_logp"):
        assert np.array_equal(a[k], b[k]), k
    assert (a["object_id"] > 0).sum() > 200
    integ.add_update_output_task()
    integ.step()
    out = None
    while True:
        o = integ.pop_output()
        if o is None:
            break
        out = o
    assert out.objects.num_objects == len(out.objects.object_list) > 0     # instance ids -> objects representation
    ids = sorted(o.object_id for o in out.objects.object_list)
    dump_ids = a["object_id"][(a["count"] > 3) & (a["confidence"] >= 0.6)]
    assert ids == sorted(set(int(i) for i in dump_ids if i >= 0))
    integ.quit()


def test_voxel_grid_adapter_flow_with_fake_grid(monkeypatch, tmp_path):
    """The point-average backend: carve sees the UNFILTERED depth before the frame is integrated, integrate_rgbd gets
    Twc and the shadow-filter flag, outputs are plain point clouds (volumetric_integrator_voxel_grid.py:232-370)."""
    from pyslam_b200 import integrator_semantic as IS

    class _FakeGrid(_FakeSemanticGrid):
        def __init__(self, voxel_size, block_size, **kw):
            super().__init__(voxel_size=voxel_size, block_size=block_size, **kw)

        def integrate_rgbd(self, depth, color, K, Twc, **kw):
            self.calls.append(("rgbd", tuple(K), np.asarray(Twc).copy(), kw))

        def get_voxels(self, min_count=1, min_confidence=0.0):
            self.calls.append(("voxels", min_count))
            return SimpleNamespace(points=np.zeros((2, 3)), colors=np.ones((2, 3), np.float32))

    monkeypatch.setattr(IS, "VoxelBlockGrid", _FakeGrid)
    Cls = P.standalone_voxel_grid_integrator_class()
    cfg = S.CONFIGS["T0"]
    integ = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_VOXEL_GRID",
                kVolumetricIntegrationVoxelGridUseCarving=True, kVolumetricIntegrationVoxelLength=0.02)
    assert integ.volume.kw["voxel_size"] == 0.02 and integ.volume.kw["capacity_blocks"] == 1 << 17
    d, c, T = S.render_frame(cfg, 0)
    integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(id=5, pose=T, img=np.ascontiguousarray(c[..., ::-1]),
                                                                depth=d))
    integ.step()
    names = [x[0] for x in integ.volume.calls]
    assert names.index("carve") < names.index("rgbd")
    rgbd = [x for x in integ.volume.calls if x[0] == "rgbd"][0]
    assert np.allclose(rgbd[2] @ T, np.eye(4), atol=1e-9) and rgbd[3]["filter_shadow_points"] is True
    assert rgbd[3]["max_depth"] == 4.0
    out = integ.pop_output()
    assert out.id == 5 and out.point_cloud.points.shape == (2, 3) and out.mesh is None
    assert ("voxels", 3) in integ.volume.calls
    integ.save(str(tmp_path))
    integ.step()
    assert os.path.exists(os.path.join(tmp_path, "dense_map.ply"))


@pytest.mark.gpu
def test_voxel_grid_adapter_end_to_end_on_gpu():
    """The point-average plugin class on the real GPU grid == the same calls made by hand."""
    from pyslam_b200 import CameraFrustrum, VoxelBlockGrid
    from tests._util import sort_dump
    cfg = S.CONFIGS["T0"]
    Cls = P.standalone_voxel_grid_integrator_class()
    integ = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_VOXEL_GRID",
                kVolumetricIntegrationVoxelLength=0.03, kVolumetricIntegrationVoxelGridUseCarving=True,
                kVolumetricIntegrationB200CapacityBlocks=4096)
    manual = VoxelBlockGrid(0.03, 8, capacity_blocks=4096)
    for i in range(4):
        d, c, T = S.render_frame(cfg, i)
        integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(id=i, pose=T, img=np.ascontiguousarray(c[..., ::-1]),
                                                                    depth=d))
        integ.step()
        fr = CameraFrustrum(cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.width, cfg.height, T, depth_max=8.0, depth_min=1e-2)
        manual.carve(fr, d, 3e-2)
        manual.integrate_rgbd(d, c, cfg.K, np.linalg.inv(T), max_depth=4.0, filter_shadow_points=True)
    a, b = sort_dump(integ.volume.dump_blocks()), sort_dump(manual.dump_blocks())
    assert np.array_equal(a["keys"], b["keys"]) and np.array_equal(a["count"], b["count"])
    assert np.allclose(a["pos_sum"], b["pos_sum"], rtol=1e-5, atol=1e-6)      # float atomics: order differs
    assert (a["count"] > 0).sum() > 1000
    integ.add_update_output_task()
    integ.step()
    out = None
    while True:
        o = integ.pop_output()
        if o is None:
            break
        out = o
    assert out.point_cloud.points.shape[1] == 3 and len(out.point_cloud.points) > 100
    integ.quit()
