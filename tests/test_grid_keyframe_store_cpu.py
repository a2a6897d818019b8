"""Pose-only rebuild messages of the grid plugins (kVolumetricIntegrationB200KeyframeStoreFrames), host logic on the
CPU with a stand-in grid: the parent's add_task with the store on and off, label images that must travel when the
stored frame lacks them, light tasks whose frame is not stored, and the TSDF plugin's light tasks unchanged."""

from types import SimpleNamespace

import numpy as np
import pytest

from pyslam_b200 import integrator_semantic as IS
from pyslam_b200 import keyframe_store as KS
from pyslam_b200 import synthetic as S
from tests import plugin_standins as P

INTEGRATE = P.VolumetricIntegrationTaskType.INTEGRATE


class _StoreGrid:
    """Stands in for both grids with a frame store: set_frame stores frames in call order while there is room,
    stage_stored hands back what was staged, and the loop body's calls are recorded."""

    def __init__(self, **kw):
        self.calls, self.max_frames, self.frames, self.last = [], 0, [], -1

    def set_frame_store(self, n):
        self.max_frames = n

    def set_rectification(self, *a, **k):
        pass

    def set_depth_threshold(self, v):
        pass

    def set_depth_decay_rate(self, v):
        pass

    def _staged(self, color, cls, inst):
        return SimpleNamespace(depth="d", filtered_depth="fd", color=int(np.asarray(color)[0, 0, 0]),
                               class_image=None if cls is None else "cls",
                               instance_image=None if inst is None else "inst")

    def set_frame(self, depth, color, class_image=None, instance_image=None, depth_scale=None,
                  filter_shadow_points=False):
        fr = self._staged(color, class_image, instance_image)
        self.last = len(self.frames) if len(self.frames) < self.max_frames else -1
        if self.last >= 0:
            self.frames.append(fr)
        self.calls.append(("set_frame", fr.color))
        return fr

    def last_stored_slot(self):
        return self.last

    def stage_stored(self, slot):
        self.calls.append(("stage_stored", slot))
        return self.frames[slot]

    def integrate_rgbd(self, depth, color, K, Twc, class_image=None, object_image=None, **kw):
        self.calls.append(("integrate_rgbd", color, class_image, object_image, float(np.linalg.inv(Twc)[0, 0])))

    def assign_object_ids_to_instance_ids(self, *a, **k):
        self.calls.append(("assoc",))
        return {}

    def remap_instance_ids(self):
        return "obj"

    def carve(self, *a, **k):
        self.calls.append(("carve",))

    def reset(self):
        self.calls.append(("reset",))

    def get_voxels(self, **kw):
        z = np.zeros((0, 3))
        return SimpleNamespace(points=z, colors=z, class_ids=np.zeros(0), object_ids=np.zeros(0))

    def close(self):
        pass


def _kd(i, ts=None, cls=True, inst=True):
    cfg = S.CONFIGS["T0"]
    d = np.full((cfg.height, cfg.width), 1.0, np.float32)
    c = np.full((cfg.height, cfg.width, 3), i, np.uint8)
    lab = np.ones((cfg.height, cfg.width), np.int32)
    return P.VolumetricIntegrationKeyframeData(
        id=i, pose=np.eye(4) * (i + 1), img=c, depth=d, timestamp=float(i) / 10 if ts is None else ts,
        semantic_img=lab if cls else None, semantic_instances_img=lab if inst else None)


def _plugin(monkeypatch, kind, frames, **kw):
    monkeypatch.setattr(IS, "VoxelBlockGrid", _StoreGrid)
    monkeypatch.setattr(IS, "VoxelBlockSemanticGrid", _StoreGrid)
    monkeypatch.setattr(IS, "VoxelBlockSemanticProbabilisticGrid", _StoreGrid)
    cfg = S.CONFIGS["T0"]
    cam = SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)
    y, x = np.mgrid[:cfg.height, :cfg.width].astype(np.float32)
    make = P.standalone_voxel_grid_integrator_class if kind == "voxel" else P.standalone_semantic_integrator_class
    return make()(cam, P.DatasetEnvironmentType.INDOOR, None, "B200", calib_maps=(x, y),
                  kVolumetricIntegrationB200KeyframeStoreFrames=frames, **kw)


def _sent(integ):
    out = []
    while not integ.q_in.empty():
        out.append(integ.q_in.get())
    return out


@pytest.mark.parametrize("kind", ["voxel", "semantic"])
def test_add_task_sends_light_tasks_for_stored_keyframes(monkeypatch, kind):
    integ = _plugin(monkeypatch, kind, 3)
    assert integ._b200_keyframe_table.labels == (kind == "semantic")
    for i in range(4):
        integ.add_keyframe_data(_kd(i))
    integ.run_pending()
    assert integ._stored_slots == {KS.keyframe_key(_kd(i)): i for i in range(3)}
    integ.reset()
    tasks = [_kd(i) for i in range(4)]
    for kd in tasks:
        kd.pose = kd.pose * 2
        integ.add_keyframe_data(kd)
    sent = _sent(integ)
    assert [KS.is_stored(t) for t in sent] == [True, True, True, False]
    for t in sent[:3]:
        assert all(getattr(t.keyframe_data, n) is None for n in KS.IMAGE_FIELDS)
    integ.volume.calls.clear()
    for t in sent:
        integ.q_in.put(t)
    integ.run_pending()
    calls = integ.volume.calls
    assert [c for c in calls if c[0] in ("stage_stored", "set_frame")] == [
        ("stage_stored", 0), ("stage_stored", 1), ("stage_stored", 2), ("set_frame", 3)]
    # the stored frames are integrated with the new poses, the labels they were stored with and their association
    ints = [c for c in calls if c[0] == "integrate_rgbd"]
    assert [c[1] for c in ints] == [0, 1, 2, 3] and [c[4] for c in ints] == [2.0 * (i + 1) for i in range(4)]
    if kind == "semantic":
        assert all(c[2] == "cls" and c[3] == "obj" for c in ints)
        assert calls.count(("assoc",)) == 4
    assert integ.last_integrated_id == 3


@pytest.mark.parametrize("kind", ["voxel", "semantic"])
def test_store_off_passes_every_task_through(monkeypatch, kind):
    integ = _plugin(monkeypatch, kind, 0)
    assert integ._b200_keyframe_table is None and integ.volume.max_frames == 0
    for _ in range(2):
        for i in range(3):
            integ.add_keyframe_data(_kd(i))
        sent = _sent(integ)
        assert not any(KS.is_stored(t) for t in sent) and all(t.keyframe_data.img is not None for t in sent)
        for t in sent:
            integ.q_in.put(t)
        integ.run_pending()
    assert [c[0] for c in integ.volume.calls if c[0] in ("set_frame", "stage_stored")] == ["set_frame"] * 6


def test_label_images_travel_when_the_stored_frame_lacks_them(monkeypatch):
    integ = _plugin(monkeypatch, "semantic", 8)
    stored = [_kd(0), _kd(1, inst=False), _kd(2, cls=False, inst=False)]
    for kd in stored:
        integ.add_keyframe_data(kd)
    integ.run_pending()
    # same label images: light; more or fewer label images than the stored frame had: the task keeps its images
    again = [(_kd(0), True), (_kd(0, inst=False), False), (_kd(1, inst=False), True), (_kd(1), False),
             (_kd(2, cls=False, inst=False), True), (_kd(2, inst=False), False)]
    for kd, _ in again:
        integ.add_keyframe_data(kd)
    assert [KS.is_stored(t) for t in _sent(integ)] == [light for _, light in again]
    # an empty label image counts as none
    empty = _kd(1, inst=False)
    empty.semantic_instances_img = np.zeros((0, 0), np.int32)
    integ.add_keyframe_data(empty)
    assert KS.is_stored(_sent(integ)[0])


@pytest.mark.parametrize("kind", ["voxel", "semantic"])
def test_light_task_for_a_frame_not_stored_is_logged_and_skipped(monkeypatch, kind):
    integ = _plugin(monkeypatch, kind, 4)
    logged = []
    monkeypatch.setattr(P.StandaloneIntegratorBase, "print", staticmethod(lambda *a, **k: logged.append(a[0])))
    integ.q_in.put(KS.light_task(P.VolumetricIntegrationTask(_kd(5), INTEGRATE), SimpleNamespace(lookup=lambda kd: 0),
                                 INTEGRATE))
    integ.run_pending()
    assert integ.volume.calls == [] and integ.last_integrated_id == -1
    assert any("keyframe 5" in m and "not in the frame store" in m for m in logged)


def test_voxel_grid_table_does_not_look_at_labels(monkeypatch):
    """The point-average grid stores no label images: a keyframe whose label images changed still travels light."""
    integ = _plugin(monkeypatch, "voxel", 4)
    integ.add_keyframe_data(_kd(0, cls=False, inst=False))
    integ.run_pending()
    integ.add_keyframe_data(_kd(0))
    t = _sent(integ)[0]
    assert KS.is_stored(t) and t.keyframe_data.semantic_img is None


def test_tsdf_table_does_not_look_at_labels(monkeypatch):
    """The TSDF plugin's table publishes no label flags: a keyframe with label images still travels light."""
    from tests import test_keyframe_store_cpu as T
    integ = T._plugin(monkeypatch, 2)
    assert not integ._b200_keyframe_table.labels
    integ.add_keyframe_data(_kd(0))
    integ.run_pending()
    integ.add_keyframe_data(_kd(0, inst=False))
    t = _sent(integ)[0]
    assert KS.is_stored(t) and t.keyframe_data.semantic_img is None
