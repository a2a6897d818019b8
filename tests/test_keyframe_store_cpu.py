"""Pose-only rebuild messages of the TSDF plugin (pyslam_b200.keyframe_store), host logic on the CPU: the parent's
add_task, the table shared with a spawned integrator process, and the split of a drained backlog into runs."""

import multiprocessing
from types import SimpleNamespace

import numpy as np

from pyslam_b200 import integrator as I
from pyslam_b200 import keyframe_store as KS
from pyslam_b200 import synthetic as S
from tests import plugin_standins as P

INTEGRATE = P.VolumetricIntegrationTaskType.INTEGRATE


class _StoreVolume:
    """Stands in for B200TsdfVolume with a frame store: frames get slots in call order while there is room."""

    def __init__(self, **kw):
        self.calls, self.max_frames, self.count, self.last = [], 0, 0, []

    def set_frame_store(self, n):
        self.max_frames = n

    def _store(self, n):
        self.last = []
        for _ in range(n):
            self.last.append(self.count if self.count < self.max_frames else -1)
            self.count += self.count < self.max_frames

    def integrate_batch(self, depths, colors, K, poses, depth_scale=None):
        self._store(len(depths))
        self.calls.append(("integrate_batch", [int(c[0, 0, 0]) for c in colors]))

    def integrate_stored(self, slots, K, poses):
        self.last = [-1] * len(slots)
        self.calls.append(("integrate_stored", [int(s) for s in slots], np.asarray(poses).copy()))

    def last_stored_slots(self):
        return np.asarray(self.last, np.int32)

    def reset(self):
        self.calls.append(("reset",))

    def extract_triangle_mesh(self):
        return SimpleNamespace(vertices=np.zeros((0, 3)), triangles=np.zeros((0, 3), np.int32),
                               vertex_colors=np.zeros((0, 3)), vertex_normals=np.zeros((0, 3)))

    def close(self):
        pass


def _kd(i, ts=None):
    cfg = S.CONFIGS["T0"]
    d = np.full((cfg.height, cfg.width), 1.0, np.float32)
    c = np.full((cfg.height, cfg.width, 3), i, np.uint8)
    return P.VolumetricIntegrationKeyframeData(id=i, pose=np.eye(4) * (i + 1), img=c, depth=d,
                                               timestamp=float(i) / 10 if ts is None else ts)


def _plugin(monkeypatch, frames, **kw):
    monkeypatch.setattr(I, "B200TsdfVolume", _StoreVolume)
    cfg = S.CONFIGS["T0"]
    cam = SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)
    return P.standalone_integrator_class()(cam, P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF",
                                           kVolumetricIntegrationB200KeyframeStoreFrames=frames, **kw)


def _sent(integ):
    """The tasks waiting in q_in, emptied."""
    out = []
    while not integ.q_in.empty():
        out.append(integ.q_in.get())
    return out


def test_add_task_sends_light_tasks_only_for_confirmed_keyframes(monkeypatch):
    integ = _plugin(monkeypatch, 3)
    for i in range(4):
        integ.add_keyframe_data(_kd(i))
    assert not any(KS.is_stored(t) for t in _sent(integ))   # nothing was confirmed yet
    for i in range(4):
        integ.add_keyframe_data(_kd(i))
    integ.run_pending()
    assert integ.volume.calls[0] == ("integrate_batch", [0, 1, 2, 3])
    assert integ._stored_slots == {KS.keyframe_key(_kd(i)): i for i in range(3)}   # the store holds 3 frames
    # rebuild: RESET, then every keyframe again with a new pose; frame 3 did not fit, another timestamp is another frame
    integ.reset()
    tasks = [_kd(i) for i in range(4)] + [_kd(1, ts=9.0)]
    for kd in tasks:
        kd.pose = kd.pose * 2
        integ.add_keyframe_data(kd)
    sent = _sent(integ)
    assert [KS.is_stored(t) for t in sent] == [True, True, True, False, False]
    for t, kd in zip(sent, tasks):
        light = t.keyframe_data
        assert light.id == kd.id and light.timestamp == kd.timestamp and np.array_equal(light.pose, kd.pose)
        if KS.is_stored(t):
            assert all(getattr(light, name) is None for name in KS.IMAGE_FIELDS)
        else:
            assert light is kd
        assert kd.img is not None and not KS.is_stored(P.VolumetricIntegrationTask(kd, INTEGRATE))  # input untouched
    # other task types pass through as they are
    integ.add_update_output_task()
    assert _sent(integ)[0].task_type == P.VolumetricIntegrationTaskType.UPDATE_OUTPUT


def test_store_off_passes_every_task_through(monkeypatch):
    integ = _plugin(monkeypatch, 0)
    assert integ._b200_keyframe_table is None and integ.volume.max_frames == 0
    for _ in range(2):
        for i in range(3):
            integ.add_keyframe_data(_kd(i))
        sent = _sent(integ)
        assert not any(KS.is_stored(t) for t in sent) and all(t.keyframe_data.img is not None for t in sent)
        for t in sent:
            integ.q_in.put(t)
        integ.run_pending()
    assert [c[0] for c in integ.volume.calls] == ["integrate_batch", "integrate_batch"]


def test_mixed_backlog_is_split_into_runs_in_order_with_one_frame_batches(monkeypatch):
    tasks = [P.VolumetricIntegrationTask(_kd(i), INTEGRATE) for i in range(7)]
    stored = [True, True, False, True, False, False, True]
    tasks = [KS.light_task(t, SimpleNamespace(lookup=lambda kd: 0), INTEGRATE) if s else t
             for t, s in zip(tasks, stored)]
    runs = KS.split_runs(tasks)
    assert [(s, [t.keyframe_data.id for t in r]) for s, r in runs] == [
        (True, [0, 1]), (False, [2]), (True, [3]), (False, [4, 5]), (True, [6])]
    # through the plugin: one integrate_stored call per stored run, integrate_batch for the others (a lone frame is a
    # one-frame batch), in queue order
    integ = _plugin(monkeypatch, 8)
    for i in range(7):
        integ.add_keyframe_data(_kd(i))
    integ.run_pending()
    assert list(integ._stored_slots.values()) == list(range(7))
    integ.volume.calls.clear()
    for i, s in enumerate(stored):
        kd = _kd(i if s else 10 + i)   # unstored keyframes are new ones
        kd.pose = kd.pose * 3
        integ.add_keyframe_data(kd)
    integ.run_pending()
    calls = [(c[0], c[1]) for c in integ.volume.calls]
    assert calls == [("integrate_stored", [0, 1]), ("integrate_batch", [12]), ("integrate_stored", [3]),
                     ("integrate_batch", [14, 15]), ("integrate_stored", [6])]
    assert np.array_equal(integ.volume.calls[0][2], np.stack([_kd(0).pose * 3, _kd(1).pose * 3]))
    assert integ.last_integrated_id == 6


def test_light_task_for_a_frame_not_stored_is_logged(monkeypatch):
    integ = _plugin(monkeypatch, 4)
    logged = []
    monkeypatch.setattr(P.StandaloneIntegratorBase, "print", staticmethod(lambda *a, **k: logged.append(a[0])))
    integ.q_in.put(KS.light_task(P.VolumetricIntegrationTask(_kd(5), INTEGRATE), SimpleNamespace(lookup=lambda kd: 0),
                                 INTEGRATE))
    integ.run_pending()
    assert integ.volume.calls == [] and any("keyframe 5" in m and "not in the frame store" in m for m in logged)


def _child_publishes(table, entries):
    """A stand-in integrator process: publishes its stored keyframes, slot by slot."""
    for slot, (kid, ts) in enumerate(entries):
        table.publish(slot, SimpleNamespace(id=kid, timestamp=ts))


def test_table_crosses_a_spawn_into_the_child():
    ctx = multiprocessing.get_context("spawn")
    table = KS.StoredKeyframeTable(4, ctx)
    entries = [(10, 0.5), (11, 0.75), (12, 1.0)]
    p = ctx.Process(target=_child_publishes, args=(table, entries))
    p.start()
    p.join(120)
    assert p.exitcode == 0
    for slot, (kid, ts) in enumerate(entries):
        assert table.lookup(SimpleNamespace(id=kid, timestamp=ts)) == slot
    assert table.lookup(SimpleNamespace(id=10, timestamp=0.25)) is None
    assert table.lookup(SimpleNamespace(id=13, timestamp=1.25)) is None
    assert table.lookup(SimpleNamespace(id=10, timestamp=None)) is None
    table.publish(9, SimpleNamespace(id=1, timestamp=0.0))   # past the table: ignored
    assert table.lookup(SimpleNamespace(id=1, timestamp=0.0)) is None


def test_a_slot_never_published_matches_nothing():
    """A slot whose frame was stored by a call that then failed is never published: its zeroed entry must not match
    keyframe (0, 0.0), which is a real key on datasets whose timestamps start at 0."""
    table = KS.StoredKeyframeTable(4)
    table.publish(1, SimpleNamespace(id=7, timestamp=0.5))
    assert table.lookup(SimpleNamespace(id=0, timestamp=0.0)) is None
    assert table.lookup(SimpleNamespace(id=7, timestamp=0.5)) == 1
    table.publish(0, SimpleNamespace(id=0, timestamp=0.0))
    table.publish(2, SimpleNamespace(id=3, timestamp=0.0))
    assert table.lookup(SimpleNamespace(id=3, timestamp=0.0)) == 2
