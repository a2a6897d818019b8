"""Pose-only rebuild messages of the TSDF plugin (`kVolumetricIntegrationB200KeyframeStoreFrames`).

After a loop closure pySLAM's `rebuild(map)` sends RESET and enqueues every keyframe again, images included
(`base.py:1242-1318`).  With the frame store on (`B200TsdfVolume.set_frame_store`), the integrator process keeps each
keyframe's packed frame on the GPU and publishes the keyframe's `(id, timestamp)` in a `StoredKeyframeTable` shared
with the parent process.  The parent's `add_task` then replaces an INTEGRATE task of a published keyframe by a light
copy without images (`light_task`): only the id, timestamp and pose cross the queue, and the integrator replays the
stored frame with that pose (`B200TsdfVolume.integrate_stored`).  A published keyframe stays stored until the plugin
stops (the store never evicts), so a light task always finds its frame.
"""

from __future__ import annotations

import copy
import ctypes
import multiprocessing

#: the image fields of pySLAM's VolumetricIntegrationKeyframeData (base.py:100-137) a light task leaves out
IMAGE_FIELDS = ("img", "img_right", "depth", "semantic_img", "semantic_instances_img")
#: set on the keyframe data of a light task
STORED_FLAG = "b200_stored"


def keyframe_key(kd) -> tuple:
    """(id, timestamp) of a keyframe, the key of its stored frame.  A keyframe without a timestamp gets a NaN one,
    which matches nothing, so it always travels with its images."""
    ts = getattr(kd, "timestamp", None)
    return int(kd.id), float("nan") if ts is None else float(ts)


class StoredKeyframeTable:
    """`(keyframe id, timestamp)` of each frame-store slot the integrator process has filled, in shared memory.

    The parent creates it before the integrator process is spawned (`ctx`: the spawn context), one entry per store
    slot; the integrator process `publish`es each slot once its frame is stored, and the parent `lookup`s keyframes.
    Slots are published in slot order, but a slot may never be (its frame was stored by a call that then failed), so
    only entries flagged as published match.  Entries are only ever added, so a pair the parent has seen stays
    valid."""

    def __init__(self, slots: int, ctx=None):
        ctx = ctx or multiprocessing.get_context("spawn")
        self.slots = int(slots)
        self._ids = ctx.RawArray(ctypes.c_int64, self.slots)
        self._ts = ctx.RawArray(ctypes.c_double, self.slots)
        self._published = ctx.RawArray(ctypes.c_bool, self.slots)   # an entry never published matches nothing
        self._count = ctx.RawValue(ctypes.c_int64, 0)   # no entry at or past count is published
        self._lock = ctx.Lock()
        self._seen, self._known = 0, {}                 # the reader's copy of the published entries

    def __getstate__(self):
        state = dict(self.__dict__)
        state["_seen"], state["_known"] = 0, {}
        return state

    def publish(self, slot: int, kd) -> None:
        """Slot `slot` holds keyframe `kd`'s frame.  A slot past the table is ignored."""
        if not 0 <= slot < self.slots:
            return
        kid, ts = keyframe_key(kd)
        with self._lock:
            self._ids[slot], self._ts[slot] = kid, ts
            self._published[slot] = True
            self._count.value = max(self._count.value, slot + 1)

    def lookup(self, kd):
        """The slot of keyframe `kd`'s stored frame, or None."""
        if self._seen < self.slots:
            with self._lock:
                n = self._count.value
                for s in range(self._seen, n):
                    if self._published[s]:
                        self._known.setdefault((self._ids[s], self._ts[s]), s)
                self._seen = n
        return self._known.get(keyframe_key(kd))


def light_task(task, table: StoredKeyframeTable, integrate_type):
    """`task`, or for an INTEGRATE task whose keyframe `table` holds, a copy of it whose keyframe data has no images
    and carries the STORED_FLAG."""
    kd = getattr(task, "keyframe_data", None)
    if task.task_type != integrate_type or kd is None or table.lookup(kd) is None:
        return task
    light, kd = copy.copy(task), copy.copy(kd)
    for name in IMAGE_FIELDS:
        if hasattr(kd, name):
            setattr(kd, name, None)
    setattr(kd, STORED_FLAG, True)
    light.keyframe_data = kd
    return light


def is_stored(task) -> bool:
    return bool(getattr(getattr(task, "keyframe_data", None), STORED_FLAG, False))


def split_runs(tasks) -> list:
    """The drained INTEGRATE tasks as runs of consecutive light tasks and of image-carrying tasks, in their order:
    [(stored, [task, ...]), ...]."""
    runs = []
    for t in tasks:
        s = is_stored(t)
        if runs and runs[-1][0] == s:
            runs[-1][1].append(t)
        else:
            runs.append((s, [t]))
    return runs
