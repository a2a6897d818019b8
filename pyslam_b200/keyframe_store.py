"""Pose-only rebuild messages of the B200 plugins (`kVolumetricIntegrationB200KeyframeStoreFrames`).

After a loop closure pySLAM's `rebuild(map)` sends RESET and enqueues every keyframe again, images included
(`base.py:1242-1318`).  With the frame store on (`B200TsdfVolume.set_frame_store`), the integrator process keeps each
keyframe's packed frame on the GPU and publishes the keyframe's `(id, timestamp)` in a `StoredKeyframeTable` shared
with the parent process.  The parent's `add_task` then replaces an INTEGRATE task of a published keyframe by a light
copy without images (`light_task`): only the id, timestamp and pose cross the queue, and the integrator replays the
stored frame with that pose (`B200TsdfVolume.integrate_stored`; the grids stage it again with
`_BlockGrid.stage_stored`).  A published keyframe stays stored until the plugin stops (the store never evicts), so a
light task always finds its frame.

The grid plugins also publish which label images each stored frame had (`label_flags`): a semantic keyframe travels
light only when its task has the same label images, so a task never loses a label image its stored frame lacks.
"""

from __future__ import annotations

import copy
import ctypes
import multiprocessing

#: the image fields of pySLAM's VolumetricIntegrationKeyframeData (base.py:100-137) a light task leaves out
IMAGE_FIELDS = ("img", "img_right", "depth", "semantic_img", "semantic_instances_img")
#: set on the keyframe data of a light task
STORED_FLAG = "b200_stored"
#: bits of label_flags
HAS_CLASS, HAS_INSTANCE = 1, 2


def _has_image(img) -> bool:
    return img is not None and getattr(img, "size", 1) > 0


def label_flags(kd) -> int:
    """HAS_CLASS | HAS_INSTANCE: the label images keyframe data `kd` carries (an empty image is none)."""
    return ((HAS_CLASS if _has_image(getattr(kd, "semantic_img", None)) else 0)
            | (HAS_INSTANCE if _has_image(getattr(kd, "semantic_instances_img", None)) else 0))


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
    valid.  With `labels` each entry also holds the `label_flags` of the keyframe whose frame the slot holds: the label
    images its task carried, not the images the grid staged.  The two match the way light_task needs because the
    semantic plugin stages a deterministic function of the task's label images and its parameters (an instance image
    is staged when the task has one and kVolumetricSemanticIntegrationUseInstanceIds is on), so a task with the same
    label images stages the same ones again.  A change that stages label images on other criteria must publish what
    it staged instead."""

    def __init__(self, slots: int, ctx=None, labels: bool = False):
        ctx = ctx or multiprocessing.get_context("spawn")
        self.slots = int(slots)
        self.labels = bool(labels)
        self._ids = ctx.RawArray(ctypes.c_int64, self.slots)
        self._ts = ctx.RawArray(ctypes.c_double, self.slots)
        self._flags = ctx.RawArray(ctypes.c_int32, self.slots)
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
            self._flags[slot] = label_flags(kd)
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

    def slot_label_flags(self, slot: int) -> int:
        """The label_flags published with slot `slot`."""
        return int(self._flags[slot])


def light_task(task, table: StoredKeyframeTable, integrate_type):
    """`task`, or for an INTEGRATE task whose keyframe `table` holds, a copy of it whose keyframe data has no images
    and carries the STORED_FLAG.  A table with labels also needs the task's label images to be those the stored frame
    had (label_flags); else the task keeps its images."""
    kd = getattr(task, "keyframe_data", None)
    slot = None if task.task_type != integrate_type or kd is None else table.lookup(kd)
    if slot is None or (getattr(table, "labels", False) and table.slot_label_flags(slot) != label_flags(kd)):
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
