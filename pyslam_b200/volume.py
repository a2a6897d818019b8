"""Host-side mirror of the reference's volume objects, over the C ABI (include/b2v.h).

Two duck types are provided, the two `self.volume` shapes pySLAM's dense front-end drives
(SURVEY.md §8b):

* `B200TsdfVolume` — the north_star API `integrate(depth, color, K, pose)` / `extract_mesh()`
  plus the Open3D-style methods the TSDF backend calls
  (`pyslam/dense/volumetric_integrator_tsdf.py:156,223,239,246,260,267`):
  `integrate(rgbd, intrinsic, extrinsic)`, `extract_triangle_mesh()`, `extract_point_cloud()`,
  `reset()`.
* `VoxelBlockGrid` — pySLAM's own `volumetric.VoxelBlockGrid` surface
  (`cpp/volumetric/volumetric_grid_module.h:732-935`): `integrate(points, colors)`,
  `get_voxels(min_count)`, `get_points()`, `get_colors()`, `clear()`, `reset()`, `size()`,
  `empty()`, `num_blocks()`, `get_block_size()`, `get_total_voxel_count()`,
  `remove_low_count_voxels(n)`.

Everything numeric happens in the CUDA library; these classes only validate arguments (same
error behaviour as the reference: `RuntimeError` on shape / dtype mismatches,
`volumetric_grid_module.h:140-258`) and move pointers.  There is no CPU fallback.
"""

from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib, map_state
from ._lib import B2VConfigEx, BLOCK_SIZE, BLOCK_VOXELS, VOXEL_PLANES


def _as_K4(K) -> np.ndarray:
    """Accept (fx, fy, cx, cy), a 3x3 matrix, or an object with fx/fy/cx/cy (camera / o3d-like)."""
    if hasattr(K, "fx") and hasattr(K, "cx"):
        return np.array([K.fx, K.fy, K.cx, K.cy], dtype=np.float64)
    if hasattr(K, "intrinsic_matrix"):
        K = np.asarray(K.intrinsic_matrix)
    K = np.asarray(K, dtype=np.float64)
    if K.shape == (3, 3):
        return np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]], dtype=np.float64)
    if K.size == 4:
        return np.ascontiguousarray(K.reshape(4))
    raise RuntimeError("K must be (fx, fy, cx, cy) or a 3x3 intrinsic matrix")


def _is_torch_cuda(x) -> bool:
    return hasattr(x, "data_ptr") and hasattr(x, "is_cuda") and bool(x.is_cuda)


def _keys4(keys) -> np.ndarray:
    """Block keys [n,3] as the library takes them: int32 [n,4] = {x, y, z, 0}, the table's own key layout."""
    k = np.asarray(keys, np.int32).reshape(-1, 3)
    k4 = np.zeros((k.shape[0], 4), np.int32)
    k4[:, :3] = k
    return k4


def _block_hashes(keys) -> np.ndarray:
    """The reference's BlockKeyHash of block keys [n,3] (b2v_block_key_hashes: the hash the kernels use)."""
    k4 = _keys4(keys)
    h = np.zeros(len(k4), np.uint64)
    if len(k4) and _lib.load().b2v_block_key_hashes(k4.ctypes.data, len(k4), h.ctypes.data) != _lib.B2V_OK:
        raise RuntimeError("b2v_block_key_hashes failed")
    return h


def _pinned_owner(x):
    """The torch tensor behind a pinned host array (a numpy view of one included), or None.  The copy engine reads
    pinned memory after the integrate call returns; pageable memory is staged before it returns."""
    while x is not None:
        if hasattr(x, "is_pinned"):
            return x if x.is_pinned() else None
        x = getattr(x, "base", None)
    return None


#: B200TsdfVolume holds the device and pinned inputs of the work in flight until a synchronising call.  Before a call
#: that would take them past this many bytes it waits for the earlier calls and releases their inputs; a storage is
#: counted once however often it is passed (a resident frame buffer, views into one pool), and an input larger than
#: the bound is still held: the wait comes only when a later call brings another storage.
HELD_INPUT_BYTES_MAX = 1 << 30
WEIGHT_MAX = 2.0 ** 24   # the largest voxel weight a TSDF block may hold (include/b2v.h)


class TriangleMesh:
    """Arrays shaped like `VolumetricIntegrationMesh` (volumetric_integrator_base.py:213-226)."""

    def __init__(self, vertices, triangles, vertex_colors, edge_ids=None):
        self.vertices = vertices                 # [V,3] float64
        self.triangles = triangles               # [T,3] int32
        self.vertex_colors = vertex_colors       # [V,3] float64 in [0,1]
        self.vertex_normals = np.zeros((0, 3), dtype=np.float64)  # Open3D leaves them empty too
        self.edge_ids = edge_ids                 # [V,4] int32 canonical weld key (parity hook)


class PointCloud:
    """Arrays shaped like `VolumetricIntegrationPointCloud` (volumetric_integrator_base.py:159-210)."""

    def __init__(self, points, colors, edge_ids=None):
        self.points = points
        self.colors = colors
        self.edge_ids = edge_ids                 # [N,4] int32 voxel (x,y,z) + axis of each zero crossing, if known


class _MapState:
    """`save_state` / `load_state` of the TSDF volume and the voxel grids (`map_state` holds the file format).  A map
    kind names itself in `_STATE_KIND` and provides `_state_config()` (what the voxels mean: must match to load),
    `_state_arrays()` (per-block array specs, keys first), `_export_state()`, `_state_capacity()` (the most blocks it
    can hold), `_clear_state()` and `_upload_state(blocks)`; the semantic grids add restored settings, and a map with
    `_STATE_LABELS` its overflow label pairs (`_export_labels()`, `_check_labels(labels)`, `_upload_labels(keys,
    labels)`)."""

    _STATE_KIND = ""
    _STATE_BOUNDS: dict = {}
    _STATE_LABELS = False   # the map has overflow label pairs (a Bayesian semantic grid)

    def _state_semantic_kind(self) -> int:
        return -1

    def _state_settings(self) -> dict:
        return {}

    def _restore_settings(self, settings: dict) -> None:
        pass

    def _check_blocks(self, blocks: dict) -> None:
        """Raise ValueError for block values the map does not take (checked before the map is cleared)."""

    def save_state(self, path) -> None:
        """Write the map's state to `path` (one uncompressed `.npz`; one file per shard for a sharded map), after the
        work in flight is done.  The state is every block's raw voxels plus the configuration and settings a load
        restores.  Not part of it: rectification maps and staged frames, bench counters and, on semantic grids, the
        label-overflow counter (counts from 0 after a load) and the last association's instance map
        (`remap_instance_ids` needs a new association, as on a fresh grid)."""
        map_state.write(path, self._STATE_KIND, self._state_semantic_kind(), self._state_config(),
                        self._state_settings(), self.shard_rank, self.shard_count, self._export_state(),
                        self._export_labels() if self._STATE_LABELS else None)

    def load_state(self, paths) -> None:
        """Replace the map with the state in `paths`: one file, or a list such as the files of every shard of an
        N-rank map.  Only the blocks this object owns under its own shard setting are kept (`sharding.owner_of`), so a
        map saved by N ranks loads into any number of ranks, one included, with the same voxels bit for bit.  The
        files are validated first: a wrong format version, kind or configuration, missing or malformed arrays,
        duplicate keys, out-of-range values or more owned blocks than this object's ceiling raise ValueError and leave
        the map as it was.  The blocks are uploaded in bounded chunks.  What is not part of the state: `save_state`."""
        spec = self._state_arrays()
        settings, blocks, *labels = map_state.read(
            paths, self._STATE_KIND, self._state_semantic_kind(), self._state_config(),
            {name: np.asarray(v).dtype for name, v in self._state_settings().items()}, spec, self.shard_rank,
            self.shard_count, self._state_capacity(), self._STATE_BOUNDS, labels=self._STATE_LABELS)
        labels = labels[0] if labels else None
        self._check_blocks(blocks)
        if labels is not None:
            self._check_labels(labels)
        self._clear_state()
        block_bytes = sum(np.dtype(dt).itemsize * int(np.prod(shape)) for dt, shape in spec.values())
        for a, b in map_state.chunks(len(blocks["keys"]), block_bytes):
            part = {name: x[a:b] for name, x in blocks.items()}
            self._upload_state(part)
            if labels is not None:
                self._upload_labels(part["keys"], map_state.label_slice(labels, a, b))
        self._restore_settings(settings)


class B200TsdfVolume(_MapState):
    """H100-native TSDF + colour volume on 8^3 voxel blocks in a GPU hash table.

    Parameters mirror `o3d.pipelines.integration.ScalableTSDFVolume(voxel_length, sdf_trunc, ...)`
    as constructed at volumetric_integrator_tsdf.py:104-108, plus the depth truncation the reference
    applies while building the RGBD image (tsdf.py:215-221).
    """

    def __init__(self, voxel_length: float, sdf_trunc: float, depth_trunc: float = 4.0,
                 capacity_blocks: int = 1 << 18, device: int = 0, depth_sampling_stride: int = 4,
                 block_size: int = BLOCK_SIZE, shard_rank: int = 0, shard_count: int = 1,
                 volume_unit_resolution: int = 16, max_capacity_blocks: int | None = None,
                 color_float64: bool = False):
        """`volume_unit_resolution`: Open3D's parameter of that name.  16 (the reference's value) allocates every
        8^3 block of each 16^3 unit `ScalableTSDFVolume::LocateVolumeUnit` touches - the same voxels Open3D updates;
        8 is SURVEY decision D1 (the float32 pyslam key range of the +-sdf_trunc box, ~9 % fewer blocks).
        `max_capacity_blocks`: growth ceiling of the block pool.  Above `capacity_blocks`, the pool starts with
        `capacity_blocks` blocks of storage and grows on demand; the volume then holds, bit for bit, what a volume
        created with `capacity_blocks=max_capacity_blocks` holds.  None (or `capacity_blocks`) keeps the pool fixed.
        `color_float64`: keep each voxel's colour as Open3D's TSDFVoxel does, a float64 running mean
        (c * w + rgb) / (w + 1), so voxel, mesh and point-cloud colours equal Open3D's bit for bit.  A block then takes
        16 KiB instead of 10 KiB; tsdf and weights are the same in both modes.  False keeps the float32 running mean."""
        self._L = _lib.load()
        self._h = C.c_void_p()
        self.voxel_length = float(voxel_length)
        self.sdf_trunc = float(sdf_trunc)
        self.depth_trunc = float(depth_trunc)
        self.block_size = int(block_size)
        self.capacity_blocks = int(capacity_blocks)
        self.max_capacity_blocks = int(max_capacity_blocks or 0)
        self.device = int(device)
        self.shard_rank, self.shard_count = int(shard_rank), int(shard_count)
        self.volume_unit_resolution = int(volume_unit_resolution)
        self.depth_sampling_stride = int(depth_sampling_stride)
        self.color_float64 = bool(color_float64)
        cfg = B2VConfigEx(voxel_length, block_size, sdf_trunc, depth_trunc, depth_sampling_stride,
                        capacity_blocks, device, shard_rank, shard_count, int(volume_unit_resolution),
                        float(voxel_length), float(sdf_trunc), self.max_capacity_blocks, int(self.color_float64))
        rc = self._L.b2v_create(C.byref(cfg), C.byref(self._h))
        if rc != _lib.B2V_OK:
            msg = self._L.b2v_last_error(self._h).decode() if self._h else "invalid configuration"
            if self._h:
                self._L.b2v_destroy(self._h)
                self._h = C.c_void_p()
            raise RuntimeError(f"b2v_create failed (status {rc}): {msg}")
        # Inputs the library may still read (device tensors, pinned host memory), by storage address, until a
        # synchronising call; see HELD_INPUT_BYTES_MAX.
        self._held, self._held_bytes = {}, 0
        self._input_event_set = False     # set_input_event named the next call's input event
        self._producer_event = None       # torch.cuda.Event: device inputs' producers on torch's current stream
        self._last_frames = 0             # frames of the most recent integrate call (last_stored_slots)

    # ---- lifetime ----
    def close(self):
        if getattr(self, "_h", None):
            self._L.b2v_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, what: str):
        if rc != _lib.B2V_OK:
            raise RuntimeError(f"{what} failed (status {rc}): {self._L.b2v_last_error(self._h).decode()}")

    def _order_after_producer(self, tensor, stream):
        """Device inputs without a caller stream are read on the library's streams, which do not wait for torch's:
        the call's input event is then recorded on torch's current stream, after the inputs' producers (unless
        set_input_event named one)."""
        if stream or self._input_event_set:
            return
        import torch
        if self._producer_event is None:
            self._producer_event = torch.cuda.Event()
        self._producer_event.record(torch.cuda.current_stream(tensor.device))
        self._check(self._L.b2v_set_input_event(self._h, C.c_void_p(self._producer_event.cuda_event)),
                    "b2v_set_input_event")

    def _to_hold(self, inputs) -> dict:
        """The storages of `inputs` the enqueued work may read after the call returns and that are not held yet:
        device tensors and pinned host memory (a freed block would be handed to the next allocation while queued
        kernels or copies still read it).  Pageable host arrays are staged before the call returns."""
        new = {}
        for x in inputs:
            t = x if _is_torch_cuda(x) else _pinned_owner(x)
            if t is not None and t.untyped_storage().data_ptr() not in self._held:
                new[t.untyped_storage().data_ptr()] = t
        return new

    def _release_held(self) -> int:
        """Wait for the work in flight and drop the inputs held for it, whatever the status (returned)."""
        rc = self._L.b2v_synchronize(self._h)
        self._held, self._held_bytes = {}, 0
        return rc

    # ---- integrate ----
    def integrate(self, depth, color=None, K=None, pose=None, stream=None, depth_scale=None):
        """north_star: `integrate(depth, color, K, pose)` with depth float32 [H,W] metres, colour
        uint8 RGB [H,W,3], K = (fx,fy,cx,cy) | 3x3, pose = Tcw 4x4 float64.
        Open3D style (tsdf.py:223): `integrate(rgbd, intrinsic, extrinsic)` where `rgbd` has
        `.color` / `.depth`.  Inputs may be numpy arrays or CUDA torch tensors.  Asynchronous.
        `stream`: optional cudaStream_t handle (int) to launch on; device inputs only.
        `depth_scale`: given with a RAW uint16 depth image (numpy) - it is uploaded as 16-bit and widened on the
        GPU to float32(depth) * float32(depth_scale), like `depth.astype(np.float32) * depth_factor`."""
        if hasattr(depth, "depth") and hasattr(depth, "color"):
            rgbd, K, pose = depth, color, K
            depth, color = rgbd.depth, rgbd.color
        if K is None or pose is None or color is None:
            raise RuntimeError("integrate(depth, color, K, pose): missing argument")
        K4 = _as_K4(K)
        T = np.ascontiguousarray(np.asarray(pose, dtype=np.float64).reshape(4, 4)).reshape(16)
        if _is_torch_cuda(depth):
            if not _is_torch_cuda(color):
                raise RuntimeError("depth and color must both be CUDA tensors or both host arrays")
            if str(depth.dtype) != "torch.float32" or str(color.dtype) != "torch.uint8":
                raise RuntimeError("depth must be float32 and color uint8")
            if not depth.is_contiguous() or not color.is_contiguous():
                raise RuntimeError("depth and color must be contiguous")
            H, W = int(depth.shape[0]), int(depth.shape[1])
            if depth.dim() != 2 or tuple(color.shape) != (H, W, 3):
                raise RuntimeError("depth must be [H,W] and color [H,W,3]")
            dp, cp = depth.data_ptr(), color.data_ptr()
        else:
            d = np.asarray(depth)
            c = np.asarray(color)
            if d.ndim != 2:
                raise RuntimeError("depth must have 2 dimensions [H,W]")
            if c.ndim != 3 or c.shape[2] != 3 or c.shape[:2] != d.shape:
                raise RuntimeError("color must be [H,W,3] with the depth image's size")
            if c.dtype != np.uint8:
                raise RuntimeError("color must be uint8 RGB")
            raw16 = depth_scale is not None and d.dtype == np.uint16
            if depth_scale is not None and not raw16:
                raise RuntimeError("depth_scale goes with a uint16 depth image")
            # reference: depth.astype(float32), base.py:1008-1017 (raw uint16 is widened on the GPU instead)
            d = np.ascontiguousarray(d) if raw16 else np.ascontiguousarray(d, dtype=np.float32)
            c = np.ascontiguousarray(c)
            H, W = d.shape
            dp, cp = d.ctypes.data, c.ctypes.data
            depth, color = d, c
            if raw16:
                self._enqueue("b2v_integrate_batch_u16", self._L.b2v_integrate_batch_u16,
                              (1, dp, float(depth_scale), cp, H, W, K4.ctypes.data, T.ctypes.data, None), (d, c), None)
                return
        if depth_scale is not None:
            raise RuntimeError("depth_scale is supported for host (numpy) uint16 depth images")
        self._enqueue("b2v_integrate_batch", self._L.b2v_integrate_batch,
                      (1, dp, cp, H, W, K4.ctypes.data, T.ctypes.data, C.c_void_p(stream) if stream else None),
                      (depth, color), stream)

    def integrate_batch(self, depths, colors, K, poses, stream=None, depth_scale=None):
        """n frames back to back (the rebuild(map) bulk path, base.py:1242-1318): depths [n,H,W] f32,
        colors [n,H,W,3] u8, poses [n,4,4] Tcw.  One C call enqueues every frame.  With `depth_scale`, depths
        is RAW uint16 [n,H,W] (numpy, or a CUDA uint16 / int16 tensor) widened on the GPU."""
        K4 = _as_K4(K)
        T = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(-1, 16))
        n = T.shape[0]
        raw16 = depth_scale is not None
        if _is_torch_cuda(depths):
            if not (depths.is_contiguous() and colors.is_contiguous()):
                raise RuntimeError("depths and colors must be contiguous")
            if raw16 and depths.element_size() != 2:
                raise RuntimeError("depth_scale goes with 16-bit depth images")
            H, W = int(depths.shape[1]), int(depths.shape[2])
            dp, cp = depths.data_ptr(), colors.data_ptr()
            inputs = (depths, colors)
        else:
            if raw16 and np.asarray(depths).dtype != np.uint16:
                raise RuntimeError("depth_scale goes with uint16 depth images")
            d = np.ascontiguousarray(depths) if raw16 else np.ascontiguousarray(depths, dtype=np.float32)
            c = np.ascontiguousarray(colors, dtype=np.uint8)
            if d.ndim != 3 or c.shape != d.shape + (3,) or d.shape[0] != n:
                raise RuntimeError("depths must be [n,H,W], colors [n,H,W,3], poses [n,4,4]")
            H, W = d.shape[1:]
            dp, cp = d.ctypes.data, c.ctypes.data
            inputs = (d, c)
        s = C.c_void_p(stream) if stream else None
        if raw16:
            self._enqueue("b2v_integrate_batch_u16", self._L.b2v_integrate_batch_u16,
                          (n, dp, float(depth_scale), cp, H, W, K4.ctypes.data, T.ctypes.data, s), inputs, stream)
        else:
            self._enqueue("b2v_integrate_batch", self._L.b2v_integrate_batch,
                          (n, dp, cp, H, W, K4.ctypes.data, T.ctypes.data, s), inputs, stream)

    def _enqueue(self, what, fn, args, inputs, stream):
        """One integrate entry point: device inputs are ordered after their producers, and the inputs the enqueued
        work reads are held."""
        new = self._to_hold(inputs)
        new_bytes = sum(t.untyped_storage().nbytes() for t in new.values())
        if new_bytes and self._held and self._held_bytes + new_bytes > HELD_INPUT_BYTES_MAX:
            # bounded: wait for the earlier calls and release their inputs first (only when this call brings new
            # storage: inputs that stay resident, such as a reused frame buffer, are held once and cost no wait).
            # A full pool is reported by the next synchronising call, as without this wait.
            rc = self._release_held()
            if rc not in (_lib.B2V_OK, _lib.B2V_ERR_CAPACITY):
                self._check(rc, "b2v_synchronize")
        if inputs and _is_torch_cuda(inputs[0]):
            self._order_after_producer(inputs[0], stream)
        self._last_frames = max(int(args[0]), 0)
        try:
            rc = fn(self._h, *args)
        finally:
            self._input_event_set = False     # one-shot: the call consumed it
        self._check(rc, what)
        self._held.update(new)
        self._held_bytes += new_bytes

    # ---- frame store (rebuild(map) from keyframes on the GPU) ----
    def set_frame_store(self, max_frames: int):
        """Keep the packed image of up to `max_frames` integrated frames on the GPU (8 bytes per pixel, 2.46 MB per
        640x480 frame), so that `integrate_stored` can integrate them again with new poses without their images.
        0 turns the store off (the default).  Frames are stored in call order while there is room, at the size of the
        first stored frame; nothing is evicted.  reset() and load_state() keep the store.  Empties the store and
        synchronises (b2v_set_frame_store)."""
        self._check(self._L.b2v_set_frame_store(self._h, int(max_frames)), "b2v_set_frame_store")

    def clear_frame_store(self):
        """Empty the frame store and release its memory; synchronises."""
        self._check(self._L.b2v_frame_store_clear(self._h), "b2v_frame_store_clear")

    def last_stored_slots(self) -> np.ndarray:
        """int32 [n]: the store slot of each frame of the most recent integrate / integrate_batch call, -1 where the
        frame was not stored (store off or full, another frame size; an integrate_stored call stores nothing)."""
        slots = np.full(self._last_frames, -1, np.int32)
        self._check(self._L.b2v_frame_store_last(self._h, slots.ctypes.data, len(slots)), "b2v_frame_store_last")
        return slots

    def frame_store_stats(self):
        """(frames the store holds, device bytes it has mapped for them)."""
        n, b = C.c_int64(0), C.c_int64(0)
        self._check(self._L.b2v_frame_store_stats(self._h, C.byref(n), C.byref(b)), "b2v_frame_store_stats")
        return int(n.value), int(b.value)

    def integrate_stored(self, slots, K, poses, stream=None):
        """Integrate stored frames again (slots from `last_stored_slots`) with poses [n,4,4] Tcw: the map equals
        the one `integrate_batch` of the same frames' images at those poses gives, bit for bit.  Asynchronous, like
        integrate_batch; there are no images to hold."""
        sl = np.ascontiguousarray(np.asarray(slots).reshape(-1), dtype=np.int32)
        K4 = _as_K4(K)
        T = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(-1, 16))
        if T.shape[0] != len(sl):
            raise RuntimeError("integrate_stored: one pose per slot")
        self._enqueue("b2v_integrate_stored", self._L.b2v_integrate_stored,
                      (len(sl), sl.ctypes.data, K4.ctypes.data, T.ctypes.data,
                       C.c_void_p(stream) if stream else None), (), stream)

    def synchronize(self):
        """Wait for the work in flight; the inputs held for it are released."""
        self._check(self._release_held(), "b2v_synchronize")

    def capacity(self):
        """(blocks the pool has storage for now, growths since creation); synchronises."""
        n, g = C.c_int64(0), C.c_int64(0)
        self._check(self._L.b2v_capacity(self._h, C.byref(n), C.byref(g)), "b2v_capacity")
        return int(n.value), int(g.value)

    def reset(self):
        """`self.volume.reset()` (tsdf.py:156; base.py:642)."""
        rc = self._L.b2v_reset(self._h)
        self._held, self._held_bytes = {}, 0
        self._check(rc, "b2v_reset")

    # ---- inspection ----
    def num_blocks(self) -> int:
        n = self._L.b2v_num_blocks(self._h)
        if n < 0:
            raise RuntimeError(self._L.b2v_last_error(self._h).decode())
        return int(n)

    def last_mesh_stats(self) -> dict:
        """How the most recent mesh / point extraction narrowed its work (b2v_last_mesh_stats)."""
        st = (C.c_int64 * 5)()
        self._check(self._L.b2v_last_mesh_stats(self._h, st), "b2v_last_mesh_stats")
        return dict(zip(("blocks", "candidate_tiles", "tiles_with_both_signs", "vertex_blocks", "triangle_blocks"),
                        (int(x) for x in st)))

    def last_frame_stats(self):
        t, n = C.c_int64(0), C.c_int64(0)
        self._check(self._L.b2v_last_frame_stats(self._h, C.byref(t), C.byref(n)), "b2v_last_frame_stats")
        return int(t.value), int(n.value)

    def counters(self):
        """(total (block, frame) updates, kernel launches) since create/reset."""
        u, k, b = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        self._check(self._L.b2v_counters(self._h, C.byref(u), C.byref(k), C.byref(b)), "b2v_counters")
        return int(u.value), int(k.value)

    def block_visits(self) -> int:
        """Blocks read + written since create/reset (== updates frame by frame; fewer when fused)."""
        u, k, b = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        self._check(self._L.b2v_counters(self._h, C.byref(u), C.byref(k), C.byref(b)), "b2v_counters")
        return int(b.value)

    def set_fusion(self, enable: bool):
        """integrate_batch: fuse groups of frames per block visit (default, see set_group_size) or go frame by frame."""
        self._check(self._L.b2v_set_fusion(self._h, 1 if enable else 0), "b2v_set_fusion")

    def set_input_event(self, cuda_event):
        """The next integrate / integrate_batch call's device frames are ready when `cuda_event` (a raw cudaEvent_t
        handle, e.g. `torch.cuda.Event.cuda_event`) fires; see b2v_set_input_event.  Without it, the device frames of
        a call without a stream wait for torch's current stream."""
        self._check(self._L.b2v_set_input_event(self._h, C.c_void_p(int(cuda_event))), "b2v_set_input_event")
        self._input_event_set = True

    def set_group_size(self, frames: int):
        """Frames per fused group of integrate_batch (1..32, default 16); results do not depend on it."""
        self._check(self._L.b2v_set_group_size(self._h, int(frames)), "b2v_set_group_size")

    def set_rectification(self, map_x, map_y, swap_rb: bool = False):
        """Install the undistortion maps of `cv2.initUndistortRectifyMap(K, D, None, new_K, (w, h), CV_32FC1)`
        (volumetric_integrator_base.py:766-778): integrate() then takes the RAW images and rectifies them on the
        GPU exactly like `cv2.remap` (colour bilinear, depth nearest; base.py:1034-1039).  `swap_rb=True` also
        converts BGR input to RGB (base.py:1054).  `None` maps remove the stage."""
        self._check(_set_rectification(self._L.b2v_set_rectification, self._h, map_x, map_y, swap_rb),
                    "b2v_set_rectification")

    def set_overlap(self, enable: bool):
        """Run allocate(f+1) concurrently with integrate(f) (default) or serialise them."""
        self._check(self._L.b2v_set_overlap(self._h, 1 if enable else 0), "b2v_set_overlap")

    def profile_enable(self, enable: bool = True):
        self._check(self._L.b2v_profile_enable(self._h, 1 if enable else 0), "b2v_profile_enable")

    def profile_read(self):
        """(allocate_ms, integrate_ms, frames, integrate launches) summed since the last read."""
        a, b, n, l = C.c_double(0), C.c_double(0), C.c_int64(0), C.c_int64(0)
        self._check(self._L.b2v_profile_read(self._h, C.byref(a), C.byref(b), C.byref(n), C.byref(l)),
                    "b2v_profile_read")
        return a.value, b.value, int(n.value), int(l.value)

    def last_touched_keys(self) -> np.ndarray:
        n = self._L.b2v_last_touched_keys(self._h, None, 0)
        keys = np.zeros((max(int(n), 0), 4), np.int32)
        if n > 0:
            self._L.b2v_last_touched_keys(self._h, keys.ctypes.data, int(n))
        return np.ascontiguousarray(keys[:, :3])

    def _raw_shape(self, n: int) -> tuple:
        """Shape of n blocks in the pool's raw layout as float32 words: [n,5,512] planes (tsdf, weight, r, g, b), or
        with float64 colour [n,4096], the tsdf and weight planes followed by the float64 r, g, b planes."""
        return (n, RAW_F64_WORDS) if self.color_float64 else (n, VOXEL_PLANES, BLOCK_VOXELS)

    def _export_blocks(self, empty):
        """(keys int32 [nb,4] = {x,y,z,0}, raw float32 blocks, `_raw_shape`) of every block in arrays
        `empty(shape, dtype name)` makes, host or device (b2v_export_blocks, which waits for the frames in flight)."""
        n = self._L.b2v_export_blocks(self._h, None, None, 0)
        if n < 0:
            raise RuntimeError(self._L.b2v_last_error(self._h).decode())
        keys, vox = empty((n, 4), "int32"), empty(self._raw_shape(n), "float32")
        ptr = (lambda a: a.data_ptr()) if hasattr(keys, "data_ptr") else (lambda a: a.ctypes.data)
        if n and self._L.b2v_export_blocks(self._h, ptr(keys), ptr(vox), n) != n:
            raise RuntimeError(self._L.b2v_last_error(self._h).decode())
        return keys, vox

    def dump_blocks(self):
        """Parity hook: keys int32 [nb,3], hashes uint64 [nb] (reference BlockKeyHash),
        vox float32 [nb,5,512] planes (tsdf, weight, r, g, b).  With float64 colour also rgb64 float64 [nb,3,512], the
        colours as the volume keeps them; vox then holds them rounded to float32."""
        d = self._export_state()
        out = dict(keys=d["keys"], hashes=_block_hashes(d["keys"]), vox=d["vox"])
        if self.color_float64:
            out["rgb64"] = d["rgb64"]
            out["vox"] = np.concatenate([d["vox"], d["rgb64"].astype(np.float32)], axis=1)
        return out

    def upload_blocks(self, keys, vox, rgb64=None):
        """Restore / seed blocks: keys int32 [n,3] (unique), vox float32 [n,5,512].  A float64-colour volume takes
        its colours from rgb64 float64 [n,3,512] (vox's colour planes are ignored) and requires it; a float32 volume
        refuses it (ValueError).  Every weight must lie in [0, 2^24] (include/b2v.h); otherwise RuntimeError and the
        volume is unchanged."""
        if (rgb64 is None) == self.color_float64:
            raise ValueError("upload_blocks: rgb64 is required by a float64-colour volume and refused by a float32 one")
        k = _keys4(keys)
        n = k.shape[0]
        x = np.ascontiguousarray(vox, np.float32).reshape(n, VOXEL_PLANES, BLOCK_VOXELS)
        if self.color_float64:
            x = _pack_f64_blocks(x[:, :2], np.asarray(rgb64, np.float64).reshape(n, 3, BLOCK_VOXELS))
        self._upload_raw(keys, x)

    def _upload_raw(self, keys, raw):
        """upload_blocks from keys int32 [n,3] and host blocks in the raw layout (`_raw_shape`)"""
        k = _keys4(keys)
        x = np.ascontiguousarray(raw, np.float32).reshape(self._raw_shape(k.shape[0]))
        self._check(self._L.b2v_upload_blocks(self._h, k.shape[0], k.ctypes.data, x.ctypes.data),
                    "b2v_upload_blocks")

    # ---- map state (_MapState) ----
    _STATE_KIND = "tsdf"

    def _state_config(self) -> dict:
        # The colour precision is recorded by float64-colour volumes only, so the files of float32 volumes keep the
        # configuration they had before the mode existed.  Either way a file of the other mode does not load: a
        # float32 file lacks color_f64, and a float64 file has an rgb64 array a float32 volume does not take.
        c = dict(voxel_size=np.float32(self.voxel_length), voxel_length=np.float64(self.voxel_length),
                 sdf_trunc=np.float32(self.sdf_trunc), sdf_trunc_d=np.float64(self.sdf_trunc),
                 depth_trunc=np.float32(self.depth_trunc), depth_stride=np.int32(self.depth_sampling_stride),
                 unit_resolution=np.int32(self.volume_unit_resolution))
        if self.color_float64:
            c["color_f64"] = np.int32(1)
        return c

    def _state_arrays(self) -> dict:
        """keys and vox [n,5,512] (float32 colour planes); a float64-colour volume keeps the tsdf and weight planes in
        vox [n,2,512] and its colours in rgb64 float64 [n,3,512]."""
        if self.color_float64:
            return dict(keys=(np.int32, (3,)), vox=(np.float32, (2, BLOCK_VOXELS)),
                        rgb64=(np.float64, (3, BLOCK_VOXELS)))
        return dict(keys=(np.int32, (3,)), vox=(np.float32, (VOXEL_PLANES, BLOCK_VOXELS)))

    def _state_capacity(self) -> int:
        return max(self.capacity_blocks, self.max_capacity_blocks)

    def _export_state(self) -> dict:
        keys4, raw = self._export_blocks(np.empty)
        keys = np.ascontiguousarray(keys4[:, :3])
        if not self.color_float64:
            return dict(keys=keys, vox=raw)
        vox, rgb64 = _split_f64_blocks(raw)
        return dict(keys=keys, vox=vox, rgb64=rgb64)

    def _clear_state(self) -> None:
        self.reset()

    def _check_blocks(self, blocks: dict) -> None:
        w = blocks["vox"][:, 1]
        if w.size and not np.all((w >= 0) & (w <= WEIGHT_MAX)):
            raise ValueError("voxel weights outside [0, 2^24] in the state")

    def _upload_state(self, blocks: dict) -> None:
        if not len(blocks["keys"]):
            return
        if self.color_float64:
            self._upload_raw(blocks["keys"], _pack_f64_blocks(blocks["vox"], blocks["rgb64"]))
        else:
            self.upload_blocks(blocks["keys"], blocks["vox"])

    def export_blocks_torch(self):
        """(keys int32 [n,4] = {x,y,z,0}, vox float32 [n,5,512]) as torch CUDA tensors on this volume's device:
        device-to-device copies of the block keys and the block pool (multi-GPU mesh gather).  A float64-colour
        volume's vox is its raw layout, float32 [n,4096] (tsdf and weight planes, then the float64 r, g, b planes)."""
        import torch
        dev = torch.device("cuda", self.device)
        return self._export_blocks(lambda shape, dt: torch.empty(shape, dtype=getattr(torch, dt), device=dev))

    def import_blocks_torch(self, keys, vox):
        """Inverse of export_blocks_torch: contiguous torch CUDA tensors on this volume's device, read in place."""
        if keys.shape[0] == 0:
            return
        if not (keys.is_cuda and vox.is_cuda and keys.is_contiguous() and vox.is_contiguous()):
            raise RuntimeError("keys and vox must be contiguous CUDA tensors")
        if tuple(vox.shape) != self._raw_shape(int(keys.shape[0])):
            raise ValueError(f"vox must be the raw layout {self._raw_shape(int(keys.shape[0]))} of this volume")
        self._check(self._L.b2v_upload_blocks(self._h, int(keys.shape[0]), keys.data_ptr(), vox.data_ptr()),
                    "b2v_upload_blocks")

    # ---- outputs ----
    def extract_mesh(self) -> TriangleMesh:
        """north_star `extract_mesh()` == Open3D `extract_triangle_mesh()` (tsdf.py:239,260)."""
        nv, nt = C.c_int64(0), C.c_int64(0)
        self._check(self._L.b2v_extract_mesh(self._h, C.byref(nv), C.byref(nt)), "b2v_extract_mesh")
        return self._copy_mesh(nv.value, nt.value)

    extract_triangle_mesh = extract_mesh

    # ---- sharded extraction: face-halo exchange (pyslam_b200.sharding.extract_mesh_sharded) ----
    def export_halo_torch(self, world: int):
        """Halo records this shard sends the other ranks of a `world`-rank sharding (b2v_export_halo_device):
        (headers int32 [R,4] = {x,y,z,mask}, payload float32 [P,5] = {tsdf, weight, r, g, b}, records per destination
        rank, payload voxels per destination rank), CUDA tensors grouped by destination rank.  With float64 colour the
        payload is float32 [P,8]: tsdf, weight and the r, g, b float64 words.  Only reads the volume."""
        import torch
        world = int(world)
        rec, pay = (C.c_int64 * world)(), (C.c_int64 * world)()
        self._check(self._L.b2v_export_halo_device(self._h, world, rec, pay, None, None, 0, 0), "b2v_export_halo_device")
        nrec, nvox = [int(x) for x in rec], [int(x) for x in pay]
        dev = torch.device("cuda", self.device)
        headers = torch.empty((sum(nrec), 4), dtype=torch.int32, device=dev)
        payload = torch.empty((sum(nvox), self._halo_words), dtype=torch.float32, device=dev)
        if headers.shape[0]:
            self._check(self._L.b2v_export_halo_device(self._h, world, rec, pay, headers.data_ptr(), payload.data_ptr(),
                                                       headers.shape[0], payload.shape[0]), "b2v_export_halo_device")
        return headers, payload, nrec, nvox

    @property
    def _halo_words(self) -> int:
        """float32 words per voxel of a halo payload"""
        return HALO_F64_WORDS if self.color_float64 else VOXEL_PLANES

    def _halo_args(self, headers, payload):
        import torch
        dev = torch.device("cuda", self.device)
        h = torch.as_tensor(headers, dtype=torch.int32).to(dev).contiguous().reshape(-1, 4)
        x = torch.as_tensor(payload, dtype=torch.float32).to(dev).contiguous().reshape(-1, self._halo_words)
        torch.cuda.current_stream(dev).synchronize()
        return h, x

    def extract_mesh_with_halo(self, headers, payload) -> TriangleMesh:
        """The mesh piece rooted in this shard's blocks, given the halo records the other ranks sent it
        (b2v_extract_mesh_with_halo).  Seam vertices may repeat in other ranks' pieces; `sharding.weld` merges them."""
        h, x = self._halo_args(headers, payload)
        nv, nt = C.c_int64(0), C.c_int64(0)
        self._check(self._L.b2v_extract_mesh_with_halo(self._h, h.shape[0], h.data_ptr(), x.data_ptr(), C.byref(nv),
                                                       C.byref(nt)), "b2v_extract_mesh_with_halo")
        return self._copy_mesh(nv.value, nt.value)

    def extract_point_cloud_with_halo(self, headers, payload) -> PointCloud:
        """The zero crossings rooted in this shard's blocks (b2v_extract_points_with_halo): the ranks' pieces are
        disjoint and together make the unsharded volume's point cloud."""
        h, x = self._halo_args(headers, payload)
        n = C.c_int64(0)
        self._check(self._L.b2v_extract_points_with_halo(self._h, h.shape[0], h.data_ptr(), x.data_ptr(), C.byref(n)),
                    "b2v_extract_points_with_halo")
        m = self._copy_mesh(n.value, 0)
        return PointCloud(m.vertices, m.vertex_colors, m.edge_ids)

    def _copy_mesh(self, nv: int, nt: int) -> TriangleMesh:
        """The result of the last extraction (b2v_copy_mesh), float64 like Open3D's TriangleMesh."""
        V = np.zeros((nv, 3), np.float64)
        Cc = np.zeros((nv, 3), np.float64)
        E = np.zeros((nv, 4), np.int32)
        T = np.zeros((nt, 3), np.int32)
        self._check(self._L.b2v_copy_mesh(self._h, V.ctypes.data, Cc.ctypes.data, E.ctypes.data, T.ctypes.data),
                    "b2v_copy_mesh")
        return TriangleMesh(V, T, Cc, E)

    def extract_point_cloud(self) -> PointCloud:
        n = C.c_int64(0)
        self._check(self._L.b2v_extract_points(self._h, C.byref(n)), "b2v_extract_points")
        m = self._copy_mesh(n.value, 0)
        return PointCloud(m.vertices, m.vertex_colors, m.edge_ids)


# float64-colour blocks (include/b2v.h B2V_BLOCK_BYTES_F64) as float32 words, and a halo payload voxel of such a volume
RAW_F64_WORDS = 2 * BLOCK_VOXELS + 3 * 2 * BLOCK_VOXELS
HALO_F64_WORDS = 2 + 3 * 2


def _split_f64_blocks(raw):
    """float64-colour blocks, float32 [n,4096] -> (vox float32 [n,2,512] tsdf and weight, rgb64 float64 [n,3,512])"""
    raw = np.ascontiguousarray(raw, np.float32)
    n = raw.shape[0]
    vox = raw[:, :2 * BLOCK_VOXELS].reshape(n, 2, BLOCK_VOXELS).copy()
    rgb64 = raw[:, 2 * BLOCK_VOXELS:].view(np.float64).reshape(n, 3, BLOCK_VOXELS).copy()
    return vox, rgb64


def _pack_f64_blocks(tw, rgb64):
    """Inverse of _split_f64_blocks: tw float32 [n,2,512] (tsdf, weight), rgb64 float64 [n,3,512] -> [n,4096]"""
    n = tw.shape[0]
    raw = np.empty((n, RAW_F64_WORDS), np.float32)
    raw[:, :2 * BLOCK_VOXELS] = np.asarray(tw, np.float32).reshape(n, 2 * BLOCK_VOXELS)
    raw[:, 2 * BLOCK_VOXELS:].view(np.float64)[:] = np.asarray(rgb64, np.float64).reshape(n, 3 * BLOCK_VOXELS)
    return raw


def filter_shadow_points(depth, delta_depth=None, delta_x=2, delta_y=2, fill_value=-1, device=0):
    """GPU version of `pyslam.utilities.depth.filter_shadow_points` (depth.py:103-146) for the default
    `delta_depth=None` (median-based threshold).  depth float32 [H,W] -> filtered copy."""
    if delta_depth is not None:
        raise NotImplementedError("only the median-based threshold (delta_depth=None) is implemented")
    d = np.ascontiguousarray(depth, dtype=np.float32)
    if d.ndim != 2:
        raise RuntimeError("depth must be a 2D array")
    out = np.empty_like(d)
    rc = _lib.load().b2v_filter_shadow_points(d.ctypes.data, d.shape[0], d.shape[1], int(delta_x), int(delta_y),
                                             float(fill_value), out.ctypes.data, int(device))
    if rc != _lib.B2V_OK:
        raise RuntimeError(f"b2v_filter_shadow_points failed (status {rc})")
    return out


def remap(src, map_x, map_y, interpolation="linear", swap_rb=False, device=0):
    """GPU `cv2.remap(src, map_x, map_y, interpolation)` for the two cases the dense front-end uses
    (volumetric_integrator_base.py:1017-1047): uint8 [H,W,3] with INTER_LINEAR, and float32 / int32 [H,W] with
    INTER_NEAREST; constant zero border.  Bit-exact with OpenCV's fixed-point arithmetic."""
    a = np.ascontiguousarray(src)
    mx = np.ascontiguousarray(map_x, np.float32)
    my = np.ascontiguousarray(map_y, np.float32)
    if a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3 and interpolation == "linear":
        kind = 0
    elif a.dtype in (np.float32, np.int32) and a.ndim == 2 and interpolation == "nearest":
        kind = 1
    else:
        raise RuntimeError("remap supports uint8 [H,W,3] + 'linear' and float32/int32 [H,W] + 'nearest'")
    if mx.shape != a.shape[:2] or my.shape != a.shape[:2]:
        raise RuntimeError("maps must have the image's height and width")
    out = np.empty_like(a)
    rc = _lib.load().b2v_remap(a.ctypes.data, kind, a.shape[0], a.shape[1], mx.ctypes.data, my.ctypes.data,
                              out.ctypes.data, 1 if swap_rb else 0, int(device))
    if rc != _lib.B2V_OK:
        raise RuntimeError(f"b2v_remap failed (status {rc})")
    return out


class DeviceImage:
    """One image a grid's `set_frame` staged on the device (or the object image of `remap_instance_ids`): memory the
    grid owns, valid until that grid stages its next frame or is closed.  The grid's `integrate_rgbd`, `carve` and
    `assign_object_ids_to_instance_ids` accept it in place of an array and read it where it is.  `torch()` is a
    zero-copy CUDA tensor view, `numpy()` a host copy."""

    def __init__(self, grid, ptr, shape, dtype):
        self._grid, self._gen = grid, grid._frame_gen
        self.ptr, self.shape, self.dtype = int(ptr), tuple(int(s) for s in shape), np.dtype(dtype)

    def _ptr_for(self, grid, dtype=None):
        if grid is not self._grid:
            raise RuntimeError("a staged image can only be used with the grid that staged it")
        if self._gen != grid._frame_gen or not grid._h:
            raise RuntimeError("stale staged image: its grid has staged a newer frame or was closed")
        if dtype is not None and self.dtype != np.dtype(dtype):
            raise RuntimeError(f"staged image of dtype {self.dtype} where {np.dtype(dtype)} is expected")
        return self.ptr

    @property
    def __cuda_array_interface__(self):
        return {"shape": self.shape, "typestr": self.dtype.str, "data": (self._ptr_for(self._grid), False),
                "strides": None, "version": 3}

    def torch(self):
        import torch
        self._ptr_for(self._grid)   # raise here: torch.as_tensor would report a stale image as an unknown type
        return torch.as_tensor(self, device=torch.device("cuda", self._grid.device))

    def numpy(self) -> np.ndarray:
        return self.torch().cpu().numpy()


class GridFrame:
    """What `set_frame` staged: `depth` (rectified, float32 metres), `filtered_depth` (after the shadow-point filter;
    the same image as `depth` when the filter is off), `color` (rectified RGB uint8) and, on semantic grids,
    `class_image` / `instance_image` (int32, None when not given) and `object_image` (set by `remap_instance_ids`)."""

    def __init__(self, grid, f):
        hw = (int(f.height), int(f.width))
        self.height, self.width = hw
        self.depth = DeviceImage(grid, f.depth, hw, np.float32)
        self.filtered_depth = (self.depth if f.filtered_depth == f.depth
                               else DeviceImage(grid, f.filtered_depth, hw, np.float32))
        self.color = DeviceImage(grid, f.color, hw + (3,), np.uint8)
        self.class_image = DeviceImage(grid, f.class_image, hw, np.int32) if f.class_image else None
        self.instance_image = DeviceImage(grid, f.instance_image, hw, np.int32) if f.instance_image else None
        self.object_image = None


def _image_arg(grid, a, dtype, hold, convert=True):
    """(pointer, shape, dtype) of an image argument: a DeviceImage staged by `grid` is read in place, anything else
    becomes a contiguous host array (of `dtype` when `convert`) kept alive in `hold`."""
    if isinstance(a, DeviceImage):
        return a._ptr_for(grid, dtype if convert else None), a.shape, a.dtype
    b = np.ascontiguousarray(a, dtype) if convert else np.ascontiguousarray(a)
    hold.append(b)
    return b.ctypes.data, b.shape, b.dtype


def _set_rectification(fn, h, map_x, map_y, swap_rb):
    """Status of `fn(h, map_x, map_y, H, W, swap_rb)`, a set_rectification entry point: the maps as float32 [H,W]
    arrays of one shape, or NULL when either is None (which removes the stage)."""
    if map_x is None or map_y is None:
        return fn(h, None, None, 0, 0, 0)
    mx = np.ascontiguousarray(map_x, np.float32)
    my = np.ascontiguousarray(map_y, np.float32)
    if mx.ndim != 2 or mx.shape != my.shape:
        raise RuntimeError("map_x and map_y must be float32 [H,W] arrays of the same shape")
    return fn(h, mx.ctypes.data, my.ctypes.data, mx.shape[0], mx.shape[1], 1 if swap_rb else 0)


def _frame_input(a, dtype, name, hold):
    """Pointer of one set_frame input: a contiguous CUDA tensor of `dtype` in place, or a host array."""
    if _is_torch_cuda(a):
        if str(a.dtype) != f"torch.{np.dtype(dtype).name}" or not a.is_contiguous():
            raise RuntimeError(f"{name} must be a contiguous {np.dtype(dtype).name} tensor")
        hold.append(a)
        return a.data_ptr(), tuple(a.shape), True
    b = np.ascontiguousarray(a, dtype)
    hold.append(b)
    return b.ctypes.data, b.shape, False


class CameraFrustrum:
    """Mirror of `volumetric.CameraFrustrum(fx, fy, cx, cy, width, height, T_cw, depth_max, depth_min)`
    (cpp/volumetric/camera_frustrum.h:36-48): the arguments of carve / frustum queries."""

    def __init__(self, fx, fy, cx, cy, width, height, T_cw=None, depth_max=10.0, depth_min=1e-2):
        self.fx, self.fy, self.cx, self.cy = float(fx), float(fy), float(cx), float(cy)
        self.width, self.height = int(width), int(height)
        self.depth_max, self.depth_min = float(depth_max), float(depth_min)
        self.T_cw = np.eye(4) if T_cw is None else np.asarray(T_cw, np.float64).reshape(4, 4)

    def set_T_cw(self, T_cw):
        self.T_cw = np.asarray(T_cw, np.float64).reshape(4, 4)

    def get_width(self):
        return self.width

    def get_height(self):
        return self.height

    def _args(self):
        K = np.array([self.fx, self.fy, self.cx, self.cy], np.float32)
        T = np.ascontiguousarray(self.T_cw, np.float64).reshape(16)
        return K, T


class BoundingBox3D:
    """Mirror of `volumetric.BoundingBox3D(min_x, min_y, min_z, max_x, max_y, max_z)`
    (cpp/volumetric/bounding_boxes_3d.h:40-80)."""

    def __init__(self, min_x, min_y, min_z, max_x, max_y, max_z):
        self.bounds = np.array([min_x, min_y, min_z, max_x, max_y, max_z], np.float64)


class TBBUtils:
    """`volumetric.TBBUtils` of the reference module (cpp/volumetric/volumetric_module.cpp:43-50): the integrators call
    `TBBUtils.set_max_threads(n)` to size the CPU thread pool of the voxel grids.  The GPU grids have no CPU pool; the
    value is kept so that `get_max_threads()` answers what was set."""
    _max_threads = 0

    @staticmethod
    def set_max_threads(num_threads: int) -> None:
        TBBUtils._max_threads = int(num_threads)

    @staticmethod
    def get_max_threads() -> int:
        import os
        return TBBUtils._max_threads if TBBUtils._max_threads > 0 else (os.cpu_count() or 1)


class VoxelGridData:
    """`VoxelGridDataT` (cpp/volumetric/voxel_grid_data.h:36-50): points / colors SoA."""

    def __init__(self, points, colors):
        self.points = points
        self.colors = colors
        self.class_ids = None
        self.object_ids = None
        self.confidences = None


class _BlockGrid(_MapState):
    """What the point-average and the semantic grids share: the library handle and its lifetime, the checks of
    `integrate`'s points and colours, the frame stage, carving and the read-outs both grids answer alike.  A subclass
    names its entry points by their prefix `_P` and stages frames with `_stage_frame`."""

    _P = ""
    # block sides the grids take (pySLAM's kVolumetricIntegrationBlockSize): powers of two, so the block key stays a
    # shift and the local key a mask; 4 keeps the rejection every size but 8 had before block sizes were supported
    SUPPORTED_BLOCK_SIZES = (1, 2, 8, 16)

    def __init__(self, voxel_size, block_size, capacity_blocks, device, max_capacity_blocks, shard_rank, shard_count,
                 *kind):
        self._L = _lib.load()
        self._h = C.c_void_p()
        self.voxel_size = float(voxel_size)
        self._block_size = int(block_size)
        self._block_voxels = self._block_size ** 3   # voxels per block: the per-voxel axis of dumps and uploads
        self.capacity_blocks = int(capacity_blocks)
        self.max_capacity_blocks = int(max_capacity_blocks or 0)
        self.device = int(device)
        self._frame_gen, self._frame = 0, None
        rc = self._c("create_ex")(float(voxel_size), int(block_size), int(capacity_blocks), self.max_capacity_blocks,
                                  *kind, int(device), C.byref(self._h))
        if rc != _lib.B2V_OK:
            msg = self._c("last_error")(self._h).decode() if self._h else (
                "invalid configuration (block_size must be one of "
                f"{', '.join(map(str, self.SUPPORTED_BLOCK_SIZES))}; got {block_size})"
                if self._block_size not in self.SUPPORTED_BLOCK_SIZES else "invalid configuration")
            if self._h:
                self._c("destroy")(self._h)
                self._h = C.c_void_p()
            raise RuntimeError(f"{self._P}create failed (status {rc}): {msg}")
        self.shard_rank, self.shard_count = 0, 1
        self.set_shard(shard_rank, shard_count)

    def _c(self, name):
        """The grid's entry point `name` (without the prefix)."""
        return getattr(self._L, self._P + name)

    def close(self):
        if getattr(self, "_h", None):
            self._c("destroy")(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != _lib.B2V_OK:
            raise RuntimeError(f"{what} failed (status {rc}): {self._c('last_error')(self._h).decode()}")

    @staticmethod
    def _points_colors(points, colors):
        """(points, colours, colours are uint8) of `integrate`, checked like the reference
        (volumetric_grid_module.h:140-258): points float32 | float64 [N,3]; colours None, uint8 [N,3] or float [N,3]
        (as float32).  Both contiguous."""
        pts = np.asarray(points)
        if pts.ndim != 2 or pts.shape[1] != 3:
            raise RuntimeError("points must be a 2D array with shape (N, 3)")
        if pts.dtype not in (np.float32, np.float64):
            raise RuntimeError("points must be float32 or float64")
        pts = np.ascontiguousarray(pts)
        if colors is None or np.asarray(colors).size == 0:
            return pts, None, 0
        cols = np.asarray(colors)
        if cols.ndim != 2 or cols.shape[1] != 3:
            raise RuntimeError("colors must be a 2D array with shape (N, 3)")
        if cols.shape[0] != pts.shape[0]:
            raise RuntimeError("points and colors must have the same number of rows")
        if cols.dtype == np.uint8:
            return pts, np.ascontiguousarray(cols), 1
        if cols.dtype in (np.float32, np.float64):
            return pts, np.ascontiguousarray(cols, dtype=np.float32), 0
        raise RuntimeError("colors must be uint8 or float32")

    def set_rectification(self, map_x, map_y, swap_rb: bool = False):
        """Install the undistortion maps of `cv2.initUndistortRectifyMap(..., CV_32FC1)` for `set_frame`, which then
        rectifies on the device exactly like `cv2.remap` (colour bilinear, depth and the semantic grids' class and
        instance images nearest); `swap_rb=True` also converts BGR colour to RGB.  `None` maps remove the stage.  See
        B200TsdfVolume.set_rectification."""
        self._check(_set_rectification(self._c("set_rectification"), self._h, map_x, map_y, swap_rb),
                    "set_rectification")

    def set_frame(self, depth, color, class_image=None, instance_image=None, depth_scale=None,
                  filter_shadow_points=False) -> GridFrame:
        """Stage one raw camera frame on the device: each image is uploaded once (numpy) or read in place (contiguous
        CUDA tensors), raw uint16 depth with `depth_scale` is widened to `depth.astype(float32) * depth_scale`, the
        images are rectified with the installed maps, and `filter_shadow_points=True` computes the filtered depth
        once.  Returns a `GridFrame` whose images `integrate_rgbd` and `carve` accept; they stay valid until the
        next `set_frame`.  Bit-identical to preparing the frame on the host with cv2 and numpy.  The label images
        `class_image` / `instance_image` (int32 [H,W], or anything numpy casts to it) belong to the semantic grids,
        where they are staged too and feed `assign_object_ids_to_instance_ids` and `remap_instance_ids`."""
        hold = []
        u16 = depth_scale is not None
        if u16 and not _is_torch_cuda(depth) and np.asarray(depth).dtype != np.uint16:
            raise RuntimeError("depth_scale goes with a uint16 depth image")
        dp, shape, dev_d = _frame_input(depth, np.uint16 if u16 else np.float32, "depth", hold)
        if len(shape) != 2:
            raise RuntimeError("depth must be [H,W]")
        cp, cshape, dev_c = _frame_input(color, np.uint8, "color", hold)
        if cshape != shape + (3,):
            raise RuntimeError("color must be uint8 [H,W,3] with the depth image's size")
        labels, on_device = [], dev_d or dev_c
        for img, name in ((class_image, "class_image"), (instance_image, "instance_image")):
            if img is None or (not _is_torch_cuda(img) and np.asarray(img).size == 0):
                labels.append(None)
                continue
            p, lshape, dev = _frame_input(img, np.int32, name, hold)
            if lshape != shape:
                raise RuntimeError(f"{name} must have the depth image's shape")
            labels.append(p)
            on_device = on_device or dev
        if on_device:   # the library reads device inputs on its own stream
            import torch
            torch.cuda.synchronize()
        f = _lib.B2VFrame()
        rc = self._stage_frame((dp, 1 if u16 else 0, float(depth_scale) if u16 else 0.0, cp), labels, shape,
                               1 if filter_shadow_points else 0, C.byref(f))
        if rc != _lib.B2V_ERR_INVALID_ARGUMENT:
            self._frame_gen += 1   # the previous frame's images are gone
            self._frame = None
        self._check(rc, "set_frame")
        self._frame = GridFrame(self, f)
        return self._frame

    # ---- frame store (rebuild(map) from keyframes on the GPU) ----
    def set_frame_store(self, max_frames: int):
        """Keep what `set_frame` staged for up to `max_frames` frames on the GPU, so that `stage_stored` can stage them
        again without their images: 8 bytes per pixel on the point-average grid (2.46 MB per 640x480 frame), 16 on the
        semantic grids (4.9 MB).  0 turns the store off (the default).  Frames are stored in call order while there is
        room, at the size of the first stored frame; nothing is evicted.  clear() and load_state() keep the store.
        Empties the store and synchronises."""
        self._check(self._c("set_frame_store")(self._h, int(max_frames)), self._P + "set_frame_store")

    def clear_frame_store(self):
        """Empty the frame store and release its memory; synchronises."""
        self._check(self._c("frame_store_clear")(self._h), self._P + "frame_store_clear")

    def last_stored_slot(self) -> int:
        """The store slot of the most recent `set_frame`'s frame, or -1 (store off or full, another frame size, or a
        failing call)."""
        s = C.c_int32(-1)
        self._check(self._c("frame_store_last")(self._h, C.byref(s)), self._P + "frame_store_last")
        return int(s.value)

    def frame_store_stats(self):
        """(frames the store holds, device bytes it has mapped for them)."""
        n, b = C.c_int64(0), C.c_int64(0)
        self._check(self._c("frame_store_stats")(self._h, C.byref(n), C.byref(b)), self._P + "frame_store_stats")
        return int(n.value), int(b.value)

    def stage_stored(self, slot: int) -> GridFrame:
        """Stage stored frame `slot` again (from `last_stored_slot`): the `GridFrame` the frame's `set_frame` returned,
        its images bit for bit the same, so carving, the association, `remap_instance_ids` and `integrate_rgbd` give
        the same map.  Like `set_frame`, earlier staged images go stale; a slot the store does not hold raises and
        leaves the staged frame as it was."""
        f = _lib.B2VFrame()
        rc = self._c("stage_stored")(self._h, int(slot), C.byref(f))
        if rc != _lib.B2V_ERR_INVALID_ARGUMENT:
            self._frame_gen += 1
            self._frame = None
        self._check(rc, self._P + "stage_stored")
        self._frame = GridFrame(self, f)
        return self._frame

    def carve(self, camera_frustrum, depth_image, depth_threshold: float = 1e-2):
        """carve(camera_frustrum, depth_image, depth_threshold) (voxel_block_grid.hpp:616-622): reset voxels
        in the frustum that lie in front of the observed depth by more than the threshold.  Like the
        reference (voxel_grid_carving.h:51-58) an empty or wrongly sized image is a soft failure.  depth_image may
        be an image of a staged frame (`set_frame`)."""
        d = depth_image if isinstance(depth_image, DeviceImage) else np.asarray(depth_image)
        if d.shape != (camera_frustrum.height, camera_frustrum.width) or not np.prod(d.shape):
            print("volumetric::carve: depth image is empty or has the wrong size")
            return
        hold = []
        dp, _, _ = _image_arg(self, d, np.float32, hold)
        K, T = camera_frustrum._args()
        self._check(self._c("carve")(self._h, K.ctypes.data, camera_frustrum.width, camera_frustrum.height,
                                     T.ctypes.data, camera_frustrum.depth_max, camera_frustrum.depth_min,
                                     dp, float(depth_threshold)), self._P + "carve")

    def get_points(self):
        return self.get_voxels(1).points

    def get_colors(self):
        return self.get_voxels(1).colors

    def set_shard(self, shard_rank: int, shard_count: int):
        """Hash sharding over `shard_count` ranks, like `B200TsdfVolume(shard_rank=, shard_count=)`: from now on the
        grid keeps only the blocks with `BlockKeyHash(key) % shard_count == shard_rank` (`sharding.owner_of`).  Feed
        every rank every frame; each rank then holds, voxel for voxel, the blocks of the unsharded grid it owns, and
        the edits apply per rank.  `pyslam_b200.sharding` gathers the read-outs and runs the association.  Only on a
        grid without blocks; raises otherwise, or for a bad rank or count, and changes nothing.  `clear` keeps it."""
        self._check(self._c("set_shard")(self._h, int(shard_rank), int(shard_count)), self._P + "set_shard")
        self.shard_rank, self.shard_count = int(shard_rank), int(shard_count)

    def clear(self):
        """Empties the grid; grown storage and the shard setting are kept."""
        self._check(self._c("clear")(self._h), self._P + "clear")

    reset = clear

    def capacity(self):
        """(blocks the grid has storage for now, growths since creation); synchronises."""
        n, g = C.c_int64(0), C.c_int64(0)
        self._check(self._c("capacity")(self._h, C.byref(n), C.byref(g)), self._P + "capacity")
        return int(n.value), int(g.value)

    def num_blocks(self) -> int:
        n = self._c("num_blocks")(self._h)
        if n < 0:
            raise RuntimeError(f"{self._P}num_blocks failed")
        return int(n)

    def empty(self) -> bool:
        return self.num_blocks() == 0

    def get_block_size(self) -> int:
        return self._block_size

    # ---- map state (_MapState): the grid's kind adds its arrays, `_export_state` and `_upload_state` ----
    _STATE_BOUNDS = {"count": (0, None)}

    def _state_config(self) -> dict:
        return dict(voxel_size=np.float64(self.voxel_size), block_size=np.int32(self._block_size))

    def _state_capacity(self) -> int:
        return max(self.capacity_blocks, self.max_capacity_blocks)

    def _clear_state(self) -> None:
        self.clear()


class VoxelBlockGrid(_BlockGrid):
    """GPU drop-in for pySLAM's `volumetric.VoxelBlockGrid(voxel_size, block_size=8)`."""

    _P = "b2v_grid_"

    def __init__(self, voxel_size: float, block_size: int = 8, capacity_blocks: int = 1 << 17,
                 device: int = 0, max_capacity_blocks: int | None = None, shard_rank: int = 0, shard_count: int = 1,
                 input_order_sums: bool = False):
        """`max_capacity_blocks`: growth ceiling of the block pool.  Above `capacity_blocks`, the pool starts with
        `capacity_blocks` blocks of storage and grows inside the integrate call that needs more; the grid then holds
        what a grid created with `capacity_blocks=max_capacity_blocks` holds.  None (or `capacity_blocks`) keeps the
        pool fixed.  `shard_rank` / `shard_count`: see `set_shard`.

        `input_order_sums`: each voxel adds its points in input order with IEEE float32 adds instead of float atomics,
        so the position and colour sums equal the sequential reference's bit for bit and are the same on every run, in
        every shard layout and after every growth.  Off (the default), the sums equal the reference's up to the order
        of the atomic adds, which no two runs share; keys, hashes and counts are the same either way.  A call in this
        mode takes at most 0x7FFFFFF0 points.  Saved map states load into a grid of either mode."""
        super().__init__(voxel_size, block_size, capacity_blocks, device, max_capacity_blocks, shard_rank, shard_count)
        self._input_order_sums = bool(input_order_sums)
        if self._input_order_sums:
            rc = self._L.b2v_grid_set_input_order_sums(self._h, 1)
            if rc != _lib.B2V_OK:
                msg = self._L.b2v_grid_last_error(self._h).decode()
                self.close()
                raise RuntimeError(f"input_order_sums: {msg} (status {rc})")

    @property
    def input_order_sums(self) -> bool:
        """True when each voxel sums its points in input order (see the constructor)."""
        return self._input_order_sums

    def _stage_frame(self, images, labels, shape, filter_shadow_points, out):
        if labels[0] is not None or labels[1] is not None:
            raise NotImplementedError("label images need a semantic grid")
        return self._L.b2v_grid_set_frame(self._h, *images, shape[0], shape[1], filter_shadow_points, out)

    def integrate(self, points, colors=None, class_ids=None, instance_ids=None, depths=None):
        """integrate(points [N,3] f32|f64, colors [N,3] u8|f32 | None)
        (volumetric_grid_module.h:131-467).  float64 points take the reference's float64 overload (:737-749): voxel
        keys from the float64 coordinates, sums accumulate float32(x); uint8 colours are scaled on the device by the
        float32 constant 1/255 exactly as voxel_data.h:82-85 does (b2v_grid_integrate_ex)."""
        if class_ids is not None or instance_ids is not None or depths is not None:
            raise NotImplementedError("semantic integration is a SURVEY.md §8(f) 'next' row")
        pts, cols, cu8 = self._points_colors(points, colors)
        self._check(self._L.b2v_grid_integrate_ex(self._h, pts.ctypes.data, 1 if pts.dtype == np.float64 else 0,
                                                  None if cols is None else cols.ctypes.data, cu8, pts.shape[0]),
                    "b2v_grid_integrate_ex")
        self._check(self._L.b2v_grid_synchronize(self._h), "b2v_grid_synchronize")

    def integrate_rgbd(self, depth, color, K, Twc, max_depth=np.inf, min_depth=0.0, filter_shadow_points=False):
        """Fused front-end of `VolumetricIntegratorVoxelGrid.volume_integration`
        (volumetric_integrator_voxel_grid.py:247-300): `depth2pointcloud(depth, color, fx, fy, cx, cy,
        max_depth)` + `Twc` transform + `integrate(points, colors)` in one GPU call.  depth float32 [H,W]
        metres, color uint8 RGB [H,W,3], Twc = inv_T(pose) 4x4 float64.  `filter_shadow_points=True` applies
        the reference's shadow-point filter first (kVolumetricIntegrationVoxelGridShadowPointsFilter,
        voxel_grid.py:236-245).  depth / color may be the images of a staged frame (`set_frame`)."""
        hold = []
        dp, dshape, _ = _image_arg(self, depth, np.float32, hold)
        cp, cshape, cdt = _image_arg(self, color, np.uint8, hold, convert=False)
        if len(dshape) != 2 or cshape != tuple(dshape) + (3,) or cdt != np.uint8:
            raise RuntimeError("depth must be float32 [H,W] and color uint8 [H,W,3]")
        K4 = _as_K4(K)
        T = np.ascontiguousarray(np.asarray(Twc, np.float64).reshape(4, 4)).reshape(16)
        mx = float(np.finfo(np.float32).max) if not np.isfinite(max_depth) else float(max_depth)
        self._check(self._L.b2v_grid_integrate_rgbd(self._h, dp, cp, dshape[0], dshape[1],
                                                    K4.ctypes.data, T.ctypes.data, mx, float(min_depth),
                                                    1 if filter_shadow_points else 0),
                    "b2v_grid_integrate_rgbd")
        self._check(self._L.b2v_grid_synchronize(self._h), "b2v_grid_synchronize")

    def get_voxels(self, min_count: int = 1, min_confidence: float = 0.0) -> VoxelGridData:
        """get_voxels(min_count, min_confidence): min_confidence is ignored for the non-semantic grid,
        as in the reference (voxel_block_grid.hpp:750-752)."""
        return self._collect(self._L.b2v_grid_get_voxels(self._h, int(min_count)))

    def size(self) -> int:
        return int(self._L.b2v_grid_size(self._h))

    def get_total_voxel_count(self) -> int:
        return self.size()

    def remove_low_count_voxels(self, min_count: int):
        self._check(self._L.b2v_grid_remove_low_count_voxels(self._h, int(min_count)),
                    "b2v_grid_remove_low_count_voxels")

    def remove_low_confidence_voxels(self, min_confidence: float):
        # no-op for the non-semantic grid, as in the reference (voxel_block_grid.hpp:650-676)
        return None

    _STATE_KIND = "grid"
    _PLANES = 7   # a pool block's 32-bit planes of B^3 voxels: count (int32), pos_sum x, y, z, col_sum r, g, b

    def _state_arrays(self) -> dict:
        v = self._block_voxels
        return dict(keys=(np.int32, (3,)), count=(np.int32, (v,)), pos_sum=(np.float32, (v, 3)),
                    col_sum=(np.float32, (v, 3)))

    def _export_state(self) -> dict:
        """keys int32 [nb,3], count int32 [nb,B^3], pos_sum / col_sum float32 [nb,B^3,3] of every block, from the
        pool blocks of b2v_grid_export_blocks."""
        nb = self.num_blocks()
        keys4 = np.empty((nb, 4), np.int32)
        raw = np.empty((nb, self._PLANES, self._block_voxels), np.uint32)
        n = self._L.b2v_grid_export_blocks(self._h, keys4.ctypes.data, raw.ctypes.data)
        if n != nb:
            raise RuntimeError(f"b2v_grid_export_blocks returned {n}, expected {nb}")

        def xyz(p):
            return np.ascontiguousarray(raw[:, p:p + 3].transpose(0, 2, 1)).view(np.float32)
        return dict(keys=np.ascontiguousarray(keys4[:, :3]), count=np.ascontiguousarray(raw[:, 0]).view(np.int32),
                    pos_sum=xyz(1), col_sum=xyz(4))

    def _upload_state(self, blocks: dict) -> None:
        b = blocks
        n, v = len(b["keys"]), self._block_voxels
        raw = np.empty((n, self._PLANES, v), np.uint32)
        raw[:, 0] = np.asarray(b["count"], np.int32).reshape(n, v).view(np.uint32)
        for p, name in ((1, "pos_sum"), (4, "col_sum")):
            raw[:, p:p + 3] = np.asarray(b[name], np.float32).reshape(n, v, 3).view(np.uint32).transpose(0, 2, 1)
        keys4 = _keys4(b["keys"])
        self._check(self._L.b2v_grid_upload_blocks(self._h, n, keys4.ctypes.data, raw.ctypes.data),
                    "b2v_grid_upload_blocks")

    def dump_blocks(self):
        """Parity hook: keys int32 [nb,3], hashes uint64 [nb] (reference BlockKeyHash), count int32 [nb,B^3],
        pos_sum / col_sum float32 [nb,B^3,3]."""
        d = self._export_state()
        return dict(keys=d["keys"], hashes=_block_hashes(d["keys"]), count=d["count"], pos_sum=d["pos_sum"],
                    col_sum=d["col_sum"])

    # ---- spatial queries and carving (SURVEY.md §8(f) rank 3) ----
    def _collect(self, n):
        if n < 0:
            raise RuntimeError(self._L.b2v_grid_last_error(self._h).decode())
        P = np.zeros((n, 3), np.float32)
        Cc = np.zeros((n, 3), np.float32)
        self._check(self._L.b2v_grid_copy_voxels(self._h, P.ctypes.data, Cc.ctypes.data), "b2v_grid_copy_voxels")
        return VoxelGridData(P, Cc)

    def get_voxels_in_camera_frustrum(self, camera_frustrum, min_count: int = 1, min_confidence: float = 0.0):
        K, T = camera_frustrum._args()
        return self._collect(self._L.b2v_grid_get_voxels_in_frustum(
            self._h, K.ctypes.data, camera_frustrum.width, camera_frustrum.height, T.ctypes.data,
            camera_frustrum.depth_max, camera_frustrum.depth_min, int(min_count)))

    def get_voxels_in_bb(self, bbox, min_count: int = 1, min_confidence: float = 0.0):
        bb = np.ascontiguousarray(getattr(bbox, "bounds", bbox), np.float64).reshape(6)
        return self._collect(self._L.b2v_grid_get_voxels_in_bb(self._h, bb.ctypes.data, int(min_count)))


class OrientedBoundingBox3D:
    """`volumetric.OrientedBoundingBox3D` fields: center [3], size [3], orientation (unit quaternion w, x, y, z of the
    box -> world rotation).  `compute_from_points` is the reference's PCA method (bounding_boxes_3d.cpp:373-556):
    running centroid / covariance (Welford) in float64, eigenvectors sorted by descending eigenvalue, right-handed,
    extents from the min / max of the points in that frame."""

    def __init__(self, center=None, size=None, rotation=None):
        self.center = np.zeros(3) if center is None else np.asarray(center, np.float64)
        self.size = np.zeros(3) if size is None else np.asarray(size, np.float64)
        self.R = np.eye(3) if rotation is None else np.asarray(rotation, np.float64)

    @property
    def orientation(self):
        return _quat_wxyz(self.R)

    def get_matrix(self):
        M = np.eye(4)
        M[:3, :3], M[:3, 3] = self.R, self.center
        return M

    def get_corners(self):
        h = self.size / 2.0
        sg = np.array([[1, 1, -1], [-1, 1, -1], [-1, -1, -1], [1, -1, -1], [1, 1, 1], [-1, 1, 1], [-1, -1, 1], [1, -1, 1]], float)
        return self.center + (sg * h) @ self.R.T

    @staticmethod
    def compute_from_points(points):
        P = np.asarray(points, np.float64).reshape(-1, 3)
        n = len(P)
        if n == 0:
            return OrientedBoundingBox3D()
        if n == 1:
            return OrientedBoundingBox3D(P[0], np.zeros(3), np.eye(3))
        if n == 2:
            c, diff = 0.5 * (P[0] + P[1]), P[1] - P[0]
            dn = np.linalg.norm(diff)
            if dn < 1e-10:
                return OrientedBoundingBox3D(c, np.zeros(3), np.eye(3))
            a1 = diff / dn
            ref = np.array([1.0, 0, 0]) if abs(a1[0]) < 0.9 else np.array([0, 1.0, 0])
            a2 = np.cross(ref, a1)
            a2 /= np.linalg.norm(a2)
            a3 = np.cross(a1, a2)
            a3 /= np.linalg.norm(a3)
            R = np.stack([a1, a2, a3], axis=1)
            if np.linalg.det(R) < 0:
                R[:, 2] = -R[:, 2]
            centroid = c
        else:
            # the reference's one-pass Welford update equals the two-pass centroid / covariance up to rounding
            centroid = P.mean(axis=0)
            d = P - centroid
            cov = d.T @ d / n
            w, V = np.linalg.eigh(cov)
            R = V[:, np.argsort(-w, kind="stable")]
            if np.dot(np.cross(R[:, 0], R[:, 1]), R[:, 2]) < 0:
                R[:, 2] = -R[:, 2]
        local = (P - centroid) @ R
        lo, hi = local.min(axis=0), local.max(axis=0)
        return OrientedBoundingBox3D(centroid + R @ (0.5 * (hi + lo)), hi - lo, R)


def _quat_wxyz(R):
    """Rotation matrix -> unit quaternion (w, x, y, z), Eigen's branch order."""
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        q = [0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s]
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0) * 2
        q = [0.0] * 4
        q[0] = (R[k, j] - R[j, k]) / s
        q[1 + i] = 0.25 * s
        q[1 + j] = (R[j, i] + R[i, j]) / s
        q[1 + k] = (R[k, i] + R[i, k]) / s
    return np.array(q)


class ObjectData:
    """`volumetric.ObjectData` (voxel_grid_data.h:64-79)."""

    def __init__(self, object_id, class_id, points, colors, confidence_min, confidence_max):
        self.object_id, self.class_id = int(object_id), int(class_id)
        self.points, self.colors = points, colors
        self.confidence_min, self.confidence_max = confidence_min, confidence_max
        self.oriented_bounding_box = OrientedBoundingBox3D.compute_from_points(points)


class ObjectDataGroup:
    """`volumetric.ObjectDataGroup` (voxel_grid_data.h:87-96)."""

    def __init__(self, objects):
        self.object_vector = objects
        self.class_ids = [o.class_id for o in objects]
        self.object_ids = [o.object_id for o in objects]


class ClassData:
    """`volumetric.ClassData` (voxel_grid_data.h:110-125)."""

    def __init__(self, class_id, points, colors, confidence_min, confidence_max):
        self.class_id = int(class_id)
        self.points, self.colors = points, colors
        self.confidence_min, self.confidence_max = confidence_min, confidence_max


class ClassDataGroup:
    """`volumetric.ClassDataGroup` (voxel_grid_data.h:127-140)."""

    def __init__(self, classes):
        self.class_vector = classes
        self.class_ids = [c.class_id for c in classes]


def segment_min_count(min_count: int) -> int:
    """The `get_voxels` min_count of the segments' voxels: the reference keeps voxels with count > min_count (strict,
    unlike get_voxels' >=) and confidence >= min_confidence; the GPU read-out (count -> scan -> emit) does the scan
    and the compaction, `segments` the grouping."""
    return int(min_count) + 1


def segments(v: VoxelGridData, by_class: bool):
    """The voxels of a semantic read-out grouped by object id (ObjectDataGroup) or class id (ClassDataGroup), ids < 0
    dropped, stable: the read-out's order within a segment is kept (voxel_block_semantic_grid.hpp:204-316)."""
    ids = np.asarray(v.class_ids if by_class else v.object_ids)
    keep = ids >= 0                                   # negative = uninitialised label
    pts, cols = np.asarray(v.points)[keep], np.asarray(v.colors)[keep]
    cls, conf, ids = np.asarray(v.class_ids)[keep], np.asarray(v.confidences)[keep], ids[keep]
    order = np.argsort(ids, kind="stable")
    uniq, start = np.unique(ids[order], return_index=True)
    bounds = list(start) + [len(order)]
    out = []
    for k, seg_id in enumerate(uniq):
        sel = order[bounds[k]:bounds[k + 1]]
        cmin, cmax = float(conf[sel].min()), float(conf[sel].max())
        if by_class:
            out.append(ClassData(int(seg_id), pts[sel], cols[sel], cmin, cmax))
        else:
            out.append(ObjectData(int(seg_id), int(cls[sel[0]]), pts[sel], cols[sel], cmin, cmax))
    return ClassDataGroup(out) if by_class else ObjectDataGroup(out)


class VoxelBlockSemanticGrid(_BlockGrid):
    """GPU drop-in for `volumetric.VoxelBlockSemanticGrid(voxel_size, block_size=8)` — per-voxel label
    *voting* (cpp/volumetric/voxel_block_semantic_grid.h:59-118; voxel_data_semantic.h:106-199).

    integrate(points, colors, class_ids, instance_ids, depths) -> get_voxels(min_count, min_confidence) with
    `class_ids / object_ids / confidences`.  Observations reach a voxel in input order (the reference's
    deterministic build), so labels, counters, float64 position sums and float32 colour sums are bit-identical."""

    KIND = _lib.B2V_SEM_VOTING
    _P = "b2v_sgrid_"

    def __init__(self, voxel_size: float = 0.05, block_size: int = 8, capacity_blocks: int = 1 << 14,
                 device: int = 0, max_capacity_blocks: int | None = None, shard_rank: int = 0, shard_count: int = 1,
                 max_label_overflow_pairs: int = 0, initial_label_overflow_pairs: int | None = None):
        """`max_capacity_blocks`: growth ceiling (at most 2^22 blocks).  Above `capacity_blocks`, the per-voxel storage
        starts with `capacity_blocks` blocks and grows inside the integrate call that needs more; the grid then holds,
        bit for bit, what a grid created with `capacity_blocks=max_capacity_blocks` holds.  None (or
        `capacity_blocks`) keeps the storage fixed.  `shard_rank` / `shard_count`: see `set_shard`; the association
        of a sharded grid runs over all ranks (`sharding.assign_object_ids_to_instance_ids_sharded`).

        `max_label_overflow_pairs` (Bayesian grid only; a non-zero value raises RuntimeError on the voting grid):
        ceiling of the overflow label store, in (object, class) pairs past the 8 a voxel holds itself, shared by all
        voxels and rounded up to chunks of 8.  Below it no voxel evicts a pair and the grid equals the reference's
        unbounded label map; past it the integrate call evicts as without a store and raises ("label storage full").
        0 (the default) is the grid without a store.  The store's storage starts with `initial_label_overflow_pairs`
        (None: the ceiling, at most 2^17 pairs) and grows inside the integrate call that needs more."""
        super().__init__(voxel_size, block_size, capacity_blocks, device, max_capacity_blocks, shard_rank, shard_count,
                         self.KIND)
        max_pairs = int(max_label_overflow_pairs)
        if max_pairs < 0:
            raise RuntimeError("max_label_overflow_pairs must be >= 0")
        if max_pairs:
            first = min(max_pairs, 1 << 17) if initial_label_overflow_pairs is None else int(initial_label_overflow_pairs)
            rc = self._L.b2v_sgrid_set_label_overflow(self._h, max_pairs, max(0, first))
            if rc != _lib.B2V_OK:
                msg = self._L.b2v_sgrid_last_error(self._h).decode()
                self.close()
                raise RuntimeError(f"max_label_overflow_pairs: {msg} (status {rc})")
        # mirrors of the library's settings (class defaults, voxel_data_semantic.h:107-108, 251-254), for save_state
        self._depth_threshold = np.float32(10.0 if self.KIND == _lib.B2V_SEM_VOTING else 5.0)
        self._depth_decay_rate = np.float32(0.07)

    def _stage_frame(self, images, labels, shape, filter_shadow_points, out):
        return self._L.b2v_sgrid_set_frame(self._h, *images, *labels, shape[0], shape[1], filter_shadow_points, out)

    # ---- parameters (class-static in the reference, per grid here) ----
    def set_depth_threshold(self, depth_threshold: float):
        self._check(self._L.b2v_sgrid_set_depth_threshold(self._h, float(depth_threshold)), "set_depth_threshold")
        self._depth_threshold = np.float32(depth_threshold)

    def set_depth_decay_rate(self, depth_decay_rate: float):
        """Only the Bayesian grid has a decay rate (semantic_grid.hpp:31-36); the voting grid ignores it."""
        self._check(self._L.b2v_sgrid_set_depth_decay_rate(self._h, float(depth_decay_rate)), "set_depth_decay_rate")
        if self.KIND == _lib.B2V_SEM_PROBABILISTIC:
            self._depth_decay_rate = np.float32(depth_decay_rate)

    # ---- map state (_MapState): the raw slots of b2v_sgrid_export_blocks, the settings and next_object_id ----
    _STATE_KIND = "semantic"
    _STATE_ARRAYS = ("count", "pos_sum", "col_sum", "object_id", "class_id", "counter", "ml_logp", "conf", "lab_obj",
                     "lab_cls", "lab_logp")   # the order of b2v_sgrid_export_blocks / _upload_blocks

    def _state_semantic_kind(self) -> int:
        return self.KIND

    @property
    def _STATE_BOUNDS(self):
        bounds = {"count": (0, None)}
        if self.KIND == _lib.B2V_SEM_PROBABILISTIC:   # the number of label slots in use
            bounds["counter"] = (0, _lib.B2V_SEM_MAX_LABELS)
        return bounds

    def _state_settings(self) -> dict:
        return dict(depth_threshold=self._depth_threshold, depth_decay_rate=self._depth_decay_rate,
                    next_object_id=np.int32(self.get_next_object_id()))

    def _restore_settings(self, settings: dict) -> None:
        self.set_depth_threshold(settings["depth_threshold"])
        self.set_depth_decay_rate(settings["depth_decay_rate"])
        self.set_next_object_id(int(settings["next_object_id"]))

    def _state_arrays(self) -> dict:
        v, k = self._block_voxels, _lib.B2V_SEM_MAX_LABELS
        spec = dict(keys=(np.int32, (3,)), count=(np.int32, (v,)), pos_sum=(np.float64, (v, 3)),
                    col_sum=(np.float32, (v, 3)), object_id=(np.int32, (v,)), class_id=(np.int32, (v,)),
                    counter=(np.int32, (v,)))
        if self.KIND == _lib.B2V_SEM_PROBABILISTIC:
            spec.update(ml_logp=(np.float32, (v,)), conf=(np.float32, (v,)), lab_obj=(np.int32, (v, k)),
                        lab_cls=(np.int32, (v, k)), lab_logp=(np.float32, (v, k)))
        return spec

    def export_blocks(self) -> dict:
        """The raw state of every block (b2v_sgrid_export_blocks): keys [nb,3] and per-voxel arrays [nb,B^3,...] -
        count, pos_sum (float64), col_sum, object_id, class_id, counter (the voting counter, or the number of label
        pairs) and, on the Bayesian grid, ml_logp, conf and the label slots lab_obj / lab_cls / lab_logp
        [nb,B^3,8] in the kernel's own order.  Unlike `dump_blocks`, nothing is derived or reordered."""
        spec = self._state_arrays()
        nb = self.num_blocks()
        d = {name: np.zeros((nb,) + shape, dt) for name, (dt, shape) in spec.items()}
        if nb:
            keys4 = np.zeros((nb, 4), np.int32)
            ptrs = [d[name].ctypes.data if name in d else None for name in self._STATE_ARRAYS]
            n = self._L.b2v_sgrid_export_blocks(self._h, keys4.ctypes.data, *ptrs)
            if n != nb:
                raise RuntimeError(f"b2v_sgrid_export_blocks returned {n}, expected {nb}: "
                                   f"{self._L.b2v_sgrid_last_error(self._h).decode()}")
            d["keys"] = np.ascontiguousarray(keys4[:, :3])
        return d

    _export_state = export_blocks

    @property
    def _STATE_LABELS(self):
        return self.KIND == _lib.B2V_SEM_PROBABILISTIC

    def export_labels(self) -> dict:
        """The overflow label pairs (b2v_sgrid_export_labels): count int32 [nb,B^3] (each voxel's pairs past its 8
        in-voxel slots, in the block order of `export_blocks`) and obj / cls int32, logp float32 [total], voxel after
        voxel, each voxel's in slot order."""
        nb = self.num_blocks()
        count = np.zeros((nb, self._block_voxels), np.int32)
        total = self._L.b2v_sgrid_export_labels(self._h, count.ctypes.data, None, None, None)
        if total < 0:
            raise RuntimeError(f"b2v_sgrid_export_labels failed: {self._L.b2v_sgrid_last_error(self._h).decode()}")
        out = dict(count=count, obj=np.zeros(total, np.int32), cls=np.zeros(total, np.int32),
                   logp=np.zeros(total, np.float32))
        if total:
            n = self._L.b2v_sgrid_export_labels(self._h, count.ctypes.data, out["obj"].ctypes.data,
                                                out["cls"].ctypes.data, out["logp"].ctypes.data)
            if n != total:
                raise RuntimeError(f"b2v_sgrid_export_labels returned {n}, expected {total}")
        return out

    def _export_labels(self):
        """The overflow pairs for the state file; None (the file of a grid without them) when no voxel has any."""
        return self.export_labels() if self.label_storage()["used"] else None

    def _check_labels(self, labels: dict) -> None:
        """ValueError, before the map changes, when the label store's ceiling cannot hold the file's pairs."""
        need = int(((labels["count"].astype(np.int64) + 7) // 8).sum())
        have = self.label_storage()["max"]
        if need > have:
            raise ValueError(f"the state holds overflow label pairs in {need} chunks of 8 for this grid, more than its "
                             f"max_label_overflow_pairs ceiling of {have} chunks")

    def _upload_labels(self, keys, labels: dict) -> None:
        n, keys4 = len(keys), _keys4(keys)
        arrs = [np.ascontiguousarray(labels[k]) for k in ("count", "obj", "cls", "logp")]
        self._check(self._L.b2v_sgrid_upload_labels(self._h, n, keys4.ctypes.data if n else None,
                                                    *[a.ctypes.data if a.size else None for a in arrs]),
                    "b2v_sgrid_upload_labels")

    def _upload_state(self, blocks: dict) -> None:
        n, keys4 = len(blocks["keys"]), _keys4(blocks["keys"])
        ptrs = [blocks[name].ctypes.data if name in blocks and n else None for name in self._STATE_ARRAYS]
        self._check(self._L.b2v_sgrid_upload_blocks(self._h, n, keys4.ctypes.data if n else None, *ptrs),
                    "b2v_sgrid_upload_blocks")

    # ---- integrate (volumetric_grid_module.h: integrate(points, colors, class_ids, instance_ids, depths)) ----
    def integrate(self, points, colors=None, class_ids=None, instance_ids=None, depths=None):
        pts, cols, cu8 = self._points_colors(points, colors)
        n = pts.shape[0]
        hold = []

        def opt(a, dt, name):
            if a is None or np.asarray(a).size == 0:
                return None
            b = np.ascontiguousarray(a, dtype=dt).reshape(-1)
            if b.shape[0] != n:
                raise RuntimeError(f"points and {name} must have the same size")
            hold.append(b)
            return b.ctypes.data

        ci = opt(class_ids, np.int32, "class_ids")
        ii = opt(instance_ids, np.int32, "instance_ids")
        di = opt(depths, np.float32, "depths")
        if ii is not None and ci is None:
            raise RuntimeError("instance_ids but no class_ids is not supported")  # voxel_block_grid.hpp:43-46
        self._check(self._L.b2v_sgrid_integrate(self._h, n, pts.ctypes.data, 1 if pts.dtype == np.float64 else 0,
                                                None if cols is None else cols.ctypes.data, cu8, ci, ii, di),
                    "b2v_sgrid_integrate")

    def integrate_segment(self, points, colors, class_id: int, object_id: int):
        """`integrate_segment(points, colors, class_id, object_id)` (volumetric_grid_module.h:97-125, 564-590 ->
        voxel_block_semantic_grid.hpp:52-99): every point carries the same (class, object) label; a negative id
        skips the whole segment."""
        pts = np.asarray(points)
        cols = np.asarray(colors)
        if pts.ndim != 2 or pts.shape[1] != 3:
            raise RuntimeError("points must be a contiguous Nx3 array")
        if cols.ndim != 2 or cols.shape[1] != 3:
            raise RuntimeError("colors must be a contiguous Nx3 array")
        if cols.shape[0] != pts.shape[0]:
            raise RuntimeError("points and colors must have the same size")
        if int(object_id) < 0 or int(class_id) < 0 or pts.shape[0] == 0:
            return
        n = pts.shape[0]
        self.integrate(pts, cols, np.full(n, int(class_id), np.int32), np.full(n, int(object_id), np.int32))

    # ---- segments (voxel_block_semantic_grid.hpp:204-316) ----
    def get_object_segments(self, min_count: int = 1, min_confidence: float = 0.0):
        """`get_object_segments(min_count, min_confidence)` -> ObjectDataGroup (voxel_grid_data.h:64-96): voxels grouped
        by object id (ids < 0 dropped), each with its points / colours, the class id of its first voxel, the
        confidence range and a PCA oriented bounding box (bounding_boxes_3d.cpp:373-556, the reference's default
        OBBComputationMethod::PCA)."""
        return segments(self.get_voxels(segment_min_count(min_count), float(min_confidence)), by_class=False)

    def get_class_segments(self, min_count: int = 1, min_confidence: float = 0.0):
        """`get_class_segments(min_count, min_confidence)` -> ClassDataGroup (voxel_grid_data.h:110-140)."""
        return segments(self.get_voxels(segment_min_count(min_count), float(min_confidence)), by_class=True)

    def integrate_rgbd(self, depth, color, K, Twc, class_image=None, object_image=None, max_depth=np.inf,
                       min_depth=0.0, use_depths=True, filter_shadow_points=False):
        """The reference integrator's per-frame front-end fused on the GPU
        (volumetric_integrator_voxel_semantic_grid.py:332-461): optional `filter_shadow_points`, `depth2pointcloud`
        with the class / object-id images, world transform by `Twc` (camera -> world), `integrate`.  `use_depths`
        mirrors kVolumetricSemanticProbabilisticIntegrationUseDepth.  color is RGB uint8.  Every image may be one of
        a staged frame (`set_frame`, `remap_instance_ids`)."""
        hold = []
        dp, dshape, _ = _image_arg(self, depth, np.float32, hold)
        cp, cshape, _ = _image_arg(self, color, np.uint8, hold)
        if len(dshape) != 2 or cshape != tuple(dshape) + (3,):
            raise RuntimeError("depth must be [H,W] float32 and color [H,W,3] uint8")

        def img(a, name):
            if a is None or (not isinstance(a, DeviceImage) and np.asarray(a).size == 0):
                return None
            p, shape, _ = _image_arg(self, a, np.int32, hold)
            if shape != dshape:
                raise RuntimeError(f"{name} must have the depth image's shape")
            return p

        ci, oi = img(class_image, "class_image"), img(object_image, "object_image")
        K4 = _as_K4(K)
        T = np.ascontiguousarray(np.asarray(Twc, np.float64).reshape(16))
        md = float(np.finfo(np.float32).max) if not np.isfinite(max_depth) else float(max_depth)
        self._check(self._L.b2v_sgrid_integrate_rgbd(self._h, dp, cp, ci, oi, dshape[0],
                                                     dshape[1], K4.ctypes.data, T.ctypes.data, md, float(min_depth),
                                                     1 if use_depths else 0, 1 if filter_shadow_points else 0),
                    "b2v_sgrid_integrate_rgbd")

    def remap_instance_ids(self) -> DeviceImage:
        """`remap_instance_ids(frame.instance_image, map)` on the device, with the map of the last
        `assign_object_ids_to_instance_ids`: ids missing from the map, and every pixel when it is empty, become -1.
        Returns the object image (also the staged frame's `object_image`), valid like the frame's other images."""
        out = C.c_void_p()
        self._check(self._L.b2v_sgrid_remap_instance_ids(self._h, C.byref(out)), "b2v_sgrid_remap_instance_ids")
        f = self._frame
        f.object_image = DeviceImage(self, out.value, (f.height, f.width), np.int32)
        return f.object_image

    # ---- read-outs ----
    def get_voxels(self, min_count: int = 1, min_confidence: float = 0.0) -> VoxelGridData:
        return self._collect(self._L.b2v_sgrid_get_voxels(self._h, int(min_count), float(min_confidence)))

    def get_voxels_in_bb(self, bbox, min_count: int = 1, min_confidence: float = 0.0) -> VoxelGridData:
        bb = np.ascontiguousarray(getattr(bbox, "bounds", bbox), np.float64).reshape(6)
        return self._collect(self._L.b2v_sgrid_get_voxels_in_bb(self._h, bb.ctypes.data, int(min_count),
                                                                float(min_confidence)))

    def get_voxels_in_camera_frustrum(self, camera_frustrum, min_count: int = 1,
                                      min_confidence: float = 0.0) -> VoxelGridData:
        K, T = camera_frustrum._args()
        return self._collect(self._L.b2v_sgrid_get_voxels_in_frustum(
            self._h, K.ctypes.data, camera_frustrum.width, camera_frustrum.height, T.ctypes.data,
            camera_frustrum.depth_max, camera_frustrum.depth_min, int(min_count), float(min_confidence)))

    def _collect(self, n) -> VoxelGridData:
        if n < 0:
            raise RuntimeError(self._L.b2v_sgrid_last_error(self._h).decode())
        out = VoxelGridData(np.zeros((n, 3), np.float64), np.zeros((n, 3), np.float32))
        out.class_ids = np.zeros(n, np.int32)
        out.object_ids = np.zeros(n, np.int32)
        out.confidences = np.zeros(n, np.float32)
        if n:
            self._check(self._L.b2v_sgrid_copy_voxels(self._h, out.points.ctypes.data, out.colors.ctypes.data,
                                                      out.class_ids.ctypes.data, out.object_ids.ctypes.data,
                                                      out.confidences.ctypes.data), "b2v_sgrid_copy_voxels")
        return out

    def get_ids(self):
        """(class_ids, object_ids) of every non-empty voxel (voxel_block_semantic_grid.hpp:185-202)."""
        v = self.get_voxels(1, -np.inf)
        return v.class_ids, v.object_ids

    def size(self) -> int:
        return len(self.get_voxels(1, -np.inf).points)

    def remove_low_count_voxels(self, min_count: int):
        self._check(self._L.b2v_sgrid_remove_low_count_voxels(self._h, int(min_count)), "remove_low_count_voxels")

    def remove_low_confidence_segments(self, min_confidence: int):
        """The reference takes an `int` threshold (voxel_block_semantic_grid.h:103)."""
        self._check(self._L.b2v_sgrid_remove_low_confidence_segments(self._h, int(min_confidence)),
                    "remove_low_confidence_segments")

    def merge_segments(self, instance_id1: int, instance_id2: int):
        self._check(self._L.b2v_sgrid_merge_segments(self._h, int(instance_id1), int(instance_id2)), "merge_segments")

    def remove_segment(self, object_id: int):
        self._check(self._L.b2v_sgrid_remove_segment(self._h, int(object_id)), "remove_segment")

    def assign_object_ids_to_instance_ids(self, camera_frustrum, class_ids_image, semantic_instances_image,
                                          depth_image=None, depth_threshold: float = 0.1, do_carving: bool = False,
                                          min_vote_ratio: float = 0.5, min_votes: int = 3) -> dict:
        """`MapInstanceIdToObjectId` of the frame (voxel_block_semantic_grid.h:67-71;
        voxel_semantic_data_association.h:69-373): 2-D instance id -> 3-D object id (-1: no confident match).
        Soft failures (empty / wrongly sized label images) return an empty map like the reference (:80-103).  The
        images may be those of a staged frame (`set_frame`)."""
        hold = []
        imgs = self._assoc_images((camera_frustrum.height, camera_frustrum.width), class_ids_image,
                                  semantic_instances_image, depth_image, hold)
        if imgs is None:
            return {}
        K, T = camera_frustrum._args()
        n = self._L.b2v_sgrid_assign_object_ids_to_instance_ids(
            self._h, K.ctypes.data, camera_frustrum.width, camera_frustrum.height, T.ctypes.data,
            camera_frustrum.depth_max, camera_frustrum.depth_min, *imgs,
            float(depth_threshold), 1 if do_carving else 0, float(min_vote_ratio), int(min_votes))
        return self._instance_map(n)

    def _assoc_images(self, hw, class_ids_image, semantic_instances_image, depth_image, hold):
        """(class, instance, depth or None) image pointers of an association of [H,W] = `hw` images, or None (printed)
        when the label images are empty or wrongly sized, a soft failure like the reference's (:80-103)."""
        def arr(a):
            return a if isinstance(a, DeviceImage) else np.asarray(a)

        ci, ii = arr(class_ids_image), arr(semantic_instances_image)
        if not np.prod(ci.shape) or not np.prod(ii.shape) or ci.shape != hw or ii.shape != hw:
            print("volumetric::assign_object_ids_to_instance_ids: label images are empty or have the wrong size")
            return None
        cp, _, _ = _image_arg(self, ci, np.int32, hold)
        ip, _, _ = _image_arg(self, ii, np.int32, hold)
        dp = None
        if depth_image is not None:
            d = arr(depth_image)
            if np.prod(d.shape) and d.shape == hw:
                dp, _, _ = _image_arg(self, d, np.float32, hold)
        return cp, ip, dp

    def _instance_map(self, n) -> dict:
        """The map an association call left (its return value `n`: size or -1) as a dict."""
        if n < 0:
            raise RuntimeError(self._L.b2v_sgrid_last_error(self._h).decode())
        ids, objs = np.zeros(n, np.int32), np.zeros(n, np.int32)
        self._check(self._L.b2v_sgrid_copy_instance_map(self._h, ids.ctypes.data, objs.ctypes.data),
                    "b2v_sgrid_copy_instance_map")
        return {int(i): int(o) for i, o in zip(ids, objs)}

    def set_next_object_id(self, next_object_id: int):
        self._check(self._L.b2v_sgrid_set_next_object_id(self._h, int(next_object_id)), "set_next_object_id")

    def get_next_object_id(self) -> int:
        return int(self._L.b2v_sgrid_get_next_object_id(self._h))

    def label_overflows(self) -> int:
        out = C.c_uint64(0)
        self._check(self._L.b2v_sgrid_label_overflows(self._h, C.byref(out)), "b2v_sgrid_label_overflows")
        return int(out.value)

    def label_storage(self) -> dict:
        """The overflow label store in chunks of 8 pairs: `used` (in some voxel's chain), `mapped` (with storage),
        `max` (the ceiling; 0 without a store) and `growths` of its storage."""
        v = [C.c_int64(0) for _ in range(4)]
        self._check(self._L.b2v_sgrid_label_storage(self._h, *map(C.byref, v)), "b2v_sgrid_label_storage")
        return dict(zip(("used", "mapped", "max", "growths"), (int(x.value) for x in v)))

    def dump_blocks(self, K: int | None = None):
        """Parity hook: per-block arrays [nb,B^3,...] derived from `export_blocks` and `export_labels` - keys,
        hashes (reference BlockKeyHash), count, pos_sum, col_sum, object_id, class_id, confidence (the Bayesian
        `conf`; on the voting grid min(float32(counter) / float32(count), 1), 0 without points), aux (`counter`) and
        lab_obj / lab_cls / lab_logp [nb,B^3,K]: a Bayesian voxel's label pairs, in-voxel slots then overflow chain,
        stably sorted by (object, class), the first K, padded with (-1, -1, -inf).  K: None gives the largest pair
        count of a voxel (at least 8)."""
        raw = self.export_blocks()
        nb, nv = raw["count"].shape
        bayes = self.KIND == _lib.B2V_SEM_PROBABILISTIC
        counter = raw["counter"]
        if K is None:
            K = max(_lib.B2V_SEM_MAX_LABELS, int(counter.max()) if bayes and nb else 0)
        if bayes:
            confidence = raw["conf"]
        else:
            count = raw["count"]
            with np.errstate(divide="ignore", invalid="ignore"):
                ratio = counter.astype(np.float32) / count.astype(np.float32)
            confidence = np.where(count != 0, np.minimum(ratio, np.float32(1)), np.float32(0)).astype(np.float32)
        d = dict(keys=raw["keys"], hashes=_block_hashes(raw["keys"]), count=raw["count"],
                 pos_sum=raw["pos_sum"], col_sum=raw["col_sum"], object_id=raw["object_id"],
                 class_id=raw["class_id"], confidence=confidence, aux=counter,
                 lab_obj=np.full((nb, nv, K), -1, np.int32), lab_cls=np.full((nb, nv, K), -1, np.int32),
                 lab_logp=np.full((nb, nv, K), -np.inf, np.float32))
        if bayes and K > 0 and nb:
            # every pair with its voxel: the in-voxel slots in use, then the overflow pairs, each part in slot order
            L = _lib.B2V_SEM_MAX_LABELS
            slots = np.arange(L)[None, :] < np.minimum(counter.reshape(-1), L)[:, None]
            vox = [np.nonzero(slots)[0]]
            pairs = [[raw[name].reshape(-1, L)[slots]] for name in ("lab_obj", "lab_cls", "lab_logp")]
            over = self._export_labels()
            if over is not None:
                vox.append(np.repeat(np.arange(nb * nv), over["count"].reshape(-1)))
                for p, name in zip(pairs, ("obj", "cls", "logp")):
                    p.append(over[name])
            vox = np.concatenate(vox)
            obj, cls, logp = (np.concatenate(p) for p in pairs)
            order = np.lexsort((cls, obj, vox))   # stable: equal pairs keep slot order
            vox, obj, cls, logp = vox[order], obj[order], cls[order], logp[order]
            rank = np.arange(len(vox)) - np.searchsorted(vox, vox)   # position among the voxel's sorted pairs
            keep = rank < K
            for name, x in (("lab_obj", obj), ("lab_cls", cls), ("lab_logp", logp)):
                d[name].reshape(nb * nv, K)[vox[keep], rank[keep]] = x[keep]
        return d


class VoxelBlockSemanticProbabilisticGrid(VoxelBlockSemanticGrid):
    """GPU drop-in for `volumetric.VoxelBlockSemanticProbabilisticGrid` — Bayesian label fusion in log space
    over joint (object, class) pairs with depth-decayed evidence (voxel_data_semantic.h:249-672)."""

    KIND = _lib.B2V_SEM_PROBABILISTIC


def remap_instance_ids(instance_ids, instance_to_object: dict, invalid_instance_id: int = -1):
    """`volumetric.remap_instance_ids(instance_ids_image, map)` (cpp/volumetric/image_utils.h:69-163): every pixel's
    instance id is replaced by its object id; ids missing from the map - and everything when the map is empty -
    become `invalid_instance_id`."""
    img = np.ascontiguousarray(instance_ids, np.int32)
    if img.size == 0:
        return img
    out = np.full(img.shape, invalid_instance_id, np.int32)
    if instance_to_object:
        keys = np.fromiter(instance_to_object.keys(), np.int64, len(instance_to_object))
        vals = np.fromiter(instance_to_object.values(), np.int64, len(instance_to_object))
        order = np.argsort(keys)
        keys, vals = keys[order], vals[order]
        pos = np.clip(np.searchsorted(keys, img), 0, len(keys) - 1)
        hit = keys[pos] == img
        out[hit] = vals[pos][hit]
    return out


# The direct (non-block) grids of the reference's known-answer tests (cpp/test_volumetric_voxel_semantic.py) hold
# the same voxel records; only the container differs, so the block grids serve as their drop-in as well.
VoxelSemanticGrid = VoxelBlockSemanticGrid
VoxelSemanticGridProbabilistic = VoxelBlockSemanticProbabilisticGrid
