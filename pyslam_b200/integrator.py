"""`VolumetricIntegratorB200` — the plugin class a pySLAM maintainer registers as a new dense backend.

The reference selects a backend with `volumetric_integrator_factory`
(`pyslam/dense/volumetric_integrator_factory.py:105-150`); every backend subclasses
`VolumetricIntegratorBase` and overrides `init(...)` (runs inside the spawned integrator process,
`volumetric_integrator_base.py:845`) and `volume_integration(...)` (one task per call,
`volumetric_integrator_base.py:1100-1117`; pattern `volumetric_integrator_tsdf.py:121-314`).

This module provides that subclass *without importing pySLAM at module import time* (pySLAM does
not exist on the GPU test box): `make_integrator_class(Base, api)` builds it against whatever base
class / task / output types it is given — pySLAM's real ones (`load_pyslam_plugin()`), or the small
stand-ins in `tests/plugin_standins.py` that mirror their fields so the adapter can be exercised stand-alone.
"""

from __future__ import annotations

import time
import traceback
from types import SimpleNamespace

import numpy as np

from . import keyframe_store, map_state, shard_plugin, sharding
from .volume import B200TsdfVolume

# defaults copied by value from the reference's parameter table (pyslam/config_parameters.py:311,
# 349-351,354,346): voxel length, sdf_trunc, depth truncation indoor / outdoor, output interval,
# whether to extract a mesh (vs a point cloud)
DEFAULT_PARAMETERS = {
    "kVolumetricIntegrationVoxelLength": 0.015,
    "kVolumetricIntegrationTSdfTrunc": 0.04,
    "kVolumetricIntegrationTsdfDepthTruncIndoor": 4.0,
    "kVolumetricIntegrationTsdfDepthTruncOutdoor": 10.0,
    "kVolumetricIntegrationOutputTimeInterval": 1.0,
    "kVolumetricIntegrationTsdfExtractMesh": True,
    "kVolumetricIntegrationB200CapacityBlocks": 1 << 19,
    # growth ceiling of the block pool: > CapacityBlocks starts with CapacityBlocks blocks and maps more on demand,
    # bit-identical to a pool of this size from the start; 0 = fixed pool of CapacityBlocks
    "kVolumetricIntegrationB200MaxCapacityBlocks": 0,
    "kVolumetricIntegrationB200Device": 0,
    # CUDA device ids of a map hash-sharded over several GPUs: with N >= 2 ids this process is rank 0 on the first and
    # starts N - 1 worker processes on the others (shard_plugin.py); empty or one id: one map on one device
    "kVolumetricIntegrationB200Devices": [],
    # undistort + BGR->RGB on the GPU (b2v_set_rectification) instead of the base class's cv2.remap / cvtColor
    "kVolumetricIntegrationB200GpuRectify": True,
    # when the input queue holds a backlog (rebuild(map) re-enqueues every keyframe, base.py:1242-1318), up to this
    # many consecutive INTEGRATE tasks are drained into ONE fused integrate_batch call; 1 = one task per call
    "kVolumetricIntegrationB200MaxBatch": 32,
    # Open3D volume_unit_resolution (tsdf.py:104-108 uses 16); 8 = SURVEY decision D1
    "kVolumetricIntegrationB200UnitResolution": 16,
    # SAVE also writes the map's state beside dense_map.ply (dense_map.state.npz), which LOAD restores; off by default:
    # the file is as large as the map (10 KiB per TSDF block)
    "kVolumetricIntegrationB200SaveMapState": False,
    # keep each voxel's colour as Open3D does, a float64 running mean: voxel, mesh and point-cloud colours equal
    # Open3D's bit for bit, at 16 KiB per block instead of 10 KiB (INTEGRATION.md section 2)
    "kVolumetricIntegrationB200ColorFloat64": False,
    # keep the packed frames of up to this many keyframes on the GPU (8 bytes per pixel: 2.46 MB per 640x480 keyframe),
    # so that rebuild(map) sends only the keyframes' new poses to the integrator (keyframe_store.py); 0 = off.  The
    # grid plugins take the same parameter (integrator_semantic.py)
    "kVolumetricIntegrationB200KeyframeStoreFrames": 0,
}


def write_ply_mesh(path: str, vertices, triangles, vertex_colors=None) -> None:
    """Binary little-endian PLY, the `dense_map.ply` the SAVE task produces
    (`volumetric_integrator_base.py:574-588`; `volumetric_integrator_tsdf.py:233-249`)."""
    V = np.asarray(vertices, np.float32).reshape(-1, 3)
    T = np.asarray(triangles, np.int32).reshape(-1, 3)
    has_c = vertex_colors is not None and len(vertex_colors) == len(V)
    hdr = ["ply", "format binary_little_endian 1.0", f"element vertex {len(V)}",
           "property float x", "property float y", "property float z"]
    if has_c:
        hdr += ["property uchar red", "property uchar green", "property uchar blue"]
    hdr += [f"element face {len(T)}", "property list uchar int vertex_indices", "end_header"]
    with open(path, "wb") as f:
        f.write(("\n".join(hdr) + "\n").encode("ascii"))
        if has_c:
            C8 = np.clip(np.round(np.asarray(vertex_colors) * 255.0), 0, 255).astype(np.uint8)
            rec = np.empty(len(V), dtype=[("p", "<f4", 3), ("c", "u1", 3)])
            rec["p"], rec["c"] = V, C8
            f.write(rec.tobytes())
        else:
            f.write(V.astype("<f4").tobytes())
        if len(T):
            rec = np.empty(len(T), dtype=[("n", "u1"), ("i", "<i4", 3)])
            rec["n"], rec["i"] = 3, T
            f.write(rec.tobytes())


def write_ply_points(path: str, points, colors=None) -> None:
    write_ply_mesh(path, points, np.zeros((0, 3), np.int32), colors)


def raw_depth(depth, camera, use_cpp: bool):
    """(depth, depth_scale) of a raw keyframe depth image for the device, the conversion of base.py:1007-1015.  Raw
    uint16 depth in C++-core mode goes as is with depth_scale = camera.depth_factor: the device widens it to
    float32(depth) * factor, the value `depth.astype(np.float32) * camera.depth_factor` has on the host."""
    if depth.dtype == np.float32:
        return depth, None
    if not use_cpp:
        return depth.astype(np.float32), None
    factor = float(getattr(camera, "depth_factor", 1.0))
    if depth.dtype == np.uint16:
        return depth, np.float32(factor)
    return depth.astype(np.float32) * factor, None


class B200PluginSetup:
    """Set-up every B200 plugin shares; mixed in before pySLAM's `VolumetricIntegratorBase`.  A plugin class sets
    `_api` and `_defaults` (its parameter table)."""

    # the stored-keyframe table publishes each slot's label images (keyframe_store.label_flags)
    _STORE_LABELS = False
    # a non-INTEGRATE task met while draining a backlog: handled by the next volume_integration call
    _deferred_task, _has_deferred = None, False

    def __init__(self, camera, environment_type, sensor_type, volumetric_integrator_type, viewer_queue=None,
                 **kwargs):
        # the table of stored keyframes is created here, in the parent, before the base class spawns the
        # integrator process, which receives it with the rest of the plugin
        n = int(self._parent_parameter("kVolumetricIntegrationB200KeyframeStoreFrames", kwargs))
        self._b200_keyframe_table = (keyframe_store.StoredKeyframeTable(n, labels=self._STORE_LABELS) if n > 0
                                     else None)
        super().__init__(camera, environment_type, sensor_type, volumetric_integrator_type, viewer_queue, **kwargs)

    @classmethod
    def _parent_parameter(cls, name, kwargs):
        """A parameter as the parent process sees it: a constructor keyword, else the `parameters` dict keyword,
        else pySLAM's Parameters class, else the default."""
        if name in kwargs:
            return kwargs[name]
        if name in (kwargs.get("parameters") or {}):
            return kwargs["parameters"][name]
        return getattr(getattr(cls._api, "Parameters", None), name, cls._defaults[name])

    def add_task(self, task):
        """Every task the front end enqueues (keyframes and rebuild(map) alike, base.py:1216-1232): an INTEGRATE
        task of a keyframe the integrator has stored travels without its images (keyframe_store.light_task)."""
        if getattr(self, "_b200_keyframe_table", None) is not None:
            task = keyframe_store.light_task(task, self._b200_keyframe_table,
                                             self._api.VolumetricIntegrationTaskType.INTEGRATE)
        super().add_task(task)

    def _init_frame_store(self):
        """In the integrator process: the map's frame store per kVolumetricIntegrationB200KeyframeStoreFrames."""
        self._store_frames = int(self.b200_parameters["kVolumetricIntegrationB200KeyframeStoreFrames"])
        if self._store_frames > 0:
            self.volume.set_frame_store(self._store_frames)
        self._stored_slots = {}         # keyframe_store.keyframe_key -> slot of the keyframes stored here

    def _record_stored(self, kds, slots):
        """Note the store slots of keyframes just integrated (-1: not stored) and publish them to the parent's
        table."""
        table = getattr(self, "_b200_keyframe_table", None)
        for kd, slot in zip(kds, slots):
            if slot >= 0:
                self._stored_slots[keyframe_store.keyframe_key(kd)] = int(slot)
                if table is not None:
                    table.publish(int(slot), kd)

    def _stored_slot(self, kd):
        """The store slot of a light task's keyframe; None, logged, when its frame is not stored here."""
        slot = self._stored_slots.get(keyframe_store.keyframe_key(kd))
        if slot is None:
            getattr(type(self), "print", print)(
                f"{type(self).__name__}: ERROR: keyframe {kd.id} (timestamp {kd.timestamp}) came without "
                "images, but its frame is not in the frame store: it was not integrated")
        return slot

    def _merge_parameters(self, defaults, parameters_dict, constructor_kwargs):
        """self.b200_parameters: `defaults`, overridden by parameters_dict, then by constructor_kwargs (known keys)."""
        p = dict(defaults)
        if parameters_dict:
            p.update({k: parameters_dict[k] for k in defaults if k in parameters_dict})
        if constructor_kwargs:
            p.update({k: v for k, v in constructor_kwargs.items() if k in defaults})
        self.b200_parameters = p
        # the keys the caller set (the rest hold the plugin's defaults)
        self.b200_set_parameters = {k for k in defaults if k in (parameters_dict or {}) or k in (constructor_kwargs or {})}
        return p

    def _environment_side(self, environment_type):
        """"Indoor" or "Outdoor", the suffix of the parameters that depend on the environment: indoor unless pySLAM's
        DatasetEnvironmentType says otherwise."""
        env_t = getattr(self._api, "DatasetEnvironmentType", None)
        if env_t is not None and hasattr(env_t, "INDOOR") and environment_type != env_t.INDOOR:
            return "Outdoor"
        return "Indoor"

    def _init_gpu_rectify(self):
        """Raw frames go to the device when the base class computed undistortion maps (base.py:766-778) and no depth
        estimator runs (estimated depth needs the host path): the maps are installed on self.volume once."""
        self._gpu_rectify = False
        m1, m2 = getattr(self, "calib_map1", None), getattr(self, "calib_map2", None)
        if (self.b200_parameters["kVolumetricIntegrationB200GpuRectify"] and m1 is not None and m2 is not None
                and getattr(self, "depth_estimator", None) is None):
            self.volume.set_rectification(m1, m2, swap_rb=True)
            self._gpu_rectify = True

    # what a worker's plugin takes over from rank 0's before it builds its shard (shard_plugin.worker_plugin)
    _SHARD_ATTRS = ("b200_parameters", "b200_set_parameters", "volumetric_integration_depth_trunc", "_side",
                    "_probabilistic")

    def _start_map(self):
        """Build the map (`_build_map`): on one device, or with two or more kVolumetricIntegrationB200Devices as rank 0
        of a sharded map whose workers build theirs in the same SETUP op.  Bad device lists raise RuntimeError."""
        p = self.b200_parameters
        devices = shard_plugin.parse_devices(p["kVolumetricIntegrationB200Devices"])
        self._shards = None
        if devices and "kVolumetricIntegrationB200Device" in self.b200_set_parameters:
            getattr(type(self), "print", print)(f"{type(self).__name__}: kVolumetricIntegrationB200Device ignored: "
                                                "kVolumetricIntegrationB200Devices places the map")
        if len(devices) == 1:
            p["kVolumetricIntegrationB200Device"] = devices[0]
        if len(devices) < 2:
            self._build_map()
            return
        c = self.camera
        fx, fy, cx, cy = self._intrinsics()
        attrs = {k: getattr(self, k) for k in self._SHARD_ATTRS if hasattr(self, k)}
        attrs.update(camera=SimpleNamespace(fx=fx, fy=fy, cx=cx, cy=cy, width=getattr(c, "width", None),
                                            height=getattr(c, "height", None)),
                     calib_map1=getattr(self, "calib_map1", None), calib_map2=getattr(self, "calib_map2", None),
                     depth_estimator=None if getattr(self, "depth_estimator", None) is None else True)
        group = shard_plugin.ShardGroup(devices)
        try:
            group.plugin, self._shards = self, group
            group.run("setup", dict(kind=self._SHARD_KIND, factory=shard_plugin.WORKER_FACTORY, attrs=attrs))
        except BaseException:
            self._shards = None
            group.close()
            if getattr(self, "volume", None) is not None:
                self.volume.close()
            raise

    def _op_setup(self, meta):
        self._build_map()

    def _map_placement(self) -> dict:
        """Device and shard arguments of the map's constructor."""
        s = self._shards
        if s is None:
            return dict(device=int(self.b200_parameters["kVolumetricIntegrationB200Device"]))
        return dict(device=s.device, shard_rank=s.rank, shard_count=s.world)

    def _map_call(self, op, meta=None, **arrays):
        """`_op_<op>(meta, **arrays)` on this map, or on every rank's shard of a sharded map (rank 0's result)."""
        if getattr(self, "_shards", None) is None:
            return getattr(self, "_op_" + op)(meta or {}, **arrays)
        return self._shards.run(op, meta, arrays)

    def _agreed(self, result):
        """The int `result` of the last `_map_call` when every rank computed the same (each computes its own, such as
        the frame-store slot it filled), else -1 (ShardGroup.agreed); on one map, `result`."""
        if getattr(self, "_shards", None) is None:
            return result
        return self._shards.agreed()

    def _op_reset(self, meta):
        self.volume.reset()

    def _op_save_state(self, meta):
        self.volume.save_state(map_state.shard_state_path(meta["path"], self._shards.rank, self._shards.world))

    def _op_load_state(self, meta):
        self.volume.load_state(meta["paths"])
        self._after_load()

    def load(self, path):
        """The LOAD task of the map saved in directory `path`, the mirror of the base class's `save(path)`: it reads
        `path/dense_map.state.npz` (written by SAVE with kVolumetricIntegrationB200SaveMapState).  The integrator then
        sets `load_request_completed` to 1 and notifies `load_request_condition`; on failure the flag stays 0."""
        TaskType = self._api.VolumetricIntegrationTaskType
        task_t = getattr(self._api, "VolumetricIntegrationTask", SimpleNamespace)
        self.load_request_completed.value = 0
        self.q_in.put(task_t(keyframe_data=None, task_type=TaskType.LOAD, load_save_path=path + "/dense_map.ply"))

    def _save_map_state(self, ply_path):
        """The part of SAVE that writes the map's state beside the .ply, when kVolumetricIntegrationB200SaveMapState."""
        if not self.b200_parameters["kVolumetricIntegrationB200SaveMapState"]:
            return
        if self._shards is None:
            self.volume.save_state(map_state.state_path(ply_path))
        else:   # every rank writes its own shard file (dense_map.state.<r>-of-<N>.npz)
            map_state.remove_other_states(ply_path, self._shards.world)
            self._shards.run("save_state", dict(path=ply_path))

    def _load_map_state(self, task, completed, condition):
        """LOAD: replace the map with the state beside `task.load_save_path` (`map_state.state_files`: the single file,
        or the shard files of a map saved by several ranks); the next output shows it.  The waiter is notified either
        way; `completed` becomes 1 only on success on every rank (a failure raises, leaving the map as it was, and the
        task loop logs it)."""
        loaded = False
        try:
            self._map_call("load_state", dict(paths=map_state.state_files(task.load_save_path)))
            loaded = True
        finally:
            with condition:
                if loaded:
                    completed.value = 1
                condition.notify_all()

    def _after_load(self):
        pass

    def _intrinsics(self):
        if hasattr(self, "get_camera_intrinsics_for_depth"):
            return self.get_camera_intrinsics_for_depth()
        c = self.camera
        return c.fx, c.fy, c.cx, c.cy

    def volume_integration(self, q_in, q_out, q_out_condition, q_management, viewer_queue,
                           is_running, load_request_completed, load_request_condition,
                           save_request_completed, save_request_condition,
                           time_volumetric_integration):
        """One task of the integrator process (base.py:905-915): RESET from the management queue first, then the next
        task.  The plugin class provides `_integrate_tasks` (INTEGRATE), `_write_ply` (SAVE) and `_make_output`."""
        api = self._api
        TaskType = api.VolumetricIntegrationTaskType
        t_start = time.perf_counter()
        last_output = None
        do_output = False
        try:
            if is_running.value == 1:
                # management queue first: RESET
                task = None
                try:
                    task = q_management.get_nowait()
                except Exception:
                    pass
                if task is not None and task.task_type == TaskType.RESET:
                    self._map_call("reset")
                if self._has_deferred:
                    self.last_input_task, self._deferred_task, self._has_deferred = self._deferred_task, None, False
                else:
                    self.last_input_task = q_in.get()  # blocking
                if self.last_input_task is None:
                    is_running.value = 0  # a None asks the loop to exit
                else:
                    ttype = self.last_input_task.task_type
                    if ttype == TaskType.INTEGRATE:
                        # backlog (rebuild(map), base.py:1242-1318): drain the consecutive INTEGRATE tasks that are
                        # already queued, up to kVolumetricIntegrationB200MaxBatch (the grid plugins have no such
                        # parameter and take one per call); anything else waits for the next call
                        tasks = [self.last_input_task]
                        max_batch = int(self.b200_parameters.get("kVolumetricIntegrationB200MaxBatch", 1))
                        while len(tasks) < max_batch:
                            try:
                                nxt = q_in.get_nowait()
                            except Exception:
                                break
                            if nxt is None or nxt.task_type != TaskType.INTEGRATE:
                                self._deferred_task, self._has_deferred = nxt, True
                                break
                            tasks.append(nxt)
                        self.last_input_task = tasks[-1]
                        done = self._integrate_tasks(tasks)
                        if done:
                            self.last_integrated_id = done[-1].id
                            self.integrated_frames = getattr(self, "integrated_frames", 0) + len(done)
                            do_output = True
                            if self.last_output is not None:
                                dt = time.perf_counter() - self.last_output.timestamp
                                if dt < self.b200_parameters["kVolumetricIntegrationOutputTimeInterval"]:
                                    do_output = False
                    elif ttype == TaskType.SAVE:
                        self._write_ply(self.last_input_task.load_save_path)
                        self._save_map_state(self.last_input_task.load_save_path)
                        last_output = api.VolumetricIntegrationOutput(ttype)
                    elif ttype == TaskType.LOAD:
                        self._load_map_state(self.last_input_task, load_request_completed, load_request_condition)
                    elif ttype == TaskType.UPDATE_OUTPUT:
                        do_output = True
                    if do_output:
                        last_output = self._make_output(ttype)
                        self.last_output = last_output
                    if is_running.value == 1 and last_output is not None:
                        if last_output.task_type in (TaskType.INTEGRATE, TaskType.UPDATE_OUTPUT):
                            with q_out_condition:
                                last_output.timestamp = time.perf_counter()
                                q_out.put(last_output)
                                q_out_condition.notify_all()
                        elif last_output.task_type == TaskType.SAVE:
                            with save_request_condition:
                                save_request_completed.value = 1
                                save_request_condition.notify_all()
        except Exception as e:  # the reference logs and keeps the loop alive (tsdf.py:303-307)
            printer = getattr(type(self), "print", print)
            printer(f"{type(self).__name__}: EXCEPTION: {e} !!!")
            printer(traceback.format_exc())
        time_volumetric_integration.value = time.perf_counter() - t_start

    def _stop_volume_integrator_implementation(self):
        if getattr(self, "_shards", None) is not None:
            self._shards.close()
        if getattr(self, "volume", None) is not None:
            self.volume.close()


def make_integrator_class(Base, api):
    """Build the plugin class against a base class and an `api` namespace providing
    `VolumetricIntegrationTaskType`, `VolumetricIntegrationOutput`, `VolumetricIntegrationMesh`,
    `VolumetricIntegrationPointCloud`, `DatasetEnvironmentType` (or None) and `Parameters` (or None); optionally
    `VolumetricIntegrationTask`, the task type `load` enqueues (else a namespace with the task's fields)."""

    class VolumetricIntegratorB200(B200PluginSetup, Base):
        """TSDF + colour integration on an H100 (replaces VolumetricIntegratorTsdf + Open3D)."""

        _api = api
        _defaults = DEFAULT_PARAMETERS
        _SHARD_KIND = "tsdf"

        # -- runs inside the integrator process: the CUDA context is created here, never in the parent
        def init(self, camera, environment_type, sensor_type, parameters_dict, constructor_kwargs):
            Base.init(self, camera, environment_type, sensor_type, parameters_dict, constructor_kwargs)
            p = self._merge_parameters(DEFAULT_PARAMETERS, parameters_dict, constructor_kwargs)
            self.volumetric_integration_depth_trunc = p[
                f"kVolumetricIntegrationTsdfDepthTrunc{self._environment_side(environment_type)}"]
            self._start_map()

        def _build_map(self):
            p = self.b200_parameters
            self.volume = B200TsdfVolume(
                voxel_length=p["kVolumetricIntegrationVoxelLength"],
                sdf_trunc=p["kVolumetricIntegrationTSdfTrunc"],
                depth_trunc=self.volumetric_integration_depth_trunc,
                capacity_blocks=int(p["kVolumetricIntegrationB200CapacityBlocks"]),
                max_capacity_blocks=int(p["kVolumetricIntegrationB200MaxCapacityBlocks"]) or None,
                volume_unit_resolution=int(p["kVolumetricIntegrationB200UnitResolution"]),
                color_float64=bool(p["kVolumetricIntegrationB200ColorFloat64"]), **self._map_placement())
            self._init_frame_store()
            self.last_output = None
            self.last_integrated_id = -1
            self._init_gpu_rectify()

        def _prepare_frame(self, kd):
            """(color RGB or raw BGR when the GPU rectifies, depth, depth_scale).  With GPU rectification and no
            depth estimator the raw images go straight to the device: remap + channel swap happen there,
            bit-identically to cv2.remap / cvtColor (base.py:1017-1054), and the depth is converted by `raw_depth`."""
            if self._gpu_rectify and kd.depth is not None and kd.depth.size and kd.img is not None:
                return (kd.img, *raw_depth(kd.depth, self.camera, getattr(api, "USE_CPP", False)))
            if self._gpu_rectify:
                return None, None, None
            rect = self.estimate_depth_if_needed_and_rectify(kd)
            return rect[0], rect[1], None

        def _make_output(self, task_type):
            p = self.b200_parameters
            mesh_out, pc_out = None, None
            if p["kVolumetricIntegrationTsdfExtractMesh"]:
                mesh_out = api.VolumetricIntegrationMesh(self._map_call("mesh"))
            else:
                pc_out = api.VolumetricIntegrationPointCloud(self._map_call("points"))
            return api.VolumetricIntegrationOutput(task_type, self.last_integrated_id, pc_out, mesh_out)

        def _op_mesh(self, meta):
            if self._shards is None:
                return self.volume.extract_triangle_mesh()
            return sharding.extract_mesh_sharded(self.volume)

        def _op_points(self, meta):
            if self._shards is None:
                return self.volume.extract_point_cloud()
            return sharding.extract_point_cloud_sharded(self.volume)

        def _op_integrate(self, meta, depths, colors):
            """The last store slot the call filled (-1: none, or the store is off): rank 0 records the call's slots only
            when every rank filled the same.  Slots are filled in call order, so a rank's store holds that slot + 1
            frames, and a rank whose store stopped early (each rank maps its own) never agrees again."""
            self.volume.integrate_batch(depths, colors, meta["K"], meta["poses"], depth_scale=meta["scale"])
            return int(self.volume.last_stored_slots().max()) if getattr(self, "_store_frames", 0) else -1

        def _op_integrate_stored(self, meta):
            self.volume.integrate_stored(meta["slots"], meta["K"], meta["poses"])

        def _integrate_tasks(self, tasks):
            """Light tasks (keyframe_store) and image-carrying ones may alternate in a drained backlog: their runs in
            order; the keyframes integrated, in order."""
            done = []
            for stored, run in keyframe_store.split_runs(tasks):
                done += self._integrate_stored(run) if stored else self._integrate_images(run)
            return done

        def _integrate_images(self, tasks):
            """Tasks that carry their images: one fused integrate_batch when there are several frames of one shape,
            dtype and depth scale, else one integrate_batch per frame.  On a sharded map rank 0 uploads each batch
            once (raw uint16 depth stays 16-bit) and broadcasts it.  Every rank stores the same frames in the same
            slots while every rank's store has room; rank 0's are recorded only when every rank's store holds as many
            frames as rank 0's (a rank whose store stopped early never catches up, so its slots can no longer be
            replayed).  The keyframes integrated, in order."""
            frames = []
            for t in tasks:
                kd = t.keyframe_data
                color, depth, scale = self._prepare_frame(kd)
                if color is not None and depth is not None:
                    frames.append((kd, color, depth, scale))
            if not frames:
                return []
            K4 = tuple(self._intrinsics())
            same = all(f[1].shape == frames[0][1].shape and f[2].shape == frames[0][2].shape
                       and f[2].dtype == frames[0][2].dtype and f[3] == frames[0][3]
                       for f in frames)
            store = getattr(self, "_store_frames", 0) > 0
            # one C call per part: groups of frames fused per block visit (b2v_integrate_batch); a lone frame is a
            # one-frame batch of views, not a copy
            for part in ([frames] if len(frames) > 1 and same else [[f] for f in frames]):
                scale = part[0][3]
                depths = np.stack([f[2] for f in part]) if len(part) > 1 else part[0][2][None]
                colors = np.stack([f[1] for f in part]) if len(part) > 1 else part[0][1][None]
                n = self._map_call(
                    "integrate", dict(K=K4, poses=np.stack([np.asarray(f[0].pose, np.float64) for f in part]),
                                      scale=scale),
                    depths=np.ascontiguousarray(depths, np.float32 if scale is None else np.uint16),
                    colors=np.ascontiguousarray(colors, np.uint8))
                if store and self._agreed(n) >= 0:
                    self._record_stored([f[0] for f in part], self.volume.last_stored_slots())
            return [f[0] for f in frames]

        def _integrate_stored(self, tasks):
            """Light tasks (keyframe_store): the stored frames with the tasks' poses, in one call; the keyframes
            integrated, in order.  A keyframe whose frame is not stored here is logged and left out."""
            kds, slots = [], []
            for t in tasks:
                kd = t.keyframe_data
                slot = self._stored_slot(kd)
                if slot is None:
                    continue
                kds.append(kd)
                slots.append(slot)
            if not kds:
                return []
            K4 = tuple(self._intrinsics())
            slots = np.asarray(slots, np.int32)
            poses = np.stack([np.asarray(kd.pose, np.float64) for kd in kds])
            self._map_call("integrate_stored", dict(K=K4, poses=poses, slots=slots))
            return kds

        def _write_ply(self, path):
            """SAVE's dense_map.ply: the mesh, or the point cloud (kVolumetricIntegrationTsdfExtractMesh)."""
            if self.b200_parameters["kVolumetricIntegrationTsdfExtractMesh"]:
                m = self._map_call("mesh")
                write_ply_mesh(path, m.vertices, m.triangles, m.vertex_colors)
            else:
                pc = self._map_call("points")
                write_ply_points(path, pc.points, pc.colors)

    return VolumetricIntegratorB200


def pyslam_api():
    """pySLAM's dense-integration module and the `api` namespace of its types that the plugin classes are built
    against (requires pySLAM on sys.path)."""
    from pyslam.config_parameters import Parameters
    from pyslam.dense import volumetric_integrator_base as B
    from pyslam.io.dataset_types import DatasetEnvironmentType
    from pyslam.slam import USE_CPP   # C++ core: raw depth reaches the integrator unscaled (base.py:29, 1008-1012)

    return B, SimpleNamespace(
        USE_CPP=bool(USE_CPP),
        VolumetricIntegrationTaskType=B.VolumetricIntegrationTaskType,
        VolumetricIntegrationTask=B.VolumetricIntegrationTask,
        VolumetricIntegrationOutput=B.VolumetricIntegrationOutput,
        VolumetricIntegrationMesh=B.VolumetricIntegrationMesh,
        VolumetricIntegrationPointCloud=B.VolumetricIntegrationPointCloud,
        DatasetEnvironmentType=DatasetEnvironmentType, Parameters=Parameters)


def load_pyslam_plugin():
    """Build the plugin against the real pySLAM types (requires pySLAM on sys.path).
    INTEGRATION.md shows the three-line registration in the reference's factory / enum."""
    B, api = pyslam_api()
    return make_integrator_class(B.VolumetricIntegratorBase, api)
