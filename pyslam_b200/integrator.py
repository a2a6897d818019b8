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

from . import map_state
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
    """Set-up every B200 plugin shares; mixed in before pySLAM's `VolumetricIntegratorBase`."""

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

    def _init_gpu_rectify(self):
        """Raw frames go to the device when the base class computed undistortion maps (base.py:766-778) and no depth
        estimator runs (estimated depth needs the host path): the maps are installed on self.volume once."""
        self._gpu_rectify = False
        m1, m2 = getattr(self, "calib_map1", None), getattr(self, "calib_map2", None)
        if (self.b200_parameters["kVolumetricIntegrationB200GpuRectify"] and m1 is not None and m2 is not None
                and getattr(self, "depth_estimator", None) is None):
            self.volume.set_rectification(m1, m2, swap_rb=True)
            self._gpu_rectify = True

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
        if self.b200_parameters["kVolumetricIntegrationB200SaveMapState"]:
            self.volume.save_state(map_state.state_path(ply_path))

    def _load_map_state(self, task, completed, condition):
        """LOAD: replace the map with the state file beside `task.load_save_path`; the next output shows it.  The
        waiter is notified either way; `completed` becomes 1 only on success (a failure raises, leaving the map as it
        was, and the task loop logs it)."""
        loaded = False
        try:
            self.volume.load_state(map_state.state_path(task.load_save_path))
            self._after_load()
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


def make_integrator_class(Base, api):
    """Build the plugin class against a base class and an `api` namespace providing
    `VolumetricIntegrationTaskType`, `VolumetricIntegrationOutput`, `VolumetricIntegrationMesh`,
    `VolumetricIntegrationPointCloud`, `DatasetEnvironmentType` (or None) and `Parameters` (or None); optionally
    `VolumetricIntegrationTask`, the task type `load` enqueues (else a namespace with the task's fields)."""

    TaskType = api.VolumetricIntegrationTaskType

    class VolumetricIntegratorB200(B200PluginSetup, Base):
        """TSDF + colour integration on an H100 (replaces VolumetricIntegratorTsdf + Open3D)."""

        _api = api

        def __init__(self, camera, environment_type, sensor_type, volumetric_integrator_type,
                     viewer_queue=None, **kwargs):
            super().__init__(camera, environment_type, sensor_type, volumetric_integrator_type,
                             viewer_queue, **kwargs)

        # -- runs inside the integrator process: the CUDA context is created here, never in the parent
        def init(self, camera, environment_type, sensor_type, parameters_dict, constructor_kwargs):
            Base.init(self, camera, environment_type, sensor_type, parameters_dict, constructor_kwargs)
            p = self._merge_parameters(DEFAULT_PARAMETERS, parameters_dict, constructor_kwargs)
            outdoor = False
            env_t = getattr(api, "DatasetEnvironmentType", None)
            if env_t is not None and hasattr(env_t, "INDOOR"):
                outdoor = environment_type != env_t.INDOOR
            self.volumetric_integration_depth_trunc = (
                p["kVolumetricIntegrationTsdfDepthTruncOutdoor"] if outdoor
                else p["kVolumetricIntegrationTsdfDepthTruncIndoor"])
            self.volume = B200TsdfVolume(
                voxel_length=p["kVolumetricIntegrationVoxelLength"],
                sdf_trunc=p["kVolumetricIntegrationTSdfTrunc"],
                depth_trunc=self.volumetric_integration_depth_trunc,
                capacity_blocks=int(p["kVolumetricIntegrationB200CapacityBlocks"]),
                max_capacity_blocks=int(p["kVolumetricIntegrationB200MaxCapacityBlocks"]) or None,
                device=int(p["kVolumetricIntegrationB200Device"]),
                volume_unit_resolution=int(p["kVolumetricIntegrationB200UnitResolution"]))
            self.last_output = None
            self.last_integrated_id = -1
            self._deferred_task = None      # a non-INTEGRATE task met while draining a backlog: handled next call
            self._has_deferred = False
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
                mesh_out = api.VolumetricIntegrationMesh(self.volume.extract_triangle_mesh())
            else:
                pc_out = api.VolumetricIntegrationPointCloud(self.volume.extract_point_cloud())
            return api.VolumetricIntegrationOutput(task_type, self.last_integrated_id, pc_out, mesh_out)

        def volume_integration(self, q_in, q_out, q_out_condition, q_management, viewer_queue,
                               is_running, load_request_completed, load_request_condition,
                               save_request_completed, save_request_condition,
                               time_volumetric_integration):
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
                        self.volume.reset()
                    if self._has_deferred:
                        self.last_input_task, self._deferred_task, self._has_deferred = self._deferred_task, None, False
                    else:
                        self.last_input_task = q_in.get()  # blocking
                    if self.last_input_task is None:
                        is_running.value = 0  # a None asks the loop to exit
                    else:
                        ttype = self.last_input_task.task_type
                        if ttype == TaskType.INTEGRATE:
                            # backlog (rebuild(map), base.py:1242-1318): drain the consecutive INTEGRATE tasks that
                            # are already queued into one fused batch; anything else waits for the next call
                            tasks = [self.last_input_task]
                            max_batch = int(self.b200_parameters["kVolumetricIntegrationB200MaxBatch"])
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
                            frames = []
                            for t in tasks:
                                kd = t.keyframe_data
                                color, depth, scale = self._prepare_frame(kd)
                                if color is not None and depth is not None:
                                    frames.append((kd, color, depth, scale))
                            if frames:
                                K4 = tuple(self._intrinsics())
                                same = all(f[1].shape == frames[0][1].shape and f[2].shape == frames[0][2].shape
                                           and f[2].dtype == frames[0][2].dtype and f[3] == frames[0][3]
                                           for f in frames)
                                if len(frames) > 1 and same:
                                    # one C call: groups of frames fused per block visit (b2v_integrate_batch)
                                    self.volume.integrate_batch(np.stack([f[2] for f in frames]),
                                                                np.stack([f[1] for f in frames]), K4,
                                                                np.stack([np.asarray(f[0].pose, np.float64) for f in frames]),
                                                                depth_scale=frames[0][3])
                                else:
                                    for kd, color, depth, scale in frames:
                                        # north_star call: integrate(depth, color, K, pose = Tcw)
                                        self.volume.integrate(depth, color, K4, kd.pose, depth_scale=scale)
                                self.last_integrated_id = frames[-1][0].id
                                self.integrated_frames = getattr(self, "integrated_frames", 0) + len(frames)
                                do_output = True
                                if self.last_output is not None:
                                    dt = time.perf_counter() - self.last_output.timestamp
                                    if dt < self.b200_parameters["kVolumetricIntegrationOutputTimeInterval"]:
                                        do_output = False
                        elif ttype == TaskType.SAVE:
                            path = self.last_input_task.load_save_path
                            if self.b200_parameters["kVolumetricIntegrationTsdfExtractMesh"]:
                                m = self.volume.extract_triangle_mesh()
                                write_ply_mesh(path, m.vertices, m.triangles, m.vertex_colors)
                            else:
                                pc = self.volume.extract_point_cloud()
                                write_ply_points(path, pc.points, pc.colors)
                            self._save_map_state(path)
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
                printer = getattr(Base, "print", print)
                printer(f"VolumetricIntegratorB200: EXCEPTION: {e} !!!")
                printer(traceback.format_exc())
            time_volumetric_integration.value = time.perf_counter() - t_start

        def _stop_volume_integrator_implementation(self):
            if getattr(self, "volume", None) is not None:
                self.volume.close()

    return VolumetricIntegratorB200


def load_pyslam_plugin():
    """Build the plugin against the real pySLAM types (requires pySLAM on sys.path).
    INTEGRATION.md shows the three-line registration in the reference's factory / enum."""
    from pyslam.config_parameters import Parameters
    from pyslam.dense import volumetric_integrator_base as B
    from pyslam.io.dataset_types import DatasetEnvironmentType
    from pyslam.slam import USE_CPP   # C++ core: raw depth reaches the integrator unscaled (base.py:29, 1008-1012)

    api = SimpleNamespace(
        USE_CPP=bool(USE_CPP),
        VolumetricIntegrationTaskType=B.VolumetricIntegrationTaskType,
        VolumetricIntegrationTask=B.VolumetricIntegrationTask,
        VolumetricIntegrationOutput=B.VolumetricIntegrationOutput,
        VolumetricIntegrationMesh=B.VolumetricIntegrationMesh,
        VolumetricIntegrationPointCloud=B.VolumetricIntegrationPointCloud,
        DatasetEnvironmentType=DatasetEnvironmentType, Parameters=Parameters)
    return make_integrator_class(B.VolumetricIntegratorBase, api)
