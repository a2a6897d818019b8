"""`VolumetricIntegratorB200SemanticGrid` — the plugin class for pySLAM's semantic dense backend
(`VolumetricIntegratorVoxelSemanticGrid`, pyslam/dense/volumetric_integrator_voxel_semantic_grid.py) on the GPU.

Same contract as `integrator.py`: a subclass of `VolumetricIntegratorBase` built against whichever base / task /
output types it is given (pySLAM's real ones, or the in-process stand-ins of `tests/plugin_standins.py`).  The per-frame
loop body (reference :326-461) maps one-to-one onto the C ABI:

    filter_shadow_points + depth2pointcloud + world transform + integrate  ->  b2v_sgrid_integrate_rgbd
    assign_object_ids_to_instance_ids (+ carving)                           ->  b2v_sgrid_assign_object_ids_to_instance_ids
    remap_instance_ids                                                      ->  pyslam_b200.remap_instance_ids
    carve (no instance ids)                                                 ->  b2v_sgrid_carve
    get_voxels(min_count, min_confidence)                                   ->  b2v_sgrid_get_voxels / copy_voxels

    get_object_segments(min_count, min_confidence)                          ->  b2v_sgrid_get_voxels + grouping / PCA boxes

With undistortion maps and no depth estimator (kVolumetricIntegrationB200GpuRectify), the base class's host preparation
(cv2.remap, cvtColor, depth widening) and the host instance remap give way to b2v_sgrid_set_frame (raw images, each
uploaded once, shadow filter once) and b2v_sgrid_remap_instance_ids; the calls above read the staged images.

Outputs: when 2-D instance ids are integrated, the reference's OBJECTS representation (:523-587:
`get_object_segments` -> `VolumetricIntegrationObjectList`, one entry per object with its points, colours, class id,
confidence range and oriented box); otherwise its single-point-cloud representation (:590-700): points, colours,
class ids, object ids.
"""

from __future__ import annotations

import time
import traceback

from types import SimpleNamespace

import numpy as np

from . import sharding
from .integrator import B200PluginSetup, raw_depth, write_ply_points
from .volume import (CameraFrustrum, VoxelBlockGrid, VoxelBlockSemanticGrid, VoxelBlockSemanticProbabilisticGrid,
                     filter_shadow_points, remap_instance_ids)

# defaults of pyslam/config_parameters.py:311-380 (overridable through parameters_dict / constructor kwargs)
DEFAULT_PARAMETERS = {
    "kVolumetricIntegrationVoxelLength": 0.015,
    "kVolumetricIntegrationBlockSize": 8,
    "kVolumetricIntegrationTsdfDepthTruncIndoor": 4.0,
    "kVolumetricIntegrationTsdfDepthTruncOutdoor": 10.0,
    "kVolumetricIntegrationOutputTimeInterval": 1.0,
    "kVolumetricIntegrationVoxelGridMinCount": 3,
    "kVolumetricIntegrationVoxelGridMinConfidence": 0.6,
    "kVolumetricIntegrationVoxelGridUseCarving": False,
    "kVolumetricIntegrationVoxelGridCarvingDepthMin": 1e-2,
    "kVolumetricIntegrationVoxelGridCarvingDepthMaxIndoor": 8.0,
    "kVolumetricIntegrationVoxelGridCarvingDepthMaxOutdoor": 15.0,
    "kVolumetricIntegrationVoxelGridCarvingDepthThreshold": 3e-2,
    "kVolumetricIntegrationVoxelGridShadowPointsFilter": True,
    "kVolumetricSemanticProbabilisticIntegrationUseDepth": True,
    "kVolumetricSemanticProbabilisticIntegrationDepthThresholdIndoor": 5.0,
    "kVolumetricSemanticProbabilisticIntegrationDepthThresholdOutdoor": 10.0,
    "kVolumetricSemanticProbabilisticIntegrationDepthDecayRateIndoor": 0.1,
    "kVolumetricSemanticProbabilisticIntegrationDepthDecayRateOutdoor": 0.05,
    "kVolumetricSemanticIntegrationUseInstanceIds": True,
    "kVolumetricSemanticIntegrationMinVoteRatio": 0.5,
    "kVolumetricSemanticIntegrationMinVotes": 3,
    "kVolumetricIntegrationB200CapacityBlocks": 1 << 15,
    # growth ceiling of the grid's storage: > CapacityBlocks starts with CapacityBlocks blocks and maps more on
    # demand, holding what a grid of this size from the start holds; 0 = fixed storage of CapacityBlocks
    "kVolumetricIntegrationB200MaxCapacityBlocks": 0,
    # Bayesian grid (use_semantic_probabilistic): ceiling of the overflow label store, in (object, class) pairs past
    # the 8 a voxel holds itself; below it no voxel evicts a pair and the labels equal the reference's unbounded map.
    # 0 = no store (a ninth pair evicts the weakest); the voting grid has no label set and ignores it
    "kVolumetricIntegrationB200LabelOverflowPairs": 0,
    # voxel-grid plugin: each voxel sums its points in input order (VoxelBlockGrid(input_order_sums=True)), so the
    # map equals the reference's sequential build bit for bit and is the same on every run; the semantic grids always
    # sum in input order and do not read it
    "kVolumetricIntegrationB200InputOrderSums": False,
    "kVolumetricIntegrationB200Device": 0,
    # device ids of a map sharded over several GPUs (integrator.py has the same parameter)
    "kVolumetricIntegrationB200Devices": [],
    "kVolumetricIntegrationB200GenerateObjects": True,   # kGenerateObjectsDefault (reference :84)
    # raw keyframe images to the grid (set_frame): upload once, undistort + BGR->RGB + depth widening + shadow filter
    # on the GPU instead of the base class's cv2.remap / cvtColor (integrator.py has the same switch)
    "kVolumetricIntegrationB200GpuRectify": True,
    # SAVE also writes the grid's state beside dense_map.ply (dense_map.state.npz), which LOAD restores; off by
    # default: the file is as large as the map (78 KiB per Bayesian block)
    "kVolumetricIntegrationB200SaveMapState": False,
}


def _grid_args(p, set_keys=()):
    """Constructor arguments of either grid from the plugin parameters.  The capacities count blocks of the configured
    kVolumetricIntegrationBlockSize B.  A capacity the caller did not set (not in `set_keys`) is the default's voxel
    budget at that size: default * 512 / B^3 blocks, rounded up, so the default memory does not change with B; a value
    the caller set is taken as given."""
    B = int(p["kVolumetricIntegrationBlockSize"])

    def blocks(key):
        n = int(p[key])
        return n if key in set_keys or B <= 0 else -(-n * 512 // B ** 3)

    return dict(voxel_size=p["kVolumetricIntegrationVoxelLength"], block_size=B,
                capacity_blocks=blocks("kVolumetricIntegrationB200CapacityBlocks"),
                device=int(p["kVolumetricIntegrationB200Device"]),
                max_capacity_blocks=blocks("kVolumetricIntegrationB200MaxCapacityBlocks") or None)


def make_semantic_integrator_class(Base, api):
    """Build the semantic plugin class against a base class and an `api` namespace (see `integrator.py`)."""
    TaskType = api.VolumetricIntegrationTaskType

    class VolumetricIntegratorB200SemanticGrid(B200PluginSetup, Base):
        """GPU semantic voxel-grid integrator; `use_semantic_probabilistic` selects Bayesian fusion (:131-141)."""

        _defaults = DEFAULT_PARAMETERS
        _api = api
        _SHARD_KIND = "semantic"
        _LABELS = True     # the grid takes class and instance images

        def __init__(self, camera, environment_type, sensor_type, volumetric_integrator_type,
                     viewer_queue=None, **kwargs):
            super().__init__(camera, environment_type, sensor_type, volumetric_integrator_type,
                             viewer_queue, **kwargs)

        # -- runs inside the integrator process: the CUDA context is created here, never in the parent
        def init(self, camera, environment_type, sensor_type, parameters_dict, constructor_kwargs):
            Base.init(self, camera, environment_type, sensor_type, parameters_dict, constructor_kwargs)
            p = self._merge_parameters(self._defaults, parameters_dict, constructor_kwargs)
            indoor = True
            env_t = getattr(api, "DatasetEnvironmentType", None)
            if env_t is not None and hasattr(env_t, "INDOOR"):
                indoor = environment_type == env_t.INDOOR
            self._side = "Indoor" if indoor else "Outdoor"
            self._probabilistic = bool((constructor_kwargs or {}).get("use_semantic_probabilistic", False))
            self.volumetric_integration_depth_trunc = p[f"kVolumetricIntegrationTsdfDepthTrunc{self._side}"]
            self._start_map()

        def _build_map(self):
            p, side = self.b200_parameters, self._side
            self.volume = self._make_grid(p, side, {"use_semantic_probabilistic": self._probabilistic})
            fx, fy, cx, cy = self._intrinsics()
            self.camera_frustrum = CameraFrustrum(
                fx, fy, cx, cy, self.camera.width, self.camera.height, np.eye(4),
                depth_max=p[f"kVolumetricIntegrationVoxelGridCarvingDepthMax{side}"],
                depth_min=p["kVolumetricIntegrationVoxelGridCarvingDepthMin"])
            self.last_output = None
            self.last_integrated_id = -1
            self.last_instance_map = {}
            self._init_gpu_rectify()

        def _after_load(self):
            """The restored grid has no association yet, and until the next keyframe the output represents it as
            objects when the configuration integrates instance ids."""
            self.last_instance_map = {}
            self.integrated_instance_ids = bool(self.b200_parameters["kVolumetricSemanticIntegrationUseInstanceIds"])

        def _make_grid(self, p, side, constructor_kwargs):
            probabilistic = bool(constructor_kwargs.get("use_semantic_probabilistic", False))
            grid_t = VoxelBlockSemanticProbabilisticGrid if probabilistic else VoxelBlockSemanticGrid
            pairs = int(p["kVolumetricIntegrationB200LabelOverflowPairs"])
            if pairs and not probabilistic:
                getattr(Base, "print", print)("VolumetricIntegratorB200SemanticGrid: "
                                              "kVolumetricIntegrationB200LabelOverflowPairs ignored: it applies to "
                                              "use_semantic_probabilistic only")
                pairs = 0
            grid = grid_t(**dict(_grid_args(p, self.b200_set_parameters), **self._map_placement()),
                          max_label_overflow_pairs=pairs)
            grid.set_depth_threshold(p[f"kVolumetricSemanticProbabilisticIntegrationDepthThreshold{side}"])
            grid.set_depth_decay_rate(p[f"kVolumetricSemanticProbabilisticIntegrationDepthDecayRate{side}"])
            return grid

        def _raw_frame(self, kd):
            """(depth, depth_scale) of a keyframe for `set_frame` (see `raw_depth`), or None when it takes the host
            path."""
            if not self._gpu_rectify or kd.depth is None or not kd.depth.size or kd.img is None:
                return None
            if kd.depth.shape != (self.camera_frustrum.height, self.camera_frustrum.width):
                return None   # the frustum's label / carve calls reject such frames: the host path handles them
            return raw_depth(kd.depth, self.camera, getattr(api, "USE_CPP", False))

        def _uses_instances(self, classes, instances):
            """The frame's instance ids are associated and integrated (host arrays)."""
            return (self._LABELS and bool(self.b200_parameters["kVolumetricSemanticIntegrationUseInstanceIds"])
                    and instances is not None and np.asarray(instances).size > 0 and classes is not None)

        def _assign_object_ids(self, *args, **kwargs):
            """The grid's association; over all ranks for a sharded grid."""
            if self._shards is None:
                return self.volume.assign_object_ids_to_instance_ids(*args, **kwargs)
            return sharding.assign_object_ids_to_instance_ids_sharded(self.volume, *args, **kwargs)

        def _integrate_raw(self, kd, depth, scale, use_instances):
            """The loop body on the raw images: one set_frame uploads, rectifies and shadow-filters them on the
            device; association (or carving), the instance remap and the integration read the staged images."""
            p = self.b200_parameters
            flt = bool(p["kVolumetricIntegrationVoxelGridShadowPointsFilter"])
            classes, instances = kd.semantic_img, kd.semantic_instances_img
            fr = self.volume.set_frame(depth, kd.img, class_image=classes,
                                       instance_image=instances if use_instances else None, depth_scale=scale,
                                       filter_shadow_points=flt)
            self.integrated_instance_ids = False
            self.camera_frustrum.set_T_cw(kd.pose)
            carve_thr = float(p["kVolumetricIntegrationVoxelGridCarvingDepthThreshold"])
            object_image = None
            if use_instances:   # association and carving see the filtered depth (:349-362, :371-388)
                self.last_instance_map = self._assign_object_ids(
                    self.camera_frustrum, fr.class_image, fr.instance_image, fr.filtered_depth,
                    depth_threshold=carve_thr, do_carving=bool(p["kVolumetricIntegrationVoxelGridUseCarving"]),
                    min_vote_ratio=float(p["kVolumetricSemanticIntegrationMinVoteRatio"]),
                    min_votes=int(p["kVolumetricSemanticIntegrationMinVotes"]))
                object_image = self.volume.remap_instance_ids()
                self.integrated_instance_ids = True
            elif p["kVolumetricIntegrationVoxelGridUseCarving"]:
                self.volume.carve(self.camera_frustrum, fr.filtered_depth, carve_thr)
            fx, fy, cx, cy = self._intrinsics()
            Twc = np.linalg.inv(np.asarray(kd.pose, np.float64).reshape(4, 4))
            self.volume.integrate_rgbd(
                fr.filtered_depth, fr.color, (fx, fy, cx, cy), Twc, class_image=fr.class_image,
                object_image=object_image, max_depth=self.volumetric_integration_depth_trunc,
                use_depths=bool(p["kVolumetricSemanticProbabilisticIntegrationUseDepth"]), filter_shadow_points=False)
            self.last_integrated_id = kd.id
            return True

        def _integrate_keyframe(self, kd):
            """The reference loop body for one keyframe (:300-461): on the raw images, or on the ones the base class
            prepared on the host; on every rank's shard of a sharded grid."""
            raw = self._raw_frame(kd)
            if self._shards is not None:
                return self._integrate_keyframe_sharded(kd, raw)
            if raw is not None:
                return self._integrate_raw(kd, *raw, self._uses_instances(kd.semantic_img, kd.semantic_instances_img))
            rect = self.estimate_depth_if_needed_and_rectify(kd)
            color, depth = rect[0], rect[1]
            classes = rect[3] if len(rect) > 3 else None
            instances = rect[4] if len(rect) > 4 else None
            if color is None or depth is None:
                return False
            return self._integrate_prepared(kd, color, depth, classes, instances)

        def _labels(self, classes, instances, use_instances, raw):
            """The label images of a broadcast keyframe: none for the point-average grid; int32 (what set_frame
            converts them to) on the raw path, where an empty image is no image."""
            if not self._LABELS:
                return {}
            out = {}
            for name, img in (("classes", classes), ("instances", instances if use_instances or not raw else None)):
                if img is not None and raw:
                    img = np.ascontiguousarray(img, np.int32) if np.asarray(img).size else None
                out[name] = img
            return out

        def _integrate_keyframe_sharded(self, kd, raw):
            """Rank 0's part of INTEGRATE: broadcast the keyframe (raw images, or the host-prepared ones when the
            frame takes the host path); every rank then runs the loop body on its shard (`_op_frame`)."""
            meta = dict(id=kd.id, pose=np.asarray(kd.pose, np.float64), raw=raw is not None)
            if raw is not None:
                depth, scale = raw
                use = self._uses_instances(kd.semantic_img, kd.semantic_instances_img)
                meta.update(scale=scale, use_instances=use)
                arrays = dict(depth=depth, img=kd.img,
                              **self._labels(kd.semantic_img, kd.semantic_instances_img, use, True))
            else:
                rect = self.estimate_depth_if_needed_and_rectify(kd)
                color, depth = rect[0], rect[1]
                if color is None or depth is None:
                    return False
                arrays = dict(depth=depth, img=color, **self._labels(rect[3] if len(rect) > 3 else None,
                                                                     rect[4] if len(rect) > 4 else None, False, False))
            self._shards.run("frame", meta, arrays)
            return True

        def _op_frame(self, meta, depth, img, classes=None, instances=None):
            kd = SimpleNamespace(id=meta["id"], pose=meta["pose"], img=img, semantic_img=classes,
                                 semantic_instances_img=instances)
            if meta["raw"]:
                return self._integrate_raw(kd, depth, meta["scale"], meta["use_instances"])
            host = [x.cpu().numpy() if hasattr(x, "cpu") else x for x in (img, depth, classes, instances)]
            return self._integrate_prepared(kd, *host)

        def _integrate_prepared(self, kd, color, depth, classes, instances):
            """The loop body on images the base class prepared on the host."""
            p = self.b200_parameters
            depth = np.ascontiguousarray(depth, np.float32)
            flt = bool(p["kVolumetricIntegrationVoxelGridShadowPointsFilter"])
            self.integrated_instance_ids = False
            use_instances = self._uses_instances(classes, instances)
            self.camera_frustrum.set_T_cw(kd.pose)
            carve_thr = float(p["kVolumetricIntegrationVoxelGridCarvingDepthThreshold"])
            object_image = None
            if use_instances or p["kVolumetricIntegrationVoxelGridUseCarving"]:
                # association and carving look at the FILTERED depth image (:349-362, :371-388)
                depth_used = filter_shadow_points(depth) if flt else depth
                if use_instances:
                    self.last_instance_map = self._assign_object_ids(
                        self.camera_frustrum, classes, instances, depth_used, depth_threshold=carve_thr,
                        do_carving=bool(p["kVolumetricIntegrationVoxelGridUseCarving"]),
                        min_vote_ratio=float(p["kVolumetricSemanticIntegrationMinVoteRatio"]),
                        min_votes=int(p["kVolumetricSemanticIntegrationMinVotes"]))
                    object_image = remap_instance_ids(instances, self.last_instance_map)
                    self.integrated_instance_ids = True
                else:
                    self.volume.carve(self.camera_frustrum, depth_used, carve_thr)
            fx, fy, cx, cy = self._intrinsics()
            Twc = np.linalg.inv(np.asarray(kd.pose, np.float64).reshape(4, 4))
            self.volume.integrate_rgbd(
                depth, color, (fx, fy, cx, cy), Twc, class_image=classes, object_image=object_image,
                max_depth=self.volumetric_integration_depth_trunc,
                use_depths=bool(p["kVolumetricSemanticProbabilisticIntegrationUseDepth"]), filter_shadow_points=flt)
            self.last_integrated_id = kd.id
            return True

        def _make_output(self, task_type):
            p = self.b200_parameters
            ObjList = getattr(api, "VolumetricIntegrationObjectList", None)
            if (p["kVolumetricIntegrationB200GenerateObjects"] and getattr(self, "integrated_instance_ids", False)
                    and ObjList is not None):
                # reference :523-587: objects only when instance ids are available
                grp = self._map_call("segments", dict(
                    min_count=int(p["kVolumetricIntegrationVoxelGridMinCount"]),
                    min_confidence=float(p["kVolumetricIntegrationVoxelGridMinConfidence"])))
                sem_rgb = getattr(api, "sem_img_to_rgb", None)      # SemanticMappingShared.sem_img_to_rgb
                ids_rgb = getattr(api, "ids_to_rgb_float", None)    # IdsColorTable.ids_to_rgb_float
                n = len(grp.object_vector)
                sem_cols = (np.ascontiguousarray(sem_rgb(np.asarray(grp.class_ids), bgr=True), np.float32) / 255.0
                            if sem_rgb is not None and n else np.zeros((n, 3), np.float32))
                obj_cols = (np.ascontiguousarray(ids_rgb(np.asarray(grp.object_ids), bgr=True), np.float32)
                            if ids_rgb is not None and n else np.zeros((n, 3), np.float32))
                objects = ObjList(grp, sem_cols, obj_cols, n)
                return api.VolumetricIntegrationOutput(task_type, self.last_integrated_id, None, None, objects)
            v = self._map_call("voxels", dict(min_count=int(p["kVolumetricIntegrationVoxelGridMinCount"]),
                                              min_confidence=float(p["kVolumetricIntegrationVoxelGridMinConfidence"])))
            pc = api.VolumetricIntegrationPointCloud(points=np.ascontiguousarray(v.points, np.float32),
                                                     colors=np.ascontiguousarray(v.colors, np.float32))
            pc.semantics = v.class_ids if len(v.class_ids) else None
            pc.object_ids = v.object_ids if len(v.object_ids) else None
            return api.VolumetricIntegrationOutput(task_type, self.last_integrated_id, pc, None)

        def _op_voxels(self, meta):
            if self._shards is None:
                return self.volume.get_voxels(**meta)
            return sharding.get_voxels_sharded(self.volume, **meta)

        def _op_segments(self, meta):
            if self._shards is None:
                return self.volume.get_object_segments(**meta)
            return sharding.get_object_segments_sharded(self.volume, **meta)

        def volume_integration(self, q_in, q_out, q_out_condition, q_management, viewer_queue,
                               is_running, load_request_completed, load_request_condition,
                               save_request_completed, save_request_condition,
                               time_volumetric_integration):
            t_start = time.perf_counter()
            last_output = None
            do_output = False
            try:
                if is_running.value == 1:
                    task = None
                    try:
                        task = q_management.get_nowait()
                    except Exception:
                        pass
                    if task is not None and task.task_type == TaskType.RESET:
                        self._map_call("reset")
                    self.last_input_task = q_in.get()  # blocking
                    if self.last_input_task is None:
                        is_running.value = 0
                    else:
                        ttype = self.last_input_task.task_type
                        if ttype == TaskType.INTEGRATE:
                            if self._integrate_keyframe(self.last_input_task.keyframe_data):
                                do_output = True
                                if self.last_output is not None:
                                    dt = time.perf_counter() - self.last_output.timestamp
                                    if dt < self.b200_parameters["kVolumetricIntegrationOutputTimeInterval"]:
                                        do_output = False
                        elif ttype == TaskType.SAVE:
                            p = self.b200_parameters
                            v = self._map_call("voxels", dict(
                                min_count=int(p["kVolumetricIntegrationVoxelGridMinCount"]),
                                min_confidence=float(p["kVolumetricIntegrationVoxelGridMinConfidence"])))
                            if len(v.points):
                                write_ply_points(self.last_input_task.load_save_path, v.points, v.colors)
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
            except Exception as e:  # the reference logs and keeps the loop alive (:720-730)
                printer = getattr(Base, "print", print)
                printer(f"VolumetricIntegratorB200SemanticGrid: EXCEPTION: {e} !!!")
                printer(traceback.format_exc())
            time_volumetric_integration.value = time.perf_counter() - t_start

        def _stop_volume_integrator_implementation(self):
            self._stop_shards()
            if getattr(self, "volume", None) is not None:
                self.volume.close()

    return VolumetricIntegratorB200SemanticGrid


def make_voxel_grid_integrator_class(Base, api):
    """The point-average backend (`VolumetricIntegratorVoxelGrid`, pyslam/dense/volumetric_integrator_voxel_grid.py)
    on the GPU compat grid.  Same task loop as the semantic class; the loop body is reference :232-300: optional
    shadow filter -> depth2pointcloud -> world transform -> optional carve (with the UNFILTERED depth, :283-296) ->
    integrate, all of which `VoxelBlockGrid.carve` / `integrate_rgbd` do on the device."""
    SemanticCls = make_semantic_integrator_class(Base, api)

    class VolumetricIntegratorB200VoxelGrid(SemanticCls):
        _defaults = dict(DEFAULT_PARAMETERS, kVolumetricIntegrationB200CapacityBlocks=1 << 17)
        _SHARD_KIND = "voxel_grid"
        _LABELS = False

        def _make_grid(self, p, side, constructor_kwargs):
            return VoxelBlockGrid(**dict(_grid_args(p, self.b200_set_parameters), **self._map_placement()),
                                  input_order_sums=bool(p["kVolumetricIntegrationB200InputOrderSums"]))

        def _integrate_raw(self, kd, depth, scale, use_instances):
            """Staged raw images: carve with the UNFILTERED depth, integrate the filtered one (:283-296)."""
            p = self.b200_parameters
            fr = self.volume.set_frame(depth, kd.img, depth_scale=scale,
                                       filter_shadow_points=bool(p["kVolumetricIntegrationVoxelGridShadowPointsFilter"]))
            if p["kVolumetricIntegrationVoxelGridUseCarving"]:
                self.camera_frustrum.set_T_cw(kd.pose)
                self.volume.carve(self.camera_frustrum, fr.depth,
                                  float(p["kVolumetricIntegrationVoxelGridCarvingDepthThreshold"]))
            fx, fy, cx, cy = self._intrinsics()
            Twc = np.linalg.inv(np.asarray(kd.pose, np.float64).reshape(4, 4))
            self.volume.integrate_rgbd(fr.filtered_depth, fr.color, (fx, fy, cx, cy), Twc,
                                       max_depth=self.volumetric_integration_depth_trunc, filter_shadow_points=False)
            self.last_integrated_id = kd.id
            return True

        def _integrate_prepared(self, kd, color, depth, classes, instances):
            p = self.b200_parameters
            depth = np.ascontiguousarray(depth, np.float32)
            if p["kVolumetricIntegrationVoxelGridUseCarving"]:
                self.camera_frustrum.set_T_cw(kd.pose)
                self.volume.carve(self.camera_frustrum, depth,
                                  float(p["kVolumetricIntegrationVoxelGridCarvingDepthThreshold"]))
            fx, fy, cx, cy = self._intrinsics()
            Twc = np.linalg.inv(np.asarray(kd.pose, np.float64).reshape(4, 4))
            self.volume.integrate_rgbd(depth, color, (fx, fy, cx, cy), Twc,
                                       max_depth=self.volumetric_integration_depth_trunc,
                                       filter_shadow_points=bool(p["kVolumetricIntegrationVoxelGridShadowPointsFilter"]))
            self.last_integrated_id = kd.id
            return True

        def _make_output(self, task_type):
            v = self._map_call("voxels", dict(min_count=int(self.b200_parameters["kVolumetricIntegrationVoxelGridMinCount"])))
            pc = api.VolumetricIntegrationPointCloud(points=np.ascontiguousarray(v.points, np.float32),
                                                     colors=np.ascontiguousarray(v.colors, np.float32))
            return api.VolumetricIntegrationOutput(task_type, self.last_integrated_id, pc, None)

    return VolumetricIntegratorB200VoxelGrid


def load_pyslam_semantic_plugin():
    """The semantic plugin built against the real pySLAM types (requires pySLAM on sys.path)."""
    from types import SimpleNamespace

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
        VolumetricIntegrationObjectList=B.VolumetricIntegrationObjectList,
        DatasetEnvironmentType=DatasetEnvironmentType, Parameters=Parameters)
    try:   # colours of the viewer: semantic palette and per-object id colours (reference :535-575)
        from pyslam.semantics.semantic_mapping_shared import SemanticMappingShared
        from pyslam.utilities.colors import IdsColorTable
        api.sem_img_to_rgb = SemanticMappingShared.sem_img_to_rgb
        api.ids_to_rgb_float = IdsColorTable().ids_to_rgb_float
    except Exception:
        pass
    return make_semantic_integrator_class(B.VolumetricIntegratorBase, api)
