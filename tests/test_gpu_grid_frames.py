"""GPU: raw camera frames for the point-average and semantic grids (`set_rectification` / `set_frame` /
`remap_instance_ids`, b2v_grid.cu, b2v_semantic.cu, b2v_prep.cu).

The staged images must equal the host preparation bit for bit (live cv2.remap / cvtColor, numpy's uint16 widening,
`oracle.numpy_shadow_filter`, `remap_instance_ids`), grids fed from staged frames must equal grids fed host-prepared
frames, and both grid plugins must give the same output with the device preparation on or off."""

import os
from types import SimpleNamespace

import numpy as np
import pytest

import oracle
from pyslam_b200 import (CameraFrustrum, VoxelBlockGrid, VoxelBlockSemanticGrid, VoxelBlockSemanticProbabilisticGrid,
                         remap_instance_ids)
from pyslam_b200 import synthetic as S
from tests import _grid_prep_scenes as E
from tests import plugin_standins as P
from tests._util import GOLDEN, sort_dump

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
f32 = np.float32
SEM = {"vote": VoxelBlockSemanticGrid, "prob": VoxelBlockSemanticProbabilisticGrid}
SEM_KEYS = ("keys", "count", "pos_sum", "col_sum", "object_id", "class_id", "confidence", "aux", "lab_obj", "lab_cls",
            "lab_logp")
TUM1_D = np.array([0.262383, -0.953104, -0.005358, 0.002628, 1.163314])   # settings/TUM1.yaml distortion


def tum_maps(cfg):
    K = np.array([[cfg.fx, 0, cfg.cx], [0, cfg.fy, cfg.cy], [0, 0, 1]])
    return cv2.initUndistortRectifyMap(K, TUM1_D, None, K, (cfg.width, cfg.height), cv2.CV_32FC1)


def host_prepare(mx, my, depth, bgr, cls=None, inst=None, scale=None, flt=False):
    """The host preparation of a raw frame: depth.astype(float32) * factor, cv2.remap (depth / labels nearest, colour
    linear), cvtColor, the shadow filter."""
    d = depth.astype(f32) * f32(scale) if scale is not None else depth
    rm = (lambda a, i: cv2.remap(a, mx, my, i)) if mx is not None else (lambda a, i: a)
    out = dict(depth=rm(d, cv2.INTER_NEAREST), color=cv2.cvtColor(rm(bgr, cv2.INTER_LINEAR), cv2.COLOR_BGR2RGB))
    out["filtered_depth"] = oracle.numpy_shadow_filter(out["depth"], 2, 2, -1.0)[0] if flt else out["depth"]
    if cls is not None:
        out["class_image"] = rm(cls, cv2.INTER_NEAREST)
    if inst is not None:
        out["instance_image"] = rm(inst, cv2.INTER_NEAREST)
    return out


def raw_labels(cfg, i, d):
    cls = S.render_class_ids(cfg, i)
    inst = np.where(cls % 3 == 0, -1, cls * 7 + (np.arange(cls.shape[1])[None, :] // 400)).astype(np.int32)
    inst[d == 0] = 0
    return cls, inst


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == f32 else a


def _edge_case(kind):
    H, W = 61, 83
    mx, my = E.remap_maps(kind, H, W, seed=W)
    rng = np.random.default_rng(7)
    d = E._plane(rng, H, W)
    d[10:30, 20:50] += f32(0.5)
    return mx, my, d


# ---- staged images ---------------------------------------------------------------------------------------------------

CASES = ["T0", "C3", "none"] + [f"edge_{k}" for k in ("nan_both", "huge", "half", "ties64")]


@pytest.mark.parametrize("device_inputs", [False, True])
@pytest.mark.parametrize("u16", [False, True])
@pytest.mark.parametrize("case", CASES)
def test_staged_images_equal_host_references(case, u16, device_inputs):
    import torch
    rng = np.random.default_rng(len(case))
    if case == "T0":
        g = np.load(os.path.join(GOLDEN, "remap_T0.npz"))
        mx, my, d = g["map1"], g["map2"], g["depth"]
    elif case == "C3":
        cfg = S.CONFIGS["C3"]
        mx, my = tum_maps(cfg)
        d = S.render_frame(cfg, 0)[0]
    elif case == "none":
        mx = my = None
        d = S.render_frame(S.CONFIGS["T0"], 3)[0]
    else:
        mx, my, d = _edge_case(case[5:])
    H, W = d.shape
    raw16 = np.round(d * 5000).astype(np.uint16)
    scale = f32(1.0 / 5000) if u16 else None
    depth = raw16 if u16 else d
    bgr = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    cls = rng.integers(-2, 20, (H, W)).astype(np.int32)
    inst = rng.integers(-3, 2 ** 31 - 1, (H, W)).astype(np.int32)
    ref = host_prepare(mx, my, raw16 if u16 else d, bgr, cls, inst, scale, flt=True)
    grid = VoxelBlockSemanticGrid(0.05, 8, capacity_blocks=64)
    pgrid = VoxelBlockGrid(0.05, 8, capacity_blocks=64)
    for gr in (grid, pgrid):
        if mx is not None:
            gr.set_rectification(mx, my, swap_rb=True)
        else:   # without maps the colour is taken as it is (RGB)
            ref["color"] = bgr
    args = [depth, bgr, cls, inst]
    if device_inputs:
        args = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in args]
    for flt in (True, False):
        fr = grid.set_frame(*args, depth_scale=scale, filter_shadow_points=flt)
        for name in ("depth", "color", "class_image", "instance_image"):
            assert np.array_equal(bits(getattr(fr, name).numpy()), bits(ref[name])), name
        want = ref["filtered_depth"] if flt else ref["depth"]
        assert np.array_equal(bits(fr.filtered_depth.numpy()), bits(want))
        pf = pgrid.set_frame(args[0], args[1], depth_scale=scale, filter_shadow_points=flt)
        for name in ("depth", "filtered_depth", "color"):
            assert np.array_equal(bits(getattr(pf, name).numpy()), bits(getattr(fr, name).numpy())), name
    assert pf.depth.torch().is_cuda
    grid.set_frame(*args, depth_scale=scale)
    with pytest.raises(RuntimeError, match="stale"):
        fr.depth.numpy()
    grid.close()
    pgrid.close()


def test_device_instance_remap_equals_host_remap():
    """Labelled pixels, misses (class < 0, negative ids), an empty map (no pixel with a class)."""
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    K = g["K"]
    grid = VoxelBlockSemanticGrid(float(g["voxel_size"]), 8, capacity_blocks=1024)
    for i in range(int(g["n_frames"])):
        d, c, T = g[f"depth_{i}"], g[f"color_{i}"], g[f"Tcw_{i}"]
        cls_img, inst_img = g[f"class_image_{i}"].copy(), g[f"instance_image_{i}"].copy()
        cls_img[:, :7] = -1
        inst_img[:5] = -4
        fr = CameraFrustrum(K[0], K[1], K[2], K[3], d.shape[1], d.shape[0], T, depth_max=8.0, depth_min=1e-2)
        for labels in ((cls_img, inst_img), (np.full_like(cls_img, -1), inst_img)):
            f = grid.set_frame(d, c, *labels)
            m = grid.assign_object_ids_to_instance_ids(fr, f.class_image, f.instance_image, f.depth,
                                                       depth_threshold=0.08, do_carving=False)
            assert (len(m) > 0) == (labels[0] is cls_img)
            ref = remap_instance_ids(labels[1], m)
            got = grid.remap_instance_ids()
            assert got is f.object_image and np.array_equal(got.numpy(), ref)
            if not m:
                assert (ref == -1).all()
        grid.integrate_rgbd(d, c, K, np.linalg.inv(T), g[f"class_image_{i}"], max_depth=4.0)
    assert grid.num_blocks() > 10


# ---- grids: raw-frame path == host path --------------------------------------------------------------------------

def _semantic_run(tag, frames, mx, my, cfg, raw, flt, **kw):
    grid = SEM[tag](0.015, 8, **kw)
    grid.set_depth_threshold(1.5)
    if raw:
        grid.set_rectification(mx, my, swap_rb=True)
    maps = []
    for d16, bgr, cls, inst, Tcw in frames:
        fr_ = CameraFrustrum(cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.width, cfg.height, Tcw, depth_max=8.0, depth_min=1e-2)
        a = dict(depth_threshold=0.05, do_carving=True, min_vote_ratio=0.5, min_votes=3)
        if raw:
            f = grid.set_frame(d16, bgr, cls, inst, depth_scale=f32(1 / 5000), filter_shadow_points=flt)
            maps.append(grid.assign_object_ids_to_instance_ids(fr_, f.class_image, f.instance_image, f.filtered_depth,
                                                               **a))
            grid.integrate_rgbd(f.filtered_depth, f.color, cfg.K, np.linalg.inv(Tcw), f.class_image,
                                grid.remap_instance_ids(), max_depth=cfg.depth_trunc, filter_shadow_points=False)
        else:
            h = host_prepare(mx, my, d16, bgr, cls, inst, f32(1 / 5000))
            dd = oracle.numpy_shadow_filter(h["depth"], 2, 2, -1.0)[0] if flt else h["depth"]
            maps.append(grid.assign_object_ids_to_instance_ids(fr_, h["class_image"], h["instance_image"], dd, **a))
            grid.integrate_rgbd(h["depth"], h["color"], cfg.K, np.linalg.inv(Tcw), h["class_image"],
                                remap_instance_ids(h["instance_image"], maps[-1]), max_depth=cfg.depth_trunc,
                                filter_shadow_points=flt)
    out = sort_dump(grid.dump_blocks(8)), maps, grid.capacity()[1]
    grid.close()
    return out


@pytest.mark.parametrize("tag", ["vote", "prob"])
def test_semantic_grids_raw_frames_equal_host_path(tag):
    cfg = S.CONFIGS["C3"]
    mx, my = tum_maps(cfg)
    frames = []
    for i in (0, 25, 50):
        d, c, Tcw = S.render_frame(cfg, i)
        cls, inst = raw_labels(cfg, i, d)
        frames.append((np.round(d * 5000).astype(np.uint16), np.ascontiguousarray(c[..., ::-1]), cls, inst, Tcw))
    for flt, kw in ((True, dict(capacity_blocks=1 << 15)), (False, dict(capacity_blocks=16, max_capacity_blocks=1 << 15))):
        a, ma, _ = _semantic_run(tag, frames, mx, my, cfg, False, flt, **kw)
        b, mb, growths = _semantic_run(tag, frames, mx, my, cfg, True, flt, **kw)
        assert ma == mb and sum(len(m) for m in ma) > 5
        for k in SEM_KEYS:
            assert np.array_equal(a[k], b[k]), (flt, k)
        assert len(a["keys"]) > 500 and (a["object_id"] > 0).any()
        if "max_capacity_blocks" in kw:
            assert growths >= 2


def test_point_grid_raw_frames_equal_host_path():
    """Carve with the unfiltered staged depth, integrate the filtered one: C2 frames with TUM-like maps (float atomics:
    sums to a tolerance), and the exact-sum RGBD scene with identity maps (sums bit for bit)."""
    cfg = S.CONFIGS["C2"]
    mx, my = tum_maps(cfg)
    frames = [S.render_frame(cfg, i) for i in (0, 10, 20, 30)]

    def run(raw):
        grid = VoxelBlockGrid(0.03, 8, capacity_blocks=1 << 14)
        if raw:
            grid.set_rectification(mx, my, swap_rb=True)
        for d, c, Tcw in frames:
            bgr = np.ascontiguousarray(c[..., ::-1])
            fr = CameraFrustrum(cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.width, cfg.height, Tcw, depth_max=8.0,
                                depth_min=1e-2)
            if raw:
                f = grid.set_frame(d, bgr, filter_shadow_points=True)
                grid.carve(fr, f.depth, 3e-2)
                grid.integrate_rgbd(f.filtered_depth, f.color, cfg.K, np.linalg.inv(Tcw), max_depth=4.0)
            else:
                h = host_prepare(mx, my, d, bgr)
                grid.carve(fr, h["depth"], 3e-2)
                grid.integrate_rgbd(h["depth"], h["color"], cfg.K, np.linalg.inv(Tcw), max_depth=4.0,
                                    filter_shadow_points=True)
        return sort_dump(grid.dump_blocks())

    a, b = run(False), run(True)
    assert np.array_equal(a["keys"], b["keys"]) and np.array_equal(a["count"], b["count"])
    assert np.allclose(a["pos_sum"], b["pos_sum"], rtol=1e-5, atol=1e-6)
    assert (a["count"] > 0).sum() > 1000
    # exact sums: identity maps (every remap reads its own pixel), dyadic depths and colours
    ix, iy = np.meshgrid(np.arange(E.RGBD_W, dtype=f32), np.arange(E.RGBD_H, dtype=f32))
    grids = [VoxelBlockGrid(E.VS_EXACT, 8, capacity_blocks=1 << 12) for _ in range(2)]
    grids[1].set_rectification(ix, iy, swap_rb=True)
    for d, c, Twc in E.rgbd_frames():
        grids[0].integrate_rgbd(d, c, E.RGBD_K, Twc, filter_shadow_points=True)
        f = grids[1].set_frame(d, np.ascontiguousarray(c[..., ::-1]), filter_shadow_points=True)
        grids[1].integrate_rgbd(f.filtered_depth, f.color, E.RGBD_K, Twc)
    a, b = (sort_dump(g.dump_blocks()) for g in grids)
    for k in ("keys", "count", "pos_sum", "col_sum"):
        assert np.array_equal(a[k], b[k]), k


# ---- plugins -------------------------------------------------------------------------------------------------------

class RectifyingBase(P.StandaloneIntegratorBase):
    """The base class's host preparation (base.py:1007-1054) in full: in C++-core mode raw depth becomes
    depth.astype(float32) * camera.depth_factor, and the class / instance images are rectified with cv2.remap
    INTER_NEAREST like depth (SURVEY a1)."""
    use_cpp = False

    def estimate_depth_if_needed_and_rectify(self, kd):
        if kd.depth is None or kd.depth.size == 0:
            return None, None, None, None, None
        depth = kd.depth
        if depth.dtype != np.float32:
            depth = depth.astype(np.float32) * self.camera.depth_factor if self.use_cpp else depth.astype(np.float32)
        color, cls, inst = kd.img, kd.semantic_img, kd.semantic_instances_img
        if self.calib_map1 is not None:
            m1, m2 = self.calib_map1, self.calib_map2
            color = cv2.remap(color, m1, m2, interpolation=cv2.INTER_LINEAR)
            depth = cv2.remap(depth, m1, m2, interpolation=cv2.INTER_NEAREST)
            cls = None if cls is None else cv2.remap(cls, m1, m2, interpolation=cv2.INTER_NEAREST)
            inst = None if inst is None else cv2.remap(inst, m1, m2, interpolation=cv2.INTER_NEAREST)
        return np.ascontiguousarray(color[..., ::-1]), depth, None, cls, inst


def _plugin(kind, use_cpp, gpu, maps, **kw):
    from pyslam_b200 import integrator_semantic as IS
    base = type("Base", (RectifyingBase,), {"use_cpp": use_cpp})
    api = SimpleNamespace(**vars(P.API), USE_CPP=use_cpp)
    make = IS.make_semantic_integrator_class if kind == "semantic" else IS.make_voxel_grid_integrator_class
    cfg = S.CONFIGS["T0"]
    cam = SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None,
                          depth_factor=1.0 / 5000)
    return make(base, api)(cam, P.DatasetEnvironmentType.INDOOR, None, "B200", calib_maps=maps,
                           kVolumetricIntegrationB200GpuRectify=gpu, **kw)


def _last_output(integ):
    out = None
    while (o := integ.pop_output()) is not None:
        out = o
    return out


@pytest.mark.parametrize("kind", ["semantic", "voxel"])
@pytest.mark.parametrize("use_cpp", [False, True])
def test_plugins_same_output_with_and_without_device_preparation(kind, use_cpp):
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    r = np.load(os.path.join(GOLDEN, "remap_T0.npz"))
    maps = (r["map1"], r["map2"])
    kw = dict(kVolumetricIntegrationVoxelLength=float(g["voxel_size"]), kVolumetricIntegrationVoxelGridUseCarving=True,
              kVolumetricIntegrationVoxelGridCarvingDepthThreshold=0.08, kVolumetricIntegrationB200CapacityBlocks=1024,
              kVolumetricIntegrationVoxelGridMinCount=1)
    if kind == "semantic":
        kw["use_semantic_probabilistic"] = True
    outs = []
    for gpu in (True, False):
        integ = _plugin(kind, use_cpp, gpu, maps, **kw)
        assert integ._gpu_rectify == gpu
        for i in range(int(g["n_frames"])):
            d = g[f"depth_{i}"]
            depth = np.round(d * 5000).astype(np.uint16) if use_cpp else d
            integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(
                id=i, pose=g[f"Tcw_{i}"], img=np.ascontiguousarray(g[f"color_{i}"][..., ::-1]), depth=depth,
                semantic_img=g[f"class_image_{i}"], semantic_instances_img=g[f"instance_image_{i}"]))
            integ.step()
        integ.add_update_output_task()
        integ.step()
        out = _last_output(integ)
        dump = sort_dump(integ.volume.dump_blocks(8) if kind == "semantic" else integ.volume.dump_blocks())
        outs.append((out, dump, getattr(integ, "last_instance_map", None)))
        integ.quit()
    (oa, da, ma), (ob, db, mb) = outs
    assert ma == mb and len(da["keys"]) > 20
    if kind == "semantic":
        for k in SEM_KEYS:
            assert np.array_equal(da[k], db[k]), k
        la, lb = oa.objects.object_list, ob.objects.object_list
        assert len(la) == len(lb) > 0
        for x, y in zip(la, lb):   # voxels come out in pool order, which block inserts race for
            assert (x.object_id, x.class_id) == (y.object_id, y.class_id)
            rows = [np.concatenate([o.points, o.colors], 1) for o in (x, y)]
            assert np.array_equal(*(q[np.lexsort(q.T[::-1])] for q in rows))
            assert np.allclose(x.box_size, y.box_size, rtol=1e-5, atol=1e-6)
    else:
        assert np.array_equal(da["keys"], db["keys"]) and np.array_equal(da["count"], db["count"])
        assert np.allclose(da["pos_sum"], db["pos_sum"], rtol=1e-5, atol=1e-6)
        pa, pb = oa.point_cloud.points, ob.point_cloud.points
        assert pa.shape == pb.shape and len(pa) > 100
        assert np.allclose(np.sort(pa, axis=0), np.sort(pb, axis=0), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("kind", ["semantic", "voxel"])
def test_plugins_take_the_host_path_without_maps_or_with_a_depth_estimator(kind):
    r = np.load(os.path.join(GOLDEN, "remap_T0.npz"))
    integ = _plugin(kind, False, True, None)
    assert not integ._gpu_rectify
    integ.quit()

    class WithEstimator(RectifyingBase):
        def init(self, *a):
            super().init(*a)
            self.depth_estimator = object()

    from pyslam_b200 import integrator_semantic as IS
    make = IS.make_semantic_integrator_class if kind == "semantic" else IS.make_voxel_grid_integrator_class
    cfg = S.CONFIGS["T0"]
    cam = SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)
    integ = make(WithEstimator, P.API)(cam, P.DatasetEnvironmentType.INDOOR, None, "B200",
                                       calib_maps=(r["map1"], r["map2"]), kVolumetricIntegrationB200CapacityBlocks=256)
    assert not integ._gpu_rectify
    d, c, T = S.render_frame(cfg, 0)
    integ.volume.set_frame = None   # the host path never stages a frame
    integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(id=0, pose=T, img=c, depth=d))
    integ.step()
    assert integ.last_integrated_id == 0 and integ.volume.num_blocks() > 0
    integ.quit()


# ---- bad arguments ---------------------------------------------------------------------------------------------------

def test_bad_arguments_are_rejected_and_leave_the_grid_unchanged():
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    r = np.load(os.path.join(GOLDEN, "remap_T0.npz"))
    d, c, T = g["depth_0"], g["color_0"], g["Tcw_0"]
    cls, inst = g["class_image_0"], g["instance_image_0"]
    grid = VoxelBlockSemanticGrid(float(g["voxel_size"]), 8, capacity_blocks=1024)
    grid.set_rectification(r["map1"], r["map2"], swap_rb=True)
    f = grid.set_frame(d, c, cls, inst)
    with pytest.raises(RuntimeError, match="association"):
        grid.remap_instance_ids()                                        # no association yet
    grid.integrate_rgbd(f.depth, f.color, g["K"], np.linalg.inv(T), f.class_image, max_depth=4.0)
    before = sort_dump(grid.dump_blocks(8))
    ref_depth = f.depth.numpy()
    H, W = d.shape
    bad = [dict(depth=d[:, :-8], color=c[:, :-8]),                       # not the maps' size
           dict(depth=np.round(d * 5000).astype(np.uint16), color=c, depth_scale=0.0),
           dict(depth=np.round(d * 5000).astype(np.uint16), color=c, depth_scale=-1.0),
           dict(depth=d, color=c, instance_image=inst)]                  # instance image without class image
    for kw in bad:
        with pytest.raises(RuntimeError):
            grid.set_frame(**kw)
    with pytest.raises(RuntimeError, match="association"):
        grid.remap_instance_ids()
    after = sort_dump(grid.dump_blocks(8))
    for k in SEM_KEYS:
        assert np.array_equal(before[k], after[k]), k
    assert np.array_equal(bits(f.depth.numpy()), bits(ref_depth))     # the staged frame survives
    pgrid = VoxelBlockGrid(0.02, 8, capacity_blocks=256)
    pgrid.set_rectification(r["map1"], r["map2"], swap_rb=True)
    with pytest.raises(RuntimeError, match="different image size"):
        pgrid.set_frame(d[:-1], c[:-1])
    with pytest.raises(RuntimeError, match="depth_scale"):
        pgrid.set_frame(np.zeros((H, W), np.uint16), c, depth_scale=0.0)
    with pytest.raises(RuntimeError, match="staged it"):
        pgrid.integrate_rgbd(f.depth, f.color, g["K"], np.linalg.inv(T))
    assert pgrid.num_blocks() == 0
    grid.close()
    pgrid.close()
