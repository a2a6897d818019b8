"""GPU: the per-call images of the point-average and semantic grids (`integrate_rgbd`, `carve` and the association;
`BlockGridCore::stage_input`, b2v_grid.cu).

A host image is uploaded into buffers the grid keeps for the largest call so far, a device image is read in place, and
the shadow filter writes a buffer no call reads from.  Those buffers are not the staged frame's: a frame from
`set_frame` must survive calls made with host arrays, a call may mix staged images with host arrays, frames of any size
must give what the same frames give as device tensors (also while the grid grows and replays a call), and an image too
small for the shadow filter is rejected before anything runs.  The association leaves its instance map on the device
for `remap_instance_ids`."""

import os

import numpy as np
import pytest

from pyslam_b200 import CameraFrustrum, VoxelBlockGrid, VoxelBlockSemanticGrid, remap_instance_ids
from pyslam_b200 import synthetic as S
from tests._util import GOLDEN, sort_dump

pytestmark = pytest.mark.gpu
f32 = np.float32
SEM_KEYS = ("keys", "count", "pos_sum", "col_sum", "object_id", "class_id", "confidence", "aux", "lab_obj", "lab_cls",
            "lab_logp")
KINDS = ["point", "semantic"]
ASSOC = dict(depth_threshold=0.08, do_carving=True, min_vote_ratio=0.5, min_votes=3)


def _golden():
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    frames = [(g[f"depth_{i}"], g[f"color_{i}"], g[f"class_image_{i}"], g[f"instance_image_{i}"], g[f"Tcw_{i}"])
              for i in range(int(g["n_frames"]))]
    return float(g["voxel_size"]), g["K"], frames


def _grid(kind, vs, **kw):
    return (VoxelBlockSemanticGrid if kind == "semantic" else VoxelBlockGrid)(vs, 8, **kw)


def _dump(grid):
    return sort_dump(grid.dump_blocks(8) if isinstance(grid, VoxelBlockSemanticGrid) else grid.dump_blocks())


def _assert_same(kind, a, b):
    if kind == "semantic":
        for k in SEM_KEYS:
            assert np.array_equal(a[k], b[k]), k
    else:   # float atomics: the sums to a tolerance
        assert np.array_equal(a["keys"], b["keys"]) and np.array_equal(a["count"], b["count"])
        for k in ("pos_sum", "col_sum"):
            assert np.allclose(a[k], b[k], rtol=1e-5, atol=1e-6), k
    assert len(a["keys"]) > 10


def _frustum(K, d, Tcw):
    return CameraFrustrum(K[0], K[1], K[2], K[3], d.shape[1], d.shape[0], Tcw, depth_max=8.0, depth_min=1e-2)


def _frame_calls(grid, kind, K, d, c, cls, inst, Tcw, staged=None, use=()):
    """One frame through the grid with the shadow filter on: carve + integrate_rgbd (point grid), or the association
    with carving + the host instance remap + integrate_rgbd (semantic grid).  Each image named in `use` is taken from
    the staged frame `staged`, the others are host arrays.  Returns the instance map (semantic grid)."""
    src = dict(depth=d, color=c, class_image=cls, instance_image=inst)
    img = {k: getattr(staged, k) if k in use else v for k, v in src.items()}
    Twc = np.linalg.inv(Tcw)
    if kind == "point":
        grid.carve(_frustum(K, d, Tcw), img["depth"], 3e-2)
        grid.integrate_rgbd(img["depth"], img["color"], K, Twc, max_depth=4.0, filter_shadow_points=True)
        return None
    m = grid.assign_object_ids_to_instance_ids(_frustum(K, d, Tcw), img["class_image"], img["instance_image"],
                                               img["depth"], **ASSOC)
    grid.integrate_rgbd(img["depth"], img["color"], K, Twc, img["class_image"], remap_instance_ids(inst, m),
                        max_depth=4.0, filter_shadow_points=True)
    return m


def _stage(grid, kind, d, c, cls, inst, flt):
    labels = (cls, inst) if kind == "semantic" else ()
    return grid.set_frame(d, c, *labels, filter_shadow_points=flt)


def _snapshot(fr):
    names = ("depth", "filtered_depth", "color", "class_image", "instance_image")
    return {k: getattr(fr, k).numpy() for k in names if getattr(fr, k) is not None}


@pytest.mark.parametrize("kind", KINDS)
def test_staged_frame_survives_calls_with_host_arrays(kind):
    vs, K, frames = _golden()
    grid = _grid(kind, vs, capacity_blocks=1024)
    fr = _stage(grid, kind, *frames[0][:4], flt=True)
    before = _snapshot(fr)
    for f in frames[1:]:
        _frame_calls(grid, kind, K, *f)
    after = _snapshot(fr)
    assert before.keys() == after.keys()
    for k in before:
        assert np.array_equal(before[k].view(np.uint8), after[k].view(np.uint8)), k
    # and the staged images still feed a call
    _frame_calls(grid, kind, K, *frames[0], staged=fr, use=("depth", "color", "class_image"))
    grid.close()


@pytest.mark.parametrize("kind", KINDS)
def test_staged_images_mixed_with_host_arrays_equal_all_host(kind):
    vs, K, frames = _golden()
    use = {"point": [("depth",), ("color",)],
           "semantic": [("depth", "class_image"), ("color", "instance_image"), ("class_image",)]}[kind]
    grids = [_grid(kind, vs, capacity_blocks=1024) for _ in range(2)]
    maps = ([], [])
    for i, f in enumerate(frames):
        fr = _stage(grids[1], kind, *f[:4], flt=False)
        maps[0].append(_frame_calls(grids[0], kind, K, *f))
        maps[1].append(_frame_calls(grids[1], kind, K, *f, staged=fr, use=use[i % len(use)]))
    assert maps[0] == maps[1]
    _assert_same(kind, *(_dump(g) for g in grids))
    for g in grids:
        g.close()


def _labels(cfg, i, d):
    cls = S.render_class_ids(cfg, i)
    inst = np.where(cls % 3 == 0, -1, cls * 7 + (np.arange(cls.shape[1])[None, :] // 100)).astype(np.int32)
    inst[d == 0] = 0
    return cls, inst


@pytest.mark.parametrize("kind", KINDS)
def test_host_frames_of_changing_size_equal_device_tensors(kind):
    """Frames that grow and shrink (T0 96x72 .. C3 1200x680, after a staged C2 frame) into a grid that grows, through
    the C calls with host pointers and with torch device pointers: the replay of a growth reads the per-call images."""
    import torch
    seq = [("T0", 3), ("C1", 5), ("C3", 0), ("C2", 40), ("C3", 20), ("T0", 9)]
    frames = []
    for name, i in seq:
        cfg = S.CONFIGS[name]
        d, c, Tcw = S.render_frame(cfg, i)
        frames.append((cfg.K, d, c, *_labels(cfg, i, d), Tcw))
    staged_cfg = S.CONFIGS["C2"]
    sd, sc, _ = S.render_frame(staged_cfg, 1)

    def run(device):
        grid = _grid(kind, 0.02, capacity_blocks=16, max_capacity_blocks=1 << 16)
        _stage(grid, kind, sd, sc, *_labels(staged_cfg, 1, sd), flt=True)
        L, h = grid._L, grid._h
        maps = []
        for K, d, c, cls, inst, Tcw in frames:
            hold = []

            def ptr(a):
                a = np.ascontiguousarray(a)
                if device:
                    a = torch.from_numpy(a).cuda()
                    torch.cuda.synchronize()
                    hold.append(a)
                    return a.data_ptr()
                hold.append(a)
                return a.ctypes.data

            H, W = d.shape
            Kf, Kd = np.asarray(K, f32), np.asarray(K, np.float64)
            T = np.ascontiguousarray(Tcw, np.float64)
            Twc = np.ascontiguousarray(np.linalg.inv(T))
            if kind == "point":
                grid._check(L.b2v_grid_carve(h, Kf.ctypes.data, W, H, T.ctypes.data, 8.0, 1e-2, ptr(d), 3e-2), "carve")
                grid._check(L.b2v_grid_integrate_rgbd(h, ptr(d), ptr(c), H, W, Kd.ctypes.data, Twc.ctypes.data, 4.0,
                                                      0.0, 1), "integrate_rgbd")
                grid._check(L.b2v_grid_synchronize(h), "synchronize")
                continue
            n = L.b2v_sgrid_assign_object_ids_to_instance_ids(h, Kf.ctypes.data, W, H, T.ctypes.data, 8.0, 1e-2,
                                                              ptr(cls), ptr(inst), ptr(d), 0.08, 1, 0.5, 3)
            assert n >= 0
            ids, objs = np.zeros(n, np.int32), np.zeros(n, np.int32)
            grid._check(L.b2v_sgrid_copy_instance_map(h, ids.ctypes.data, objs.ctypes.data), "copy_instance_map")
            maps.append(dict(zip(ids.tolist(), objs.tolist())))
            grid._check(L.b2v_sgrid_integrate_rgbd(h, ptr(d), ptr(c), ptr(cls), ptr(remap_instance_ids(inst, maps[-1])),
                                                   H, W, Kd.ctypes.data, Twc.ctypes.data, 4.0, 0.0, 1, 1),
                        "integrate_rgbd")
        out = _dump(grid), maps, grid.capacity()[1]
        grid.close()
        return out

    (a, ma, ga), (b, mb, gb) = run(False), run(True)
    assert ma == mb and ga == gb >= 2
    _assert_same(kind, a, b)


@pytest.mark.parametrize("kind", KINDS)
def test_too_small_images_with_the_filter_are_rejected_and_leave_the_grid_unchanged(kind):
    vs, K, frames = _golden()
    grid = _grid(kind, vs, capacity_blocks=1024)
    _frame_calls(grid, kind, K, *frames[0])
    before = _dump(grid)
    d, c, cls, inst, Tcw = frames[1]
    for sl in (np.s_[:2, :], np.s_[:, :2], np.s_[:1, :1]):
        labels = (cls[sl], inst[sl]) if kind == "semantic" else ()
        with pytest.raises(RuntimeError, match="too small for the shadow filter"):
            grid.integrate_rgbd(d[sl], c[sl], K, np.linalg.inv(Tcw), *labels, max_depth=4.0, filter_shadow_points=True)
    _assert_same(kind, before, _dump(grid))
    grid.close()


@pytest.mark.parametrize("case", ["empty", "no_pending", "pending"])
def test_remap_after_an_association_equals_numpy(case):
    """The association's map reaches remap_instance_ids on an empty grid, on one whose voxels all lie outside the
    frustum (no pending voxels) and on one whose voxels have no object yet (pending: new object ids)."""
    vs, K, frames = _golden()
    grid = VoxelBlockSemanticGrid(vs, 8, capacity_blocks=1024)
    d, c, cls, inst, Tcw = frames[0]
    if case != "empty":   # what an empty map makes of the instances: object -1, no object yet
        grid.integrate_rgbd(d, c, K, np.linalg.inv(Tcw), cls, remap_instance_ids(inst, {}), max_depth=4.0)
        assert grid.num_blocks() > 0
    look = Tcw.copy()
    if case == "no_pending":   # the camera 100 m away: nothing in its frustum
        look[:3, 3] += 100.0
    fr = grid.set_frame(d, c, cls, inst)
    next_id = grid.get_next_object_id()
    m = grid.assign_object_ids_to_instance_ids(_frustum(K, d, look), fr.class_image, fr.instance_image, fr.depth,
                                               **ASSOC)
    assert len(m) > 0
    assert (grid.get_next_object_id() > next_id) == (case == "pending")
    if case == "pending":
        assert max(m.values()) >= next_id
    got = grid.remap_instance_ids()
    assert np.array_equal(got.numpy(), remap_instance_ids(fr.instance_image.numpy(), m))
    grid.close()
