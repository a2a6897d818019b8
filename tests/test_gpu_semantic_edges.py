"""GPU: the semantic grids (b2v_semantic.cu) at the edges of their label state machines, against
`oracle.numpy_semantic_grid` - a plain per-voxel restatement that tests/test_semantic_oracle_cpu.py pins to the
reference's committed dumps.  The scenes (tests/_semantic_scenes.py) have exact sums, so after EVERY step of a scene
every dump field (counts, float64 position sums, float32 colour sums, labels, counters, label slots, evidence,
confidence), the read-outs, the overflow count and the next object id must be equal, not close: both sides evaluate
exp and log in float64 and round once.  Only the randomised stream allows the bounds of tests/test_gpu_semantic.py on
Bayesian evidence and confidence.

Not covered: NaN depths and NaN points (the reference's behaviour is not established), label id INT32_MIN (the
association's pending marker), float64 colours."""

import numpy as np
import pytest

import oracle
from pyslam_b200 import BoundingBox3D, VoxelBlockSemanticGrid, VoxelBlockSemanticProbabilisticGrid, sharding
from tests import _grid_prep_scenes as E
from tests import _semantic_scenes as SC
from tests._util import sort_dump

pytestmark = pytest.mark.gpu
KINDS = ("voting", "probabilistic")
SCENES = SC.scenes()


def _grids(kind, scene, shards=1, **kw):
    cls_t = VoxelBlockSemanticGrid if kind == "voting" else VoxelBlockSemanticProbabilisticGrid
    kw.setdefault("capacity_blocks", 1 << 10)
    grids = [cls_t(SC.VS, 8, shard_rank=r, shard_count=shards, **kw) for r in range(shards)]
    G = oracle.numpy_semantic_grid(SC.VS, kind)
    for t in grids + [G]:
        if "depth_threshold" in scene:
            t.set_depth_threshold(scene["depth_threshold"])
        if "depth_decay_rate" in scene:
            t.set_depth_decay_rate(scene["depth_decay_rate"])
    return grids, G


def _rows(points, colors, class_ids, object_ids, confidences):
    a = np.concatenate([points, np.asarray(colors, np.float64), np.asarray(class_ids, np.float64)[:, None],
                        np.asarray(object_ids, np.float64)[:, None], np.asarray(confidences, np.float64)[:, None]], 1)
    return a[np.lexsort(a.T[::-1])]


def _same_voxels(outs, ref, exact, where):
    got = _rows(*[np.concatenate([getattr(o, n) for o in outs])
                  for n in ("points", "colors", "class_ids", "object_ids", "confidences")])
    exp = _rows(ref["points"], ref["colors"], ref["class_ids"], ref["object_ids"], ref["confidences"])
    assert got.shape == exp.shape, (where, got.shape, exp.shape)
    assert np.array_equal(got[:, :8], exp[:, :8]), where
    if exact:
        assert np.array_equal(got[:, 8], exp[:, 8]), where
    else:   # Bayesian confidence within 2e-6 relative, as tests/test_gpu_semantic.py (exp / log rounding)
        assert np.allclose(got[:, 8], exp[:, 8], rtol=2e-6, atol=1e-9), where


def _same_state(grids, G, scene, where):
    exact = not scene.get("rtol")
    d = sharding.merge_dumps([sort_dump(g.dump_blocks(8)) for g in grids])
    r = G.dump()
    for k in ("keys", "count", "pos_sum", "col_sum", "object_id", "class_id", "aux", "lab_obj", "lab_cls"):
        assert np.array_equal(d[k], r[k]), (where, k)
    if exact:
        assert np.array_equal(d["lab_logp"], r["lab_logp"]), where
        assert np.array_equal(d["confidence"], r["confidence"]), where
    else:
        # one-ulp exp differences on depth-decay weights: the bounds of tests/test_gpu_semantic.py, no more
        fin = np.isfinite(r["lab_logp"])
        assert np.array_equal(np.isfinite(d["lab_logp"]), fin), where
        assert np.allclose(d["lab_logp"][fin], r["lab_logp"][fin], rtol=1e-6, atol=0), where
        assert np.allclose(d["confidence"], r["confidence"], rtol=2e-6, atol=1e-9), where
    assert sum(g.label_overflows() for g in grids) == G.label_overflows, where
    if len(grids) == 1:
        assert grids[0].get_next_object_id() == G.next_object_id, where
    # a confidence threshold may split voxels whose confidences differ in the last bit: thresholds only when exact
    queries = [(1, 0.0), (2, 0.0)] + ([(1, c) for c in scene.get("confidences", (0.5,))] if exact else [])
    for mc, conf in queries:
        _same_voxels([g.get_voxels(mc, conf) for g in grids], G.get_voxels(mc, conf), exact, (where, mc, conf))
    for bb in scene.get("boxes", []):
        for mc, conf in queries[:3]:
            _same_voxels([g.get_voxels_in_bb(BoundingBox3D(*bb), mc, conf) for g in grids],
                         G.get_voxels_in_bb(bb, mc, conf), exact, (where, "box", mc, conf))
    for c in scene.get("cams", []):
        fr = SC._frustrum(c)
        for mc, conf in queries[:3]:
            _same_voxels([g.get_voxels_in_camera_frustrum(fr, mc, conf) for g in grids],
                         G.get_voxels_in_camera_frustrum(c["K"], c["W"], c["H"], c["Tcw"], c["depth_max"],
                                                         c["depth_min"], mc, conf), exact, (where, "frustum", mc, conf))


def _play(scene, kind, name, shards=1, **kw):
    grids, G = _grids(kind, scene, shards, **kw)
    for i, (op, step) in enumerate(scene["steps"]):
        maps = [SC.apply(g, "gpu", op, step) for g in grids]
        m = SC.apply(G, "oracle", op, step)
        if op == "assign":
            assert maps[0] == m, (name, i, maps[0], m)
        _same_state(grids, G, scene, (name, kind, i, op))
    for g in grids:
        g.close()
    return G


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name", sorted(SCENES))
def test_scene_equals_the_oracle_after_every_step(name, kind):
    """One scene per edge: slot eviction (and the same stream split at the first eviction), the order of the softmax
    fold, depths at the threshold, argmax ties, a colourless call before the first labels (fresh and after clear), a
    labelled call after every edit, the edits on -1 and equal ids, the int confidence threshold, the voting counter
    through zero, extreme label ids, the association's resolve edges (with and without depth image and carving), box
    faces and image borders on voxel means with carve, and confidence thresholds equal to a voxel's confidence."""
    G = _play(SCENES[name], kind, name)
    if name.startswith("eviction") and kind == "probabilistic":
        assert G.label_overflows == 15
    if name.startswith("frustum") or name.startswith("box"):
        assert len(G.keys) > 8


@pytest.mark.parametrize("kind", KINDS)
def test_colourless_call_on_storage_mapped_by_growth(kind):
    """The first (colourless) call touches 27 blocks of a grid created with storage for 8: the label state the later
    labelled call reads is the cleared state the growth wrote."""
    scene = SC.scene_positions_only_first(many_blocks=True)
    grids, G = _grids(kind, scene, capacity_blocks=8, max_capacity_blocks=1 << 10)
    _, growths = grids[0].capacity()
    assert growths == 0
    for i, (op, step) in enumerate(scene["steps"]):
        SC.apply(grids[0], "gpu", op, step)
        SC.apply(G, "oracle", op, step)
        _same_state(grids, G, scene, ("grown", kind, i))
        if i == 0:
            assert grids[0].capacity()[1] >= 1
    grids[0].close()


@pytest.mark.parametrize("kind", KINDS)
def test_input_variants_equal_the_oracle(kind):
    """float32 / float64 points, float32 / uint8 colours, absent instance ids (object id 0) and depths, n = 0 and
    n = 1, one 100 000-point run in a single voxel and a call where every point has its own voxel."""
    scene = dict(depth_threshold=2.0, depth_decay_rate=0.8, rtol=True)
    for name, kw in SC.input_variants():
        grids, G = _grids(kind, scene, capacity_blocks=1 << 12)
        SC.apply(grids[0], "gpu", "integrate", {k: v[:0] for k, v in kw.items() if v is not None})     # n = 0
        assert grids[0].empty()
        for t, backend in ((grids[0], "gpu"), (G, "oracle")):
            SC.apply(t, backend, "integrate", kw)
        _same_state(grids, G, scene, (name, kind))
        if name == "one_long_run":
            d = G.dump()
            assert d["count"].max() == 100000 and (d["count"] > 0).sum() == 1
            assert kind == "voting" or G.label_overflows > 1000      # 9 pairs compete for 8 slots
        if name == "one_voxel_each":
            assert G.dump()["count"].max() == 1
        if name == "no_instances":
            assert set(np.unique(G.dump()["object_id"])) <= {-1, 0}
        grids[0].close()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("layout", ["plain", "grown_from_8", "three_shards"])
def test_randomised_stream_with_edits_equals_the_oracle(layout, kind):
    """About 50 000 points in four calls, the five edits (merge, remove segment, remove low count, carve, remove low
    confidence), two more calls; compared after every step.  Also on a grid that grows from 8 blocks and on three
    shards whose dumps are merged."""
    T0, _ = E.cam_poses()
    kw = dict(plain=dict(capacity_blocks=1 << 11), grown_from_8=dict(capacity_blocks=8, max_capacity_blocks=1 << 11),
              three_shards=dict(capacity_blocks=1 << 11, shards=3))[layout]
    G = _play(SC.scene_random(T0), kind, layout, **kw)
    d = G.dump()
    assert len(d["keys"]) > 100 and (d["count"] > 0).sum() > 3000 and d["count"].max() > 8


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shadow", [False, True])
def test_labelled_rgbd_frames_equal_the_oracle(shadow, kind):
    """integrate_rgbd with class and object images on the exact-sum frames, shadow filter off and on, against the
    oracle fed the numpy front end (filter_shadow_points, depth2pointcloud, world transform)."""
    scene = dict(depth_threshold=1.5, depth_decay_rate=0.5)
    grids, G = _grids(kind, scene)
    cls_img, obj_img = SC.rgbd_labels()
    max_depth = 1.9
    removed = 0
    for i, (d, c, Twc) in enumerate(E.rgbd_frames()):
        grids[0].integrate_rgbd(d, c, E.RGBD_K, Twc, cls_img, obj_img, max_depth=max_depth, use_depths=i != 1,
                                filter_shadow_points=shadow)
        df = oracle.numpy_shadow_filter(d)[0] if shadow else d
        removed += int((df != d).sum())
        p, col = E.rgbd_points(df, c, E.RGBD_K, Twc, max_depth)
        valid = (df > 0) & (df < max_depth)
        G.integrate(p, col, cls_img[valid], obj_img[valid], df[valid] if i != 1 else None)
        _same_state(grids, G, scene, ("rgbd", shadow, kind, i))
    assert (removed > 0) == shadow and (G.dump()["count"] > 0).sum() > 2000
    grids[0].close()
