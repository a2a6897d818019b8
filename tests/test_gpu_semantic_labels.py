"""GPU: the Bayesian grid with an overflow label store (`max_label_overflow_pairs`) against the unbounded label map of
tests/_semantic_labels.py after every call: counts, sums, argmax, ml_logp (via the argmax evidence), every pair's
evidence and the number of pairs equal, not close; no eviction below the ceiling.  The randomised churn stream allows
the bounds of tests/test_gpu_semantic_edges.py on depth-decayed evidence and confidence.  Also: chunks released by the
edits are reused, clear empties the pool, the ceiling (status, chunks used, evictions counted), and ceiling 0 is the
grid without a store."""

import numpy as np
import pytest

from pyslam_b200 import VoxelBlockSemanticGrid, VoxelBlockSemanticProbabilisticGrid, sharding
from tests import _grid_prep_scenes as E
from tests import _semantic_labels as SL
from tests import _semantic_scenes as SC
from tests._util import sort_dump

pytestmark = pytest.mark.gpu
BIG = 1 << 20   # a ceiling no scene reaches


def _grids(scene, shards=1, vs=SC.VS, **kw):
    kw.setdefault("capacity_blocks", 1 << 10)
    kw.setdefault("max_label_overflow_pairs", BIG)
    grids = [VoxelBlockSemanticProbabilisticGrid(vs, 8, shard_rank=r, shard_count=shards, **kw)
             for r in range(shards)]
    G = SL.UnboundedSemanticGrid(vs)
    for t in grids + [G]:
        if "depth_threshold" in scene:
            t.set_depth_threshold(scene["depth_threshold"])
        if "depth_decay_rate" in scene:
            t.set_depth_decay_rate(scene["depth_decay_rate"])
    return grids, G


def _same_state(grids, G, exact, where):
    K = max(8, G.max_pairs())
    d = sharding.merge_dumps([sort_dump(g.dump_blocks(K)) for g in grids])
    r = G.dump(K)
    for k in ("keys", "count", "pos_sum", "col_sum", "object_id", "class_id", "aux", "lab_obj", "lab_cls"):
        assert np.array_equal(d[k], r[k]), (where, k)
    if exact:
        assert np.array_equal(d["lab_logp"], r["lab_logp"]), where
        assert np.array_equal(d["confidence"], r["confidence"]), where
    else:
        fin = np.isfinite(r["lab_logp"])
        assert np.array_equal(np.isfinite(d["lab_logp"]), fin), where
        assert np.allclose(d["lab_logp"][fin], r["lab_logp"][fin], rtol=1e-6, atol=0), where
        assert np.allclose(d["confidence"], r["confidence"], rtol=2e-6, atol=1e-9), where
    assert sum(g.label_overflows() for g in grids) == 0, where
    v = [g.get_voxels(1, 0.0) for g in grids]
    o = G.get_voxels(1, 0.0)
    assert sum(len(x.points) for x in v) == len(o["points"]), where
    used = sum(g.label_storage()["used"] for g in grids)
    assert used == sum(SL.chunks_of(len(s)) for s in G.slots.values()), (where, used)


def _play(scene, name, shards=1, **kw):
    grids, G = _grids(scene, shards, **kw)
    exact = not scene.get("rtol")
    for i, (op, step) in enumerate(scene["steps"]):
        maps = [SC.apply(g, "gpu", op, step) for g in grids]
        m = SC.apply(G, "oracle", op, step)
        if op == "assign":
            assert maps[0] == m, (name, i)
        _same_state(grids, G, exact, (name, i, op))
    return grids, G


SCENES = dict({k: v for k, v in SC.scenes().items()
               if k in ("eviction", "eviction_split", "softmax_fold", "argmax_ties", "depth_threshold",
                        "labelled_after_edits", "edit_ids", "association", "frustum0")},
              **{f"pairs{n}": SL.scene_many_pairs(n) for n in (9, 17, 40)})


@pytest.mark.parametrize("name", sorted(SCENES))
def test_scene_equals_the_unbounded_map_after_every_step(name):
    """The eviction scenes (9, 10 and 17 pairs, ties, argmax in slot 0 and slot 7, the stream cut at the ninth pair)
    keep every pair; the many-pair scenes add an argmax that arrives in a chunk, depth-decayed evidence, the edits
    followed by labelled calls, and clear.  The chunk storage starts at one chunk and grows inside the calls."""
    grids, G = _play(SCENES[name], name, initial_label_overflow_pairs=8)
    if name.startswith("eviction") or name.startswith("pairs"):
        assert G.max_pairs() > 8
        assert grids[0].label_storage()["growths"] > 0
    for g in grids:
        g.close()


def test_edits_release_chunks_that_later_calls_reuse():
    kw = SC.stream(SL.many_pair_streams(40))
    g = VoxelBlockSemanticProbabilisticGrid(SC.VS, 8, capacity_blocks=64, max_label_overflow_pairs=BIG)
    g.integrate(**kw)
    first = g.label_storage()
    assert first["used"] >= 5 * SL.chunks_of(40)
    ref = sort_dump(g.dump_blocks())
    g.remove_low_count_voxels(1 << 20)        # every voxel reset: every chain back on the free list
    assert g.label_storage()["used"] == 0
    g.integrate(**kw)
    again = g.label_storage()
    assert again["used"] == first["used"] and again["mapped"] == first["mapped"]
    assert again["growths"] == first["growths"]
    d = sort_dump(g.dump_blocks())
    for k in ("count", "lab_obj", "lab_cls", "lab_logp", "aux", "confidence", "object_id"):
        assert np.array_equal(d[k], ref[k]), k
    g.clear()
    s = g.label_storage()
    assert s["used"] == 0 and s["mapped"] == first["mapped"]
    g.integrate(**kw)
    assert g.label_storage()["used"] == first["used"]
    g.close()


@pytest.mark.parametrize("layout", ["plain", "grown_from_1_chunk", "three_shards"])
def test_churn_stream_with_edits_equals_the_unbounded_map(layout):
    """About 50 000 points in four calls whose instance ids churn (most voxels pass 8 pairs), the five edits (merge,
    remove segment, remove low count, carve, remove low confidence), two more calls; after every step."""
    T0, _ = E.cam_poses()
    kw = dict(plain=dict(capacity_blocks=1 << 11), grown_from_1_chunk=dict(capacity_blocks=8, max_capacity_blocks=1 << 11,
                                                                          initial_label_overflow_pairs=1),
              three_shards=dict(capacity_blocks=1 << 11, shards=3))[layout]
    grids, G = _play(SL.scene_churn(T0), layout, **kw)
    assert G.max_pairs() > 8
    if layout == "grown_from_1_chunk":
        assert grids[0].label_storage()["growths"] > 0
    for g in grids:
        g.close()


def test_labelled_rgbd_frames_with_object_ids_that_change_every_frame():
    """integrate_rgbd with class images and object images whose ids change every frame and jitter per pixel, at
    2^-3 m voxels (many pixels per voxel), against the unbounded map fed the numpy front end."""
    scene = dict(depth_threshold=1.5, depth_decay_rate=0.5)
    grids, G = _grids(scene, vs=0.125, initial_label_overflow_pairs=8)
    cls_img, obj_img = SC.rgbd_labels()
    rng = np.random.default_rng(4)
    frames = E.rgbd_frames(n=3) + E.rgbd_frames(seed=8, n=3)
    for i, (d, c, Twc) in enumerate(frames):
        obj = (obj_img + 1000 * i + 10 * rng.integers(0, 64, obj_img.shape)).astype(np.int32)
        grids[0].integrate_rgbd(d, c, E.RGBD_K, Twc, cls_img, obj, max_depth=1.9, use_depths=i != 1)
        p, col = E.rgbd_points(d, c, E.RGBD_K, Twc, 1.9)
        valid = (d > 0) & (d < 1.9)
        G.integrate(p, col, cls_img[valid], obj[valid], d[valid] if i != 1 else None)
        _same_state(grids, G, True, ("rgbd", i))
    assert G.max_pairs() > 8
    grids[0].close()


def test_the_ceiling():
    """A ceiling of 3 chunks on the churn stream: the call that passes it raises "label storage full", chunks in use
    stay within the ceiling, and every voxel either holds the unbounded map's pairs or has lost some to counted
    evictions (it holds as many pairs as its chain allows, never more than the map)."""
    T0, _ = E.cam_poses()
    sc = SL.scene_churn(T0)
    grids, G = _grids(sc, capacity_blocks=1 << 11, max_label_overflow_pairs=24)
    g = grids[0]
    raised = 0
    for op, kw in sc["steps"][:4]:
        try:
            SC.apply(g, "gpu", op, kw)
        except RuntimeError as e:
            assert "label storage full" in str(e)
            raised += 1
        SC.apply(G, "oracle", op, kw)
        s = g.label_storage()
        assert s["used"] <= s["max"] == 3
    assert raised > 0 and g.label_overflows() > 0
    K = max(8, G.max_pairs())
    d, r = sort_dump(g.dump_blocks(K)), G.dump(K)
    for k in ("keys", "count", "pos_sum", "col_sum"):
        assert np.array_equal(d[k], r[k]), k
    assert np.all(d["aux"] <= r["aux"])
    same = np.all((d["lab_obj"] == r["lab_obj"]) & (d["lab_cls"] == r["lab_cls"]), axis=-1) & (d["aux"] == r["aux"])
    lost = int((~same).sum())
    assert 0 < lost and int((r["aux"] - d["aux"]).sum()) <= g.label_overflows()
    g.close()


def test_ceiling_zero_is_the_grid_without_a_store():
    T0, _ = E.cam_poses()
    sc = SC.scene_random(T0)
    a = VoxelBlockSemanticProbabilisticGrid(SC.VS, 8, capacity_blocks=1 << 11)
    b = VoxelBlockSemanticProbabilisticGrid(SC.VS, 8, capacity_blocks=1 << 11, max_label_overflow_pairs=0)
    for t in (a, b):
        t.set_depth_threshold(sc["depth_threshold"])
        t.set_depth_decay_rate(sc["depth_decay_rate"])
    for step in SC.scene_eviction()["steps"] + sc["steps"]:
        for t in (a, b):
            SC.apply(t, "gpu", *step)
        x, y = sort_dump(a.dump_blocks()), sort_dump(b.dump_blocks())
        assert x["lab_obj"].shape[-1] == 8
        for k in x:
            assert np.array_equal(x[k], y[k]), k
        assert a.label_overflows() == b.label_overflows()
    assert b.label_storage() == dict(used=0, mapped=0, max=0, growths=0)
    assert a.label_overflows() > 0
    a.close()
    b.close()


def test_voting_grid_and_bad_ceilings_raise():
    with pytest.raises(RuntimeError):
        VoxelBlockSemanticGrid(SC.VS, 8, capacity_blocks=16, max_label_overflow_pairs=8)
    with pytest.raises(RuntimeError):
        VoxelBlockSemanticProbabilisticGrid(SC.VS, 8, capacity_blocks=16, max_label_overflow_pairs=1 << 40)
    g = VoxelBlockSemanticProbabilisticGrid(SC.VS, 8, capacity_blocks=16, max_label_overflow_pairs=9)
    assert g.label_storage()["max"] == 2
    g.close()


def test_semantic_plugin_with_a_label_store_equals_the_plugin_without():
    """kVolumetricIntegrationB200LabelOverflowPairs on a stream that never passes 8 pairs per voxel (the committed
    association frames): association, remap and integrate give the same grid with and without the store."""
    import os
    from types import SimpleNamespace
    from pyslam_b200 import synthetic as S
    from tests import plugin_standins as P
    from tests._util import GOLDEN
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    cfg = S.CONFIGS["T0"]
    cam = SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)
    kw = dict(kVolumetricIntegrationVoxelLength=float(g["voxel_size"]), kVolumetricIntegrationVoxelGridUseCarving=True,
              kVolumetricIntegrationB200CapacityBlocks=1024, use_semantic_probabilistic=True)
    Cls = P.standalone_semantic_integrator_class()
    plain = Cls(cam, P.DatasetEnvironmentType.INDOOR, None, "B200_SEMANTIC", **kw)
    store = Cls(cam, P.DatasetEnvironmentType.INDOOR, None, "B200_SEMANTIC",
                kVolumetricIntegrationB200LabelOverflowPairs=4096, **kw)
    assert store.volume.label_storage()["max"] == 512 and plain.volume.label_storage()["max"] == 0
    for i in range(int(g["n_frames"])):
        for integ in (plain, store):
            integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(
                id=i, pose=g[f"Tcw_{i}"], img=np.ascontiguousarray(g[f"color_{i}"][..., ::-1]), depth=g[f"depth_{i}"],
                semantic_img=g[f"class_image_{i}"], semantic_instances_img=g[f"instance_image_{i}"]))
            integ.step()
        assert plain.last_instance_map == store.last_instance_map
        a, b = sort_dump(plain.volume.dump_blocks()), sort_dump(store.volume.dump_blocks())
        assert a["aux"].max() <= 8
        for k in a:
            assert np.array_equal(a[k], b[k]), (i, k)
    assert store.volume.label_storage()["used"] == 0
    for integ in (plain, store):
        integ.quit()


def test_map_state_round_trip_continuation_and_ceiling(tmp_path):
    """save_state / load_state carry the overflow pairs: a 3-shard grid with chains saved and loaded into one grid and
    into 2 shards holds the same dump; labelled calls after the load continue as on the saved grid; a grid without
    overflow pairs writes the file of a grid without a store; a ceiling too small for the file's pairs raises
    ValueError and leaves the grid as it was."""
    kw = SC.stream(SL.many_pair_streams(40))
    more = SC.stream({k: [(o, c, 1.0) for o, c in SL.pairs(12, 5)] for k in SC.VOX})
    a = VoxelBlockSemanticProbabilisticGrid(SC.VS, 8, capacity_blocks=64)
    b = VoxelBlockSemanticProbabilisticGrid(SC.VS, 8, capacity_blocks=64, max_label_overflow_pairs=BIG)
    small = {k: v[:20] for k, v in kw.items()}
    for t, name in ((a, "a"), (b, "b")):
        t.integrate(**small)
        t.save_state(str(tmp_path / f"{name}.npz"))
    with np.load(str(tmp_path / "a.npz")) as x, np.load(str(tmp_path / "b.npz")) as y:
        assert sorted(x.files) == sorted(y.files) and all(np.array_equal(x[k], y[k]) for k in x.files)
    a.close()
    b.close()

    src = [VoxelBlockSemanticProbabilisticGrid(SC.VS, 8, capacity_blocks=64, shard_rank=r, shard_count=3,
                                               max_label_overflow_pairs=BIG) for r in range(3)]
    G = SL.UnboundedSemanticGrid(SC.VS)
    for t in src + [G]:
        t.integrate(**kw)
    paths = [str(tmp_path / f"s{r}.npz") for r in range(3)]
    for t, p in zip(src, paths):
        t.save_state(p)
    assert any("labels_count" in np.load(p).files for p in paths)
    one = VoxelBlockSemanticProbabilisticGrid(SC.VS, 8, capacity_blocks=64, max_label_overflow_pairs=BIG)
    two = [VoxelBlockSemanticProbabilisticGrid(SC.VS, 8, capacity_blocks=64, shard_rank=r, shard_count=2,
                                               max_label_overflow_pairs=BIG) for r in range(2)]
    for t in [one] + two:
        t.load_state(paths)
    _same_state([one], G, True, "loaded")
    _same_state(two, G, True, "loaded into 2 shards")
    assert one.label_storage()["used"] == sum(t.label_storage()["used"] for t in src)
    for t in src + [one] + two + [G]:   # continuation: new pairs and known ones, an edit, more pairs
        t.integrate(**more)
    _same_state([one], G, True, "continued")
    _same_state(src, G, True, "continued source")
    for t in [one, G]:
        SC.apply(t, "gpu" if t is one else "oracle", "remove_segment", dict(object_id=SL.pairs(40)[-1][0]))
        t.integrate(**kw)
    _same_state([one], G, True, "continued after an edit")

    tight = VoxelBlockSemanticProbabilisticGrid(SC.VS, 8, capacity_blocks=64, max_label_overflow_pairs=8)
    none = VoxelBlockSemanticProbabilisticGrid(SC.VS, 8, capacity_blocks=64)
    for t in (tight, none):
        t.integrate(**small)
        before = sort_dump(t.dump_blocks())
        with pytest.raises(ValueError):
            t.load_state(paths)
        after = sort_dump(t.dump_blocks())
        assert all(np.array_equal(before[k], after[k]) for k in before)
    for t in src + [one, tight, none] + two:
        t.close()


def test_association_releases_chains():
    """The association scene with every voxel first given 12 pairs (the original label stays the argmax): carving
    inside the association and the object ids it sets release real chains, then the labelled call builds them again."""
    T0, _ = E.cam_poses()
    sc = SC.scene_association(T0)
    first = sc["steps"][1][1]
    n = len(first["points"])
    reps = 12
    churn = dict(points=np.tile(first["points"], (reps, 1)), colors=np.tile(first["colors"], (reps, 1)),
                 class_ids=np.tile(first["class_ids"], reps),
                 instance_ids=(1000 + np.arange(reps * n) % (reps * n)).astype(np.int32))
    steps = sc["steps"][:2] + [("integrate", churn)] + sc["steps"][2:]
    grids, G = _grids(sc, initial_label_overflow_pairs=8)
    g = grids[0]
    used, drops = [], 0
    for i, (op, step) in enumerate(steps):
        before = g.label_storage()["used"]
        maps = SC.apply(g, "gpu", op, step)
        m = SC.apply(G, "oracle", op, step)
        if op == "assign":
            assert maps == m, i
            drops += g.label_storage()["used"] < before
        _same_state(grids, G, True, ("association", i, op))
        used.append(g.label_storage()["used"])
    assert max(used) > 0 and drops > 0
    g.close()
