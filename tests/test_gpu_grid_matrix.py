"""GPU: the grids' features in combination, at the block sides where they had not run together.

Bayesian grid with an overflow label store (`max_label_overflow_pairs`) at B = 1, 2, 16 and 8: the chain scene of
tests/_grid_matrix.py (chains in every 512-voxel slice of a B = 16 block and in every block of a B = 1 / 2 pool, each
edit that releases chains, the association), the many-pair scenes and the churn stream; on fixed grids, on grids that
grow their block pool and chunk storage from 4 blocks and one chunk, on 3 shards, through labelled RGBD frames with
association and remap, and through state files.  After every step the dump equals the unbounded label map laid out
at B, `export_labels()` holds each voxel's overflow pairs in slot order, the chunks in use equal the map's and no pair
was evicted.

Point-average grid with input-order sums at B = 1, 2, 16: growth, shards, state round trips, staged raw frames,
queries and edits after growth and the mode switched between calls, bit for bit against `oracle.numpy_grid`.

And the plugins with both parameters of each pair set."""

import copy
import os
from functools import lru_cache

import numpy as np
import pytest

import oracle
from pyslam_b200 import (BoundingBox3D, CameraFrustrum, VoxelBlockGrid, VoxelBlockSemanticProbabilisticGrid, _lib,
                         remap_instance_ids, sharding)
from pyslam_b200 import synthetic as S
from tests import _block_sizes as BS
from tests import _grid_matrix as M
from tests import _grid_order_scenes as O
from tests import _grid_prep_scenes as E
from tests import _semantic_scenes as SC
from tests._util import GOLDEN, sort_dump

pytestmark = pytest.mark.gpu
BIG = 1 << 20                                        # a label ceiling no scene reaches
SEM_CAP = {1: 1 << 16, 2: 1 << 14, 8: 1 << 11, 16: 1 << 9}
PT_CAP = {1: 1 << 21, 2: 1 << 18, 8: 1 << 15, 16: 1 << 12}


# ---- Bayesian grid with a label store ------------------------------------------------------------------------------

def _sem(B, sc=None, vs=SC.VS, **kw):
    kw.setdefault("capacity_blocks", SEM_CAP[B])
    kw.setdefault("max_label_overflow_pairs", BIG)
    g = VoxelBlockSemanticProbabilisticGrid(vs, B, **kw)
    if sc is not None:
        if "depth_threshold" in sc:
            g.set_depth_threshold(sc["depth_threshold"])
        if "depth_decay_rate" in sc:
            g.set_depth_decay_rate(sc["depth_decay_rate"])
    return g


def _grown(B, sc=None, **kw):
    return _sem(B, sc, capacity_blocks=M.GROW_BLOCKS, max_capacity_blocks=SEM_CAP[B], initial_label_overflow_pairs=8,
                **kw)


def _shards(B, sc, n):
    return [_sem(B, sc, shard_rank=r, shard_count=n) for r in range(n)]


def _check(grids, G, B, exact, where):
    """The grids (one map, maybe sharded) equal the oracle G laid out at B: dump, overflow pairs in slot order, chunks
    in use, no eviction.  Returns the merged dump."""
    K = max(8, G.max_pairs())
    d = sharding.merge_dumps([sort_dump(g.dump_blocks(K)) for g in grids])
    M.same_semantic(d, M.unbounded_dump(G, B, K), exact, where)
    got = M.sorted_labels([(g.export_blocks()["keys"], g.export_labels()) for g in grids])
    M.same_pairs(got, M.unbounded_overflow_pairs(G, B), exact, where)
    assert sum(g.label_storage()["used"] for g in grids) == M.used_chunks(G), where
    assert sum(g.label_overflows() for g in grids) == 0, where
    return d


def _same_grids(a, b, K, where):
    x, y = sort_dump(a.dump_blocks(K)), sort_dump(b.dump_blocks(K))
    for k in x:
        assert np.array_equal(x[k], y[k]), (where, k)
    la = M.sorted_labels([(a.export_blocks()["keys"], a.export_labels())])
    lb = M.sorted_labels([(b.export_blocks()["keys"], b.export_labels())])
    for k in la:
        assert np.array_equal(la[k], lb[k]), (where, k)


def _close(*grids):
    for g in grids:
        g.close()


@pytest.mark.parametrize("B", (1, 2, 8, 16))
@pytest.mark.parametrize("name", ["chains", "pairs9", "pairs17", "pairs40", "churn"])
def test_store_scenes_on_fixed_and_grown_grids(name, B):
    """Each scene on a fixed grid and on one grown from 4 blocks and one chunk: both equal the oracle after every
    step, and each other bit for bit (dump with every pair, overflow pairs)."""
    sc, snaps = M.played(name)
    exact = not sc.get("rtol")
    fixed, grown = _sem(B, sc), _grown(B, sc)
    for i, ((op, kw), (m, G)) in enumerate(zip(sc["steps"], snaps)):
        for g in (fixed, grown):
            got = SC.apply(g, "gpu", op, kw)
            if op == "assign":
                assert got == m, (name, B, i)
            _check([g], G, B, exact, (name, B, i, op, g is grown))
        _same_grids(fixed, grown, max(8, G.max_pairs()), (name, B, i))
    assert grown.capacity()[1] > 0 and grown.label_storage()["growths"] > 0
    assert max(M.used_chunks(G) for _, G in snaps) > 0
    _close(fixed, grown)


@pytest.mark.parametrize("B", (1, 2, 8, 16))
def test_grow_both_stores_in_one_call(B):
    """The first call overflows the 4-block pool and, in the same call, the one chunk (runs in blocks past the initial
    storage need chunks); then a call that only adds blocks, one that only adds pairs, and edits whose released chunks
    the next call takes again.  Equal to the oracle and to a fixed grid after every step."""
    sc, snaps = M.played("grow_both")
    grown, fixed = _grown(B), _sem(B)
    for i, ((op, kw), (_, G)) in enumerate(zip(sc["steps"], snaps)):
        cap0, lab0 = grown.capacity(), grown.label_storage()
        for g in (grown, fixed):
            SC.apply(g, "gpu", op, kw)
            _check([g], G, B, True, ("grow_both", B, i, op, g is grown))
        _same_grids(grown, fixed, max(8, G.max_pairs()), ("grow_both", B, i))
        cap1, lab1 = grown.capacity(), grown.label_storage()
        if i == 0:
            assert cap1[1] > cap0[1] and lab1["growths"] > lab0["growths"], (B, cap1, lab1)
        elif i == 1:    # blocks only
            assert lab1["growths"] == lab0["growths"]
            if len(M.blocks_at(G, B)) > cap0[0]:
                assert cap1[1] > cap0[1]
        elif i == 2:    # pairs only
            assert cap1 == cap0 and lab1["growths"] > lab0["growths"]
        elif op == "integrate":   # after an edit: the released chunks serve the call
            assert lab1["mapped"] == lab0["mapped"] and lab1["used"] > lab0["used"]
    _close(grown, fixed)


@pytest.mark.parametrize("B", (1, 16))
@pytest.mark.parametrize("name", ["chains_no_assign", "pairs40"])
def test_three_shards(name, B):
    sc, snaps = M.played(name)
    grids = _shards(B, sc, 3)
    for i, ((op, kw), (_, G)) in enumerate(zip(sc["steps"], snaps)):
        for g in grids:
            SC.apply(g, "gpu", op, kw)
        _check(grids, G, B, True, (name, B, i, op))
    for g in grids:
        assert np.all(sharding.owner_of(g.export_blocks()["keys"], 3) == g.shard_rank)
    _close(*grids)


@pytest.mark.parametrize("B", (1, 2, 16))
def test_labelled_rgbd_association_and_remap(B):
    """Staged frames (set_frame) with object ids that change every frame: association -> remap_instance_ids ->
    integrate_rgbd (the remapped image on odd frames, the raw ids on even ones), at 2^-3 m voxels (many pixels per
    voxel), against the unbounded map fed the numpy front end and the oracle's association."""
    scene = dict(depth_threshold=1.5, depth_decay_rate=0.5)
    g = _sem(B, scene, vs=0.125, initial_label_overflow_pairs=8)
    G = M.new_oracle(scene, vs=0.125)
    cls_img, obj_img = SC.rgbd_labels()
    rng = np.random.default_rng(4)
    frames = E.rgbd_frames(n=4) + E.rgbd_frames(seed=8, n=4)
    for i, (d, c, Twc) in enumerate(frames):
        inst = (obj_img + 1000 * i + 10 * rng.integers(0, 64, obj_img.shape)).astype(np.int32)
        Tcw = np.linalg.inv(Twc)
        fr = CameraFrustrum(*E.RGBD_K, d.shape[1], d.shape[0], Tcw, depth_max=10.0, depth_min=1e-2)
        f = g.set_frame(d, c, cls_img, inst)
        m = g.assign_object_ids_to_instance_ids(fr, f.class_image, f.instance_image, f.depth, 0.1, True, 0.5, 1)
        mo = G.assign_object_ids_to_instance_ids(E.RGBD_K, d.shape[1], d.shape[0], Tcw, 10.0, 1e-2, cls_img, inst, d,
                                                 0.1, True, 0.5, 1)
        assert m == mo, (B, i)
        if i % 2:
            obj, obj_o = g.remap_instance_ids(), remap_instance_ids(inst, mo)
            assert np.array_equal(obj.numpy(), obj_o), (B, i)
        else:
            obj, obj_o = f.instance_image, inst
        g.integrate_rgbd(f.depth, f.color, E.RGBD_K, Twc, class_image=f.class_image, object_image=obj, max_depth=1.9)
        p, col = E.rgbd_points(d, c, E.RGBD_K, Twc, 1.9)
        valid = (d > 0) & (d < 1.9)
        G.integrate(p, col, cls_img[valid], obj_o[valid], d[valid])
        _check([g], G, B, True, ("rgbd", B, i))
        assert g.get_next_object_id() == G.next_object_id
    assert G.max_pairs() > 8 and g.label_storage()["growths"] > 0
    g.close()


def test_state_files_with_chains_at_block_size_16(tmp_path):
    """A 3-shard B = 16 map with chains saved and loaded into one grid, into 2 shards and into a grid with 4 blocks of
    storage and one chunk (the upload grows both); the loads continue with edits and labelled calls equal to the
    oracle.  A B = 8 grid with a store refuses the files and keeps its map."""
    sc, snaps = M.played("chains_no_assign")
    B = 16
    src = _shards(B, sc, 3)
    for g in src:
        SC.apply(g, "gpu", *sc["steps"][0])
    G0 = snaps[0][1]
    _check(src, G0, B, True, "saved")
    paths = [str(tmp_path / f"s{r}.npz") for r in range(3)]
    for g, p in zip(src, paths):
        g.save_state(p)
    assert all("labels_count" in np.load(p).files for p in paths)
    one, two, grown = _sem(B, sc), _shards(B, sc, 2), _grown(B, sc)
    loaded = [[one], two, [grown]]
    for grids in loaded:
        for g in grids:
            g.load_state(paths)
        _check(grids, G0, B, True, ("loaded", len(grids)))
    assert grown.capacity()[1] > 0 and grown.label_storage()["growths"] > 0
    for i in range(1, 7):      # remove_segment, the call again, merge_segments, the call again, merge(-1), again
        op, kw = sc["steps"][i]
        G = snaps[i][1]
        for grids in loaded:
            for g in grids:
                SC.apply(g, "gpu", op, kw)
            _check(grids, G, B, True, ("continued", i, op, len(grids)))

    g8 = _sem(8, sc)
    SC.apply(g8, "gpu", *sc["steps"][0])
    before, lab = sort_dump(g8.dump_blocks()), g8.label_storage()
    with pytest.raises(ValueError):
        g8.load_state(paths)
    after = sort_dump(g8.dump_blocks())
    assert all(np.array_equal(before[k], after[k]) for k in before)
    assert g8.label_storage() == lab
    _close(g8, one, grown, *two, *src)


# ---- point-average grid with input-order sums ----------------------------------------------------------------------

PT_SIZES = (1, 2, 16)
PT_FIELDS = ("keys", "count", "pos_sum", "col_sum")


def _pt(B, vs=O.VS, grow=False, **kw):
    kw.setdefault("capacity_blocks", 4 if grow else PT_CAP[B])
    if grow:
        kw.setdefault("max_capacity_blocks", PT_CAP[B])
    return VoxelBlockGrid(vs, B, input_order_sums=True, **kw)


def _same_pt(grids, ref, where):
    d = sharding.merge_dumps([sort_dump(g.dump_blocks()) for g in grids])
    assert np.array_equal(d["hashes"], BS.block_key_hash(d["keys"])), where
    for k in PT_FIELDS:
        assert np.array_equal(d[k], ref[k]), (where, k)


def _feed(grids, frames):
    for d, c, Twc in frames:
        for g in grids:
            g.integrate_rgbd(d, c, O.frame_K(), Twc, max_depth=O.frame_max_depth())


@lru_cache(maxsize=None)
def _frames_oracle(n):
    return O.numpy_grid_of(O.frame_points()[:n])


@lru_cache(maxsize=None)
def _frames_dump(n, B):
    return BS.grid_dump(_frames_oracle(n), B)


@pytest.mark.parametrize("B", PT_SIZES)
def test_input_order_growth(B):
    """Grown from 4 blocks: the 12-call stress scene after every call, and the 10 C2 frames."""
    g = _pt(B, grow=True)
    G = oracle.numpy_grid(O.VS)
    for p, c in M.point_scenes()["stress_calls12"]:
        g.integrate(p, c)
        G.integrate(p, c)
        _same_pt([g], BS.grid_dump(G, B), ("stress", B))
    assert g.capacity()[1] > 0
    f = _pt(B, grow=True)
    _feed([f], O.frames())
    assert f.capacity()[1] > 0
    _same_pt([f], _frames_dump(O.N_FRAMES, B), ("frames", B))
    _close(g, f)


@pytest.mark.parametrize("B", PT_SIZES)
@pytest.mark.parametrize("world", [2, 3, 8])
def test_input_order_shards(world, B):
    grids = [_pt(B, shard_rank=r, shard_count=world) for r in range(world)]
    _feed(grids, O.frames())
    _same_pt(grids, _frames_dump(O.N_FRAMES, B), (world, B))
    for g in grids:
        d = sort_dump(g.dump_blocks())
        assert np.all(sharding.owner_of(d["keys"], world) == g.shard_rank)
    _close(*grids)


@pytest.mark.parametrize("B", PT_SIZES)
def test_input_order_state_round_trip(B, tmp_path):
    """Half the frames saved from a grown grid, loaded into one grid and into 3 shards, then the other half."""
    fr = O.frames()
    first = _pt(B, grow=True)
    _feed([first], fr[:5])
    path = str(tmp_path / "half.npz")
    first.save_state(path)
    one, three = _pt(B), [_pt(B, shard_rank=r, shard_count=3) for r in range(3)]
    for g in [one] + three:
        g.load_state(path)
    _same_pt([one], _frames_dump(5, B), ("loaded", B))
    _same_pt(three, _frames_dump(5, B), ("loaded 3", B))
    _feed([one] + three, fr[5:])
    _same_pt([one], _frames_dump(O.N_FRAMES, B), ("continued", B))
    _same_pt(three, _frames_dump(O.N_FRAMES, B), ("continued 3", B))
    _close(first, one, *three)


@pytest.mark.parametrize("B", PT_SIZES)
def test_input_order_staged_raw_frames(B):
    """Raw uint16 depth and BGR colour through set_frame with rectification and the shadow filter, on a grown grid:
    equal to numpy_grid fed the host preparation of the same frames."""
    pytest.importorskip("cv2")
    from tests.test_gpu_grid_frames import host_prepare, tum_maps
    mx, my = tum_maps(S.CONFIGS[O.FRAME_CFG])
    g = _pt(B, grow=True)
    g.set_rectification(mx, my, swap_rb=True)
    G = oracle.numpy_grid(O.VS)
    scale = 1.0 / 5000.0
    for d, c, Twc in O.frames()[:4]:
        raw = np.round(d * 5000.0).astype(np.uint16)
        bgr = np.ascontiguousarray(c[..., ::-1])
        f = g.set_frame(raw, bgr, depth_scale=scale, filter_shadow_points=True)
        g.integrate_rgbd(f.filtered_depth, f.color, O.frame_K(), Twc, max_depth=O.frame_max_depth())
        h = host_prepare(mx, my, raw, bgr, scale=scale, flt=True)
        G.integrate(*E.rgbd_points(h["filtered_depth"], h["color"], O.frame_K(), Twc, max_depth=O.frame_max_depth()))
    assert g.capacity()[1] > 0
    _same_pt([g], BS.grid_dump(G, B), ("staged", B))
    g.close()


def _rows(p, c):
    r = np.concatenate([p, c], 1)
    return r[np.lexsort(r.T[::-1])]


@pytest.mark.parametrize("B", PT_SIZES)
def test_input_order_queries_and_edits_after_growth(B):
    g = _pt(B, grow=True)
    _feed([g], O.frames())
    assert g.capacity()[1] > 0
    G = copy.deepcopy(_frames_oracle(O.N_FRAMES))
    d, c, Twc = O.frames()[3]
    cfg = S.CONFIGS[O.FRAME_CFG]
    Tcw = S.inv_T(Twc)
    K = (cfg.fx, cfg.fy, cfg.cx, cfg.cy)
    fr = CameraFrustrum(*K, cfg.width, cfg.height, Tcw, depth_max=3.0, depth_min=0.05)
    out = g.get_voxels_in_camera_frustrum(fr, min_count=2)
    assert len(out.points) > 1000
    assert np.array_equal(_rows(out.points, out.colors),
                          _rows(*G.get_voxels_in_frustum(fr._args()[0], cfg.width, cfg.height, Tcw, 3.0, 0.05, 2)))
    mean = (G.pos / G.count[:, None].astype(np.float32)).astype(np.float64)
    bb = np.concatenate([np.percentile(mean, 20, axis=0), np.percentile(mean, 70, axis=0)])
    ob = g.get_voxels_in_bb(BoundingBox3D(*bb), min_count=1)
    assert len(ob.points) > 100
    assert np.array_equal(_rows(ob.points, ob.colors), _rows(*G.get_voxels_in_bb(bb, 1)))
    g.remove_low_count_voxels(3)
    G.remove_low_count_voxels(3)
    _same_pt([g], BS.grid_dump(G, B), ("remove_low_count_voxels", B))
    carve_depth = np.where(d > 0, d * np.float32(1.25), d).astype(np.float32)
    g.carve(fr, carve_depth, depth_threshold=0.03)
    assert len(G.carve(fr._args()[0], cfg.width, cfg.height, Tcw, carve_depth, 0.03, 3.0, 0.05)) > 100
    _same_pt([g], BS.grid_dump(G, B), ("carve", B))
    g.close()


@pytest.mark.parametrize("B", PT_SIZES)
def test_mode_switched_between_calls(B):
    """Dyadic scenes, exact in any order: input-order sums switched on and off before every call, on a grown grid;
    numpy_grid after every call."""
    L = _lib.load()
    g = VoxelBlockGrid(E.VS_EXACT, B, capacity_blocks=4, max_capacity_blocks=PT_CAP[B])
    G = oracle.numpy_grid(E.VS_EXACT)
    on = 1
    for _, p, c in E.exact_batches():
        assert L.b2v_grid_set_input_order_sums(g._h, on) == _lib.B2V_OK
        g.integrate(p, c)
        G.integrate(p, c)
        _same_pt([g], BS.grid_dump(G, B), ("exact", B, on))
        on ^= 1
    for d, c, Twc in E.rgbd_frames():
        assert L.b2v_grid_set_input_order_sums(g._h, on) == _lib.B2V_OK
        g.integrate_rgbd(d, c, E.RGBD_K, Twc)
        G.integrate(*E.rgbd_points(d, c, E.RGBD_K, Twc))
        _same_pt([g], BS.grid_dump(G, B), ("rgbd", B, on))
        on ^= 1
    assert g.capacity()[1] > 0
    g.close()


# ---- plugins ---------------------------------------------------------------------------------------------------------

def _camera(cfg):
    from types import SimpleNamespace
    return SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)


def test_semantic_plugin_block_16_with_a_label_store_equals_block_8():
    """kVolumetricIntegrationBlockSize 16 with kVolumetricIntegrationB200LabelOverflowPairs: the same instance maps
    and, voxel for voxel, the same map as the B = 8 plugin with the same ceiling."""
    from tests import plugin_standins as P
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    cfg = S.CONFIGS["T0"]
    kw = dict(kVolumetricIntegrationVoxelLength=float(g["voxel_size"]), kVolumetricIntegrationVoxelGridUseCarving=True,
              kVolumetricIntegrationB200LabelOverflowPairs=4096, use_semantic_probabilistic=True)
    Cls = P.standalone_semantic_integrator_class()
    a = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_SEMANTIC", kVolumetricIntegrationBlockSize=16,
            **kw)
    b = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_SEMANTIC", kVolumetricIntegrationBlockSize=8, **kw)
    assert a.volume.get_block_size() == 16 and a.volume.label_storage()["max"] == b.volume.label_storage()["max"] == 512
    for i in range(int(g["n_frames"])):
        for integ in (a, b):
            integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(
                id=i, pose=g[f"Tcw_{i}"], img=np.ascontiguousarray(g[f"color_{i}"][..., ::-1]), depth=g[f"depth_{i}"],
                semantic_img=g[f"class_image_{i}"], semantic_instances_img=g[f"instance_image_{i}"]))
            integ.step()
        assert a.last_instance_map == b.last_instance_map
        K = max(8, int(a.volume.export_blocks()["counter"].max()))
        ka, va = BS.voxels(sort_dump(a.volume.dump_blocks(K)), 16, M.SEM_FIELDS)
        kb, vb = BS.voxels(sort_dump(b.volume.dump_blocks(K)), 8, M.SEM_FIELDS)
        sa, sb = va["count"] > 0, vb["count"] > 0
        assert sa.sum() > 100 and np.array_equal(ka[sa], kb[sb])
        for f in M.SEM_FIELDS:
            assert np.array_equal(va[f][sa], vb[f][sb]), (i, f)
        assert a.volume.label_storage()["used"] == b.volume.label_storage()["used"]
    for integ in (a, b):
        integ.quit()


def test_voxel_grid_plugin_block_2_with_input_order_sums_equals_numpy_grid():
    """kVolumetricIntegrationBlockSize 2 with kVolumetricIntegrationB200InputOrderSums: the plugin's map equals
    numpy_grid fed the plugin's host path (shadow filter, depth truncation 4 m), bit for bit."""
    from tests import plugin_standins as P
    cfg = S.CONFIGS["T0"]
    Cls = P.standalone_voxel_grid_integrator_class()
    integ = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_VOXEL_GRID",
                kVolumetricIntegrationVoxelLength=0.015, kVolumetricIntegrationBlockSize=2,
                kVolumetricIntegrationB200InputOrderSums=True)
    G = oracle.numpy_grid(0.015)
    for i in range(4):
        d, c, T = S.render_frame(cfg, i)
        integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(
            id=i, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=d))
        integ.step()
        dd = oracle.numpy_shadow_filter(d, 2, 2, -1.0)[0]
        G.integrate(*E.rgbd_points(dd, c, (cfg.fx, cfg.fy, cfg.cx, cfg.cy), np.linalg.inv(T), max_depth=4.0))
    assert integ.volume.get_block_size() == 2 and integ.volume.input_order_sums
    assert len(G.keys) > 1000
    _same_pt([integ.volume], BS.grid_dump(G, 2), "plugin")
    integ.quit()
