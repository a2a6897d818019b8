"""GPU: map state files of the TSDF volume and the point-average and semantic grids (`save_state` / `load_state`,
DESIGN.md §7 "Map state").

A restore gives back the same map bit for bit (TSDF and point grid: dumps sorted by key; semantic grids: the raw export
with the label slots in the kernel's own order); integrating more frames after a load equals integrating without the
break; files load into any shard layout; a growable object grows while it loads, a fixed one that is too small refuses;
malformed or mismatched files raise ValueError and leave the map as it was; the plugins save the state on SAVE and
restore it on LOAD."""

import functools
import os
from types import SimpleNamespace

import numpy as np
import pytest

import oracle
from pyslam_b200 import (B200TsdfVolume, CameraFrustrum, VoxelBlockGrid, VoxelBlockSemanticGrid,
                         VoxelBlockSemanticProbabilisticGrid, sharding)
from pyslam_b200 import synthetic as S
from pyslam_b200.volume import _as_K4
from tests import _grid_prep_scenes as E
from tests import _semantic_scenes as SS
from tests import plugin_standins as P
from tests._util import GOLDEN, sort_dump
from tests.test_gpu_grid_growth import _rgbd_frames

pytestmark = pytest.mark.gpu
SEM = {"vote": VoxelBlockSemanticGrid, "prob": VoxelBlockSemanticProbabilisticGrid}
ASSOC = dict(depth_threshold=0.08, do_carving=True, min_vote_ratio=0.5, min_votes=3)


# ---- helpers --------------------------------------------------------------------------------------------------------

def _state(m):
    """The map's blocks sorted by key: the dump of a TSDF volume / point grid, the raw export of a semantic grid."""
    if isinstance(m, VoxelBlockSemanticGrid):
        return sort_dump(m.export_blocks())
    d = m.dump_blocks()
    d.pop("hashes")
    return sort_dump(d)


def _same(a, b):
    sa, sb = _state(a), _state(b)
    assert sa.keys() == sb.keys()
    for k in sa:
        assert sa[k].dtype == sb[k].dtype and np.array_equal(sa[k], sb[k], equal_nan=True), k
    if isinstance(a, VoxelBlockSemanticGrid):
        assert a.get_next_object_id() == b.get_next_object_id()


def _roundtrip(m, make, tmp_path, name="m.npz"):
    """save m, load into make() (a fresh object), and check the two equal; returns the loaded object."""
    path = str(tmp_path / name)
    m.save_state(path)
    n = make()
    n.load_state(path)
    _same(m, n)
    return n


@functools.lru_cache(maxsize=None)
def _tsdf_frames(tag, n):
    cfg = S.CONFIGS[tag]
    return cfg, [S.render_frame(cfg, i * cfg.n_frames // n) for i in range(n)]


def _tsdf(cfg, ures=16, **kw):
    kw.setdefault("capacity_blocks", 1 << 17)
    return B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, volume_unit_resolution=ures, **kw)


def _feed(vol, cfg, frames):
    for d, c, T in frames:
        vol.integrate(d, c, cfg.K, T)
    vol.synchronize()


def _rows(p, c):
    a = np.concatenate([np.asarray(p), np.asarray(c)], 1)
    return a[np.lexsort(a.T[::-1])]


# ---- TSDF ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("ures", [16, 8])
@pytest.mark.parametrize("tag,n", [("T0", 24), ("C1", 12), ("C2", 30)])
def test_tsdf_roundtrip_and_continuation(tag, n, ures, tmp_path):
    cfg, frames = _tsdf_frames(tag, n)
    a, b = frames[: n // 2], frames[n // 2:]
    first = _tsdf(cfg, ures)
    _feed(first, cfg, a)
    loaded = _roundtrip(first, lambda: _tsdf(cfg, ures), tmp_path)
    _feed(loaded, cfg, b)
    whole = _tsdf(cfg, ures)
    _feed(whole, cfg, frames)
    _same(loaded, whole)
    ma, mb = loaded.extract_mesh(), whole.extract_mesh()
    ca = oracle.canonical_mesh(ma.vertices, ma.vertex_colors, ma.edge_ids, ma.triangles)
    cb = oracle.canonical_mesh(mb.vertices, mb.vertex_colors, mb.edge_ids, mb.triangles)
    assert len(ma.triangles) > 0
    for k in cb:
        assert np.array_equal(ca[k], cb[k]), k
    pa, pb = loaded.extract_point_cloud(), whole.extract_point_cloud()
    assert len(pa.points) == len(pb.points) > 0
    assert np.array_equal(_rows(pa.points, pa.colors), _rows(pb.points, pb.colors))


def _tsdf_sharded(cfg, world, frames):
    shards = [_tsdf(cfg, shard_rank=r, shard_count=world) for r in range(world)]
    for v in shards:
        _feed(v, cfg, frames)
    return shards


def test_tsdf_resharding_and_growth(tmp_path):
    cfg, frames = _tsdf_frames("C1", 12)
    single = _tsdf(cfg)
    _feed(single, cfg, frames)
    single.save_state(str(tmp_path / "one.npz"))
    direct = {w: _tsdf_sharded(cfg, w, frames) for w in (2, 3, 4)}
    for w in (2, 3, 4):   # 1 -> N
        for r in range(w):
            v = _tsdf(cfg, shard_rank=r, shard_count=w)
            v.load_state(str(tmp_path / "one.npz"))
            _same(v, direct[w][r])
    files = []
    for r, v in enumerate(direct[3]):   # 3 -> 1 and 3 -> 2
        files.append(str(tmp_path / f"shard{r}.npz"))
        v.save_state(files[-1])
    v = _tsdf(cfg)
    v.load_state(files[::-1])
    _same(v, single)
    for r in range(2):
        v = _tsdf(cfg, shard_rank=r, shard_count=2)
        v.load_state(files)
        _same(v, direct[2][r])
    # growth: a growable volume starting at 16 blocks maps storage while it loads
    g = _tsdf(cfg, capacity_blocks=16, max_capacity_blocks=1 << 17)
    g.load_state(str(tmp_path / "one.npz"))
    assert g.capacity()[1] > 0
    _same(g, single)
    # a fixed volume that is too small refuses before it touches its map
    small = _tsdf(cfg, capacity_blocks=single.num_blocks() - 1)
    _feed(small, cfg, frames[:1])
    before = _state(small)
    with pytest.raises(ValueError):
        small.load_state(str(tmp_path / "one.npz"))
    after = _state(small)
    assert all(np.array_equal(before[k], after[k]) for k in before)


# ---- point-average grid ----------------------------------------------------------------------------------------------

def _point_grid(**kw):
    kw.setdefault("capacity_blocks", 1 << 12)
    return VoxelBlockGrid(E.VS_EXACT, 8, **kw)


def test_point_grid_roundtrip_continuation_resharding_and_growth(tmp_path):
    batches = E.exact_batches()
    a, b = batches[:3], batches[3:]
    first = _point_grid()
    for _, p, c in a:
        first.integrate(p, c)
    loaded = _roundtrip(first, _point_grid, tmp_path)
    for _, p, c in b:
        loaded.integrate(p, c)
    whole = _point_grid()
    for _, p, c in batches:
        whole.integrate(p, c)
    _same(loaded, whole)
    whole.save_state(str(tmp_path / "whole.npz"))
    for w in (2, 3, 4):
        for r in range(w):
            direct = _point_grid(shard_rank=r, shard_count=w)
            for _, p, c in batches:
                direct.integrate(p, c)
            v = _point_grid(shard_rank=r, shard_count=w)
            v.load_state(str(tmp_path / "whole.npz"))
            _same(v, direct)
            if w == 3:
                direct.save_state(str(tmp_path / f"shard{r}.npz"))
    files = [str(tmp_path / f"shard{r}.npz") for r in range(3)]
    v = _point_grid()
    v.load_state(files)
    _same(v, whole)
    for r in range(2):
        direct = _point_grid(shard_rank=r, shard_count=2)
        for _, p, c in batches:
            direct.integrate(p, c)
        v = _point_grid(shard_rank=r, shard_count=2)
        v.load_state(files)
        _same(v, direct)
    g = _point_grid(capacity_blocks=4, max_capacity_blocks=1 << 12)
    g.load_state(str(tmp_path / "whole.npz"))
    assert g.capacity()[1] > 0
    _same(g, whole)
    small = _point_grid(capacity_blocks=whole.num_blocks() - 1)
    small.integrate(*batches[0][1:])
    before = _state(small)
    with pytest.raises(ValueError):
        small.load_state(str(tmp_path / "whole.npz"))
    after = _state(small)
    assert all(np.array_equal(before[k], after[k]) for k in before)


# ---- semantic grids --------------------------------------------------------------------------------------------------

def _golden_stream(tag):
    g = np.load(os.path.join(GOLDEN, "semantic_T0.npz"))
    steps = [(g[f"{tag}_points_{i}"], g[f"{tag}_colors_{i}"], g[f"{tag}_cls_{i}"], g[f"{tag}_inst_{i}"],
              g[f"{tag}_depths_{i}"]) for i in range(int(g["n_frames"]))]
    return float(g["voxel_size"]), float(g[f"{tag}_depth_threshold"]), float(g[f"{tag}_depth_decay_rate"]), steps


@pytest.mark.parametrize("tag", ["vote", "prob"])
def test_semantic_golden_roundtrip_continuation_resharding_and_growth(tag, tmp_path):
    vs, thr, rate, steps = _golden_stream(tag)

    def make(**kw):
        kw.setdefault("capacity_blocks", 1024)
        return SEM[tag](vs, 8, **kw)

    def feed(grid, part):
        grid.set_depth_threshold(thr)
        grid.set_depth_decay_rate(rate)
        for s in part:
            grid.integrate(*s)

    h = len(steps) // 2
    first = make()
    feed(first, steps[:h])
    first.set_next_object_id(17)
    loaded = _roundtrip(first, make, tmp_path)
    assert loaded.get_next_object_id() == 17
    assert loaded.label_overflows() == 0
    for s in steps[h:]:   # the settings come back with the state
        loaded.integrate(*s)
    whole = make()
    feed(whole, steps)
    whole.set_next_object_id(17)
    _same(loaded, whole)
    whole.save_state(str(tmp_path / "whole.npz"))
    for w in (2, 3, 4):
        for r in range(w):
            direct = make(shard_rank=r, shard_count=w)
            feed(direct, steps)
            direct.set_next_object_id(17)
            v = make(shard_rank=r, shard_count=w)
            v.load_state(str(tmp_path / "whole.npz"))
            _same(v, direct)
            if w == 3:
                direct.save_state(str(tmp_path / f"shard{r}.npz"))
    files = [str(tmp_path / f"shard{r}.npz") for r in range(3)]
    v = make()
    v.load_state(files)
    _same(v, whole)
    for r in range(2):
        direct = make(shard_rank=r, shard_count=2)
        feed(direct, steps)
        direct.set_next_object_id(17)
        v = make(shard_rank=r, shard_count=2)
        v.load_state(files)
        _same(v, direct)
    g = make(capacity_blocks=4, max_capacity_blocks=1024)
    g.load_state(str(tmp_path / "whole.npz"))
    assert g.capacity()[1] > 0
    _same(g, whole)
    small = make(capacity_blocks=whole.num_blocks() - 1)
    small.integrate(*steps[0])
    before = _state(small)
    with pytest.raises(ValueError):
        small.load_state(str(tmp_path / "whole.npz"))
    after = _state(small)
    assert all(np.array_equal(before[k], after[k], equal_nan=True) for k in before)


def _run_steps(grid, steps):
    for op, kw in steps:
        assert op == "integrate"
        grid.integrate(kw["points"], kw["colors"], kw["class_ids"], kw["instance_ids"], kw["depths"])


def _reversed_full_voxel():
    """One voxel whose 8 label slots hold, each seen once, pairs inserted in DESCENDING (object, class) order (the
    argmax is slot 0), then a ninth pair: every candidate ties and the first non-argmax slot in the kernel's order
    (slot 1) is evicted.  A restore from the dump's (object, class) order would evict the smallest pair instead."""
    pairs = SS._pairs(9)
    a = SS.stream({SS.VOX[0]: [(o, c, 1.0) for o, c in pairs[:8][::-1]]})
    b = SS.stream({SS.VOX[0]: [(*pairs[8], 1.0)]})
    return dict(steps=[("integrate", a), ("integrate", b)], depth_threshold=1.5, depth_decay_rate=1.0)


@pytest.mark.parametrize("scene", ["eviction", "reversed_slots", "argmax_ties"])
def test_semantic_slots_survive_the_restore(scene, tmp_path):
    """Continuation through a save / load where the second half evicts slots or breaks argmax ties: equal to the
    unbroken run with the raw slots, and not equal when the restore is fed the (object, class)-sorted dump."""
    sc = {"eviction": lambda: SS.scene_eviction(split_at_first_eviction=True), "reversed_slots": _reversed_full_voxel,
          "argmax_ties": lambda: dict(steps=SS.split(SS.scene_argmax_ties()["steps"][0][1], 5))}[scene]()
    steps = sc["steps"]
    assert len(steps) == 2

    def make():
        g = VoxelBlockSemanticProbabilisticGrid(SS.VS, 8, capacity_blocks=64)
        if "depth_threshold" in sc:
            g.set_depth_threshold(sc["depth_threshold"])
            g.set_depth_decay_rate(sc["depth_decay_rate"])
        return g

    first = make()
    _run_steps(first, steps[:1])
    loaded = _roundtrip(first, make, tmp_path)
    _run_steps(loaded, steps[1:])
    whole = make()
    _run_steps(whole, steps)
    _same(loaded, whole)
    if scene == "reversed_slots":
        assert whole.label_overflows() == 1
        # the sorted dump as the restore's label slots: the continuation diverges
        raw, dump = first.export_blocks(), first.dump_blocks(8)
        assert np.array_equal(raw["keys"], dump["keys"])
        wrong = dict(raw, lab_obj=dump["lab_obj"], lab_cls=dump["lab_cls"], lab_logp=dump["lab_logp"])
        assert not np.array_equal(wrong["lab_obj"], raw["lab_obj"])
        bad = make()
        bad.clear()
        bad._upload_state(wrong)
        _run_steps(bad, steps[1:])
        sb, sw = _state(bad), _state(whole)
        assert not all(np.array_equal(sb[k], sw[k]) for k in ("lab_obj", "lab_cls", "lab_logp"))


def _c3_frames(n):
    cfg = S.CONFIGS["C3"]
    out = []
    for i in range(n):
        d, c, Tcw = S.render_frame(cfg, 12 * i)
        cls = S.render_class_ids(cfg, 12 * i).astype(np.int32)
        inst = np.where(cls % 3 == 0, -1, cls * 7 + (np.arange(cls.shape[1])[None, :] // 400) + i % 2)
        inst[:40] = 0
        out.append((d, c, Tcw, cls, inst.astype(np.int32)))
    return cfg, out


@pytest.mark.parametrize("tag", ["vote", "prob"])
def test_semantic_c3_association_continuation(tag, tmp_path):
    """8 C3 frames through association -> remap_instance_ids -> integrate_rgbd, saved after 4: the loaded grid gives the
    same association maps for the last 4 frames and ends equal to the unbroken grid; a 2-shard load runs one sharded
    association round that equals the unsharded one."""
    cfg, frames = _c3_frames(8)
    K4 = _as_K4(cfg.K)

    def make(**kw):
        g = SEM[tag](0.015, 8, capacity_blocks=1 << 10, max_capacity_blocks=1 << 17, **kw)
        g.set_depth_threshold(1.5)
        return g

    def frame(g, f):
        d, c, Tcw, cls, inst = f
        fr = CameraFrustrum(*K4, d.shape[1], d.shape[0], Tcw, depth_max=cfg.depth_trunc, depth_min=1e-2)
        st = g.set_frame(d, c, cls, inst)
        m = g.assign_object_ids_to_instance_ids(fr, st.class_image, st.instance_image, st.depth, **ASSOC)
        g.integrate_rgbd(st.depth, st.color, cfg.K, S.inv_T(Tcw), st.class_image, g.remap_instance_ids(),
                         max_depth=cfg.depth_trunc)
        return m

    whole, first = make(), make()
    maps = [frame(whole, f) for f in frames]
    assert [frame(first, f) for f in frames[:4]] == maps[:4]
    path = str(tmp_path / "c3.npz")
    first.save_state(path)
    loaded = make()
    loaded.load_state(path)
    _same(first, loaded)
    with pytest.raises(RuntimeError):   # the instance map is not part of the state
        loaded.remap_instance_ids()
    assert [frame(loaded, f) for f in frames[4:]] == maps[4:]
    _same(loaded, whole)
    assert loaded.get_next_object_id() > 2 and any(o > 0 for m in maps[4:] for o in m.values())
    # one sharded association round on 2 shards loaded from the unsharded file
    shards = [make(shard_rank=r, shard_count=2) for r in range(2)]
    for s in shards:
        s.load_state(path)
    d, c, Tcw, cls, inst = frames[4]
    fr = CameraFrustrum(*K4, d.shape[1], d.shape[0], Tcw, depth_max=cfg.depth_trunc, depth_min=1e-2)
    votes = [sharding.association_votes(s, fr, cls, inst, d, ASSOC["depth_threshold"], ASSOC["do_carving"])
             for s in shards]
    for s in shards:
        assert sharding.resolve_association(s, votes, cls, inst, min_vote_ratio=0.5, min_votes=3) == maps[4]
    assert shards[0].get_next_object_id() == shards[1].get_next_object_id() >= first.get_next_object_id()


# ---- empty maps and rejection ----------------------------------------------------------------------------------------

def _makers():
    cfg = S.CONFIGS["T0"]
    return {"tsdf": (lambda: _tsdf(cfg, capacity_blocks=4096), lambda m: _feed(m, cfg, _tsdf_frames("T0", 24)[1][:3])),
            "grid": (_point_grid, lambda m: m.integrate(*E.exact_batches()[3][1:])),
            "vote": (lambda: VoxelBlockSemanticGrid(SS.VS, 8, capacity_blocks=64),
                     lambda m: _run_steps(m, SS.scene_eviction()["steps"])),
            "prob": (lambda: VoxelBlockSemanticProbabilisticGrid(SS.VS, 8, capacity_blocks=64),
                     lambda m: _run_steps(m, SS.scene_eviction()["steps"]))}


@pytest.mark.parametrize("kind", ["tsdf", "grid", "vote", "prob"])
def test_empty_map_roundtrip(kind, tmp_path):
    make, fill = _makers()[kind]
    empty = make()
    path = str(tmp_path / "empty.npz")
    empty.save_state(path)
    m = make()
    fill(m)
    assert m.num_blocks() > 0
    m.load_state(path)
    assert m.num_blocks() == 0
    _same(m, empty)


def _mutate(src, dst, **changes):
    """Copy a state file, replacing (value) or dropping (None) fields."""
    with np.load(src) as z:
        d = {k: z[k] for k in z.files}
    for k, v in changes.items():
        if v is None:
            d.pop(k)
        else:
            d[k] = v
    with open(dst, "wb") as f:
        np.savez(f, **d)
    return dst


@pytest.mark.parametrize("kind", ["tsdf", "grid", "vote", "prob"])
def test_rejected_files_leave_the_map_unchanged(kind, tmp_path):
    makers = _makers()
    make, fill = makers[kind]
    src = make()
    fill(src)
    good = str(tmp_path / "good.npz")
    src.save_state(good)
    with np.load(good) as z:
        keys, first_array = z["blocks_keys"], [k for k in z.files if k.startswith("blocks_") and k != "blocks_keys"][0]
        arr = z[first_array]
    other_kind = {"tsdf": "grid", "grid": "tsdf", "vote": "prob", "prob": "vote"}[kind]
    other = makers[other_kind][0]()
    makers[other_kind][1](other)
    other_path = str(tmp_path / "other.npz")
    other.save_state(other_path)
    bad = [
        _mutate(good, tmp_path / "version.npz", format_version=np.int32(2)),
        _mutate(good, tmp_path / "kind.npz", kind=np.str_("mesh")),
        other_path,
        _mutate(good, tmp_path / "voxel.npz", voxel_size=np.asarray(np.asarray(
            np.load(good)["voxel_size"]) * 2)),
        _mutate(good, tmp_path / "missing.npz", **{first_array: None}),
        _mutate(good, tmp_path / "dtype.npz", **{first_array: arr.astype(np.float16 if arr.dtype.kind == "f"
                                                                             else np.int64)}),
        _mutate(good, tmp_path / "shape.npz", blocks_keys=keys[:, :2].copy()),
        _mutate(good, tmp_path / "dup.npz", blocks_keys=np.concatenate([keys[:1], keys[:-1]])),
        [good, good],
        str(tmp_path / "does_not_exist.npz"),
    ]
    if kind != "tsdf":
        with np.load(good) as z:
            cnt = z["blocks_count"].copy()
        cnt[0, 0] = -1
        bad.append(_mutate(good, tmp_path / "count.npz", blocks_count=cnt))
    if kind == "prob":
        with np.load(good) as z:
            ctr = z["blocks_counter"].copy()
        ctr[0, 0] = 9
        bad.append(_mutate(good, tmp_path / "counter.npz", blocks_counter=ctr))
    m = make()
    fill(m)
    m.save_state(str(tmp_path / "held.npz"))
    before = _state(m)
    for b in bad:
        with pytest.raises(ValueError):
            m.load_state(b if isinstance(b, list) else str(b))
        after = _state(m)
        assert all(np.array_equal(before[k], after[k], equal_nan=True) for k in before), b
    m.load_state(good)   # the map still loads a good file
    _same(m, src)


# ---- plugins ---------------------------------------------------------------------------------------------------------

def _camera(cfg):
    return SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)


def _last_output(integ):
    integ.add_update_output_task()
    integ.step()
    out = None
    while True:
        o = integ.pop_output()
        if o is None:
            return out
        out = o


def _same_output(a, b):
    if a.mesh is not None:   # the mesh in canonical form: vertex rows and triangles (as vertex positions) sorted
        va, vb = np.asarray(a.mesh.vertices), np.asarray(b.mesh.vertices)
        assert len(va) == len(vb) > 0 and len(a.mesh.triangles) == len(b.mesh.triangles)
        assert np.array_equal(_rows(va, a.mesh.vertex_colors), _rows(vb, b.mesh.vertex_colors))
        fa, fb = va[np.asarray(a.mesh.triangles)].reshape(-1, 9), vb[np.asarray(b.mesh.triangles)].reshape(-1, 9)
        assert np.array_equal(fa[np.lexsort(fa.T[::-1])], fb[np.lexsort(fb.T[::-1])])
    if a.point_cloud is not None:
        assert len(a.point_cloud.points) == len(b.point_cloud.points) > 0
        assert np.array_equal(_rows(a.point_cloud.points, a.point_cloud.colors),
                              _rows(b.point_cloud.points, b.point_cloud.colors))
    if a.objects is not None:
        oa = sorted((o.object_id, o.class_id, _rows(o.points, o.colors).tobytes()) for o in a.objects.object_list)
        ob = sorted((o.object_id, o.class_id, _rows(o.points, o.colors).tobytes()) for o in b.objects.object_list)
        assert len(oa) > 0 and oa == ob


def _plugin_cases():
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    sem_kw = dict(kVolumetricIntegrationVoxelLength=float(g["voxel_size"]), kVolumetricIntegrationVoxelGridUseCarving=True,
                  kVolumetricIntegrationVoxelGridShadowPointsFilter=False,
                  kVolumetricIntegrationVoxelGridCarvingDepthThreshold=0.08, kVolumetricIntegrationB200CapacityBlocks=1024,
                  use_semantic_probabilistic=True)
    sem_frames = [P.VolumetricIntegrationKeyframeData(
        id=i, pose=g[f"Tcw_{i}"], img=np.ascontiguousarray(g[f"color_{i}"][..., ::-1]), depth=g[f"depth_{i}"],
        semantic_img=g[f"class_image_{i}"], semantic_instances_img=g[f"instance_image_{i}"])
        for i in range(int(g["n_frames"]))]
    cfg = S.CONFIGS["T0"]
    frames = [P.VolumetricIntegrationKeyframeData(id=i, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=d)
              for i, (d, c, T) in enumerate(S.render_frame(cfg, i) for i in range(8))]
    # the point grid's float sums add in atomic order: frames whose sums are exact in any order
    exact, (fx, fy, cx, cy) = _rgbd_frames(n=6)
    exact_cam = SimpleNamespace(fx=fx, fy=fy, cx=cx, cy=cy, width=exact[0][0].shape[1], height=exact[0][0].shape[0],
                                D=None)
    exact_frames = [P.VolumetricIntegrationKeyframeData(id=i, pose=np.linalg.inv(Twc), img=np.ascontiguousarray(c[..., ::-1]),
                                                        depth=d) for i, (d, c, Twc) in enumerate(exact)]
    return {"tsdf": (P.standalone_integrator_class, cfg, dict(kVolumetricIntegrationB200CapacityBlocks=4096), frames),
            "voxel_grid": (P.standalone_voxel_grid_integrator_class, exact_cam,
                           dict(kVolumetricIntegrationVoxelLength=E.VS_EXACT,
                                kVolumetricIntegrationVoxelGridMinCount=1,
                                kVolumetricIntegrationB200CapacityBlocks=1 << 14), exact_frames),
            "semantic": (P.standalone_semantic_integrator_class, cfg, sem_kw, sem_frames)}


@pytest.mark.parametrize("case", ["tsdf", "voxel_grid", "semantic"])
def test_plugin_save_and_load(case, tmp_path):
    make_cls, cfg, kw, frames = _plugin_cases()[case]
    Cls = make_cls()
    h = len(frames) // 2

    def new(**extra):
        return Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200", **kw, **extra)

    one = new(kVolumetricIntegrationB200SaveMapState=True)
    for kd in frames[:h]:
        one.add_keyframe_data(kd)
    one.run_pending()
    one.save(str(tmp_path))
    one.run_pending()
    assert one.save_request_completed.value == 1
    assert os.path.exists(tmp_path / "dense_map.ply") and os.path.exists(tmp_path / "dense_map.state.npz")
    two = new()
    two.load(str(tmp_path / "missing"))   # a failed LOAD: flag stays 0, the loop keeps running
    two.run_pending()
    assert two.load_request_completed.value == 0 and two.is_running.value == 1
    two.load(str(tmp_path))
    two.run_pending()
    assert two.load_request_completed.value == 1
    _same_output(_last_output(one), _last_output(two))
    for kd in frames[h:]:
        one.add_keyframe_data(kd)
        two.add_keyframe_data(kd)
    one.run_pending()
    two.run_pending()
    _same_output(_last_output(one), _last_output(two))
    # with the parameter off SAVE writes the .ply alone
    off = tmp_path / "off"
    off.mkdir()
    two.save(str(off))
    two.run_pending()
    assert two.save_request_completed.value == 1
    assert os.path.exists(off / "dense_map.ply") and not os.path.exists(off / "dense_map.state.npz")
    one.quit()
    two.quit()
