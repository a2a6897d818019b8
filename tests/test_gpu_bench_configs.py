"""GPU: the TSDF kernels at the bench's other configurations, C3 (Replica shape, 1200x680, 5 mm), C4 (ScanNet shape,
4 mm) and C5 (KITTI shape, 1241x376, 10 cm, the street out to z = 1973 m), bit for bit.

- Bench scale: the 300 frames bench.py integrates, in fused groups of 32 (the bench's group size) and un-fused, two
  passes (every observed voxel at weight >= 2): keys, hashes and all five planes equal the CPU twin's; the mesh
  (edges, triangles, float64 vertices and colours) equals the twin's, the point cloud oracle.numpy_point_cloud's.
- The far end of the street (16 consecutive C5 frames, z ~ 1975 m) and 16 consecutive C4 frames, as one fused group
  and frame by frame, against the Open3D-order restatement: touched blocks, keys, tsdf and weights exact, colour
  within 1e-3, mesh topology and float64 vertices exact; the float64-colour volume's voxel and mesh colours exact.
- C5 in 8 hash shards (power-of-two mask) and 3 (64-bit modulo) on one GPU: the union of the shards and the face-halo
  mesh and point cloud equal the unsharded volume's.
- C4's raw-depth leg (uint16 at 5000 units per metre, depth_scale float32(1/5000)) through FrameIngest.
- C5 in a volume that grows from 1024 blocks.

tests/test_bench_configs_cpu.py ties the twin to the Open3D-order restatement on the same far and consecutive runs."""

import time

import numpy as np
import pytest
import torch

from pyslam_b200 import B200TsdfVolume, sharding
from pyslam_b200.sharding import FrameIngest
from tests import _bench_configs as B
from tests import _halo_oracle as H
from tests._util import sort_dump, sorted_keys
from tests.test_gpu_tsdf_edges import _check_points

pytestmark = pytest.mark.gpu

GROUP = 32
# what the bench-scale runs reach (two passes over the 300 bench frames): at least these many blocks, at least this
# maximum weight (the exact values are printed)
REACH = {"C3": (110_000, 128), "C4": (140_000, 90), "C5": (235_000, 4)}


def _vol(cfg, cap, **kw):
    return B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=cap, **kw)


def _capacity(n_blocks):
    """a power of two with at least 10 % headroom"""
    return 1 << int(np.ceil(np.log2(n_blocks * 1.1)))


def _same_as(dump, ref):
    """a dump equals a key-sorted reference dump in keys, hashes and all five planes, bit for bit"""
    a = sort_dump(dump)
    assert np.array_equal(a["keys"], ref["keys"])
    assert np.array_equal(a["hashes"], ref["hashes"])
    assert np.array_equal(a["vox"].view(np.uint32), ref["vox"].view(np.uint32))


_refs = {}


def _reference(name):
    """The CPU twin after PASSES passes over the bench frames: key-sorted dump and canonical mesh.  One config is kept
    at a time besides C5, which the shard and growth tests reuse."""
    if name not in _refs:
        for k in [k for k in _refs if k != "C5"]:
            del _refs[k]
            B.release_frames(k)
        cfg, D, C, T = B.bench_frames(name)
        t0 = time.perf_counter()
        tw = B.twin(cfg, D, C, T, B.PASSES)
        dump = sort_dump(tw.dump_blocks())
        mesh = B.canon(tw.extract_mesh())
        del tw
        w = dump["vox"][:, 1]
        _refs[name] = dict(cfg=cfg, D=D, C=C, T=T, dump=dump, mesh=mesh, cap=_capacity(len(dump["keys"])))
        print(f"\n[{name} twin] {B.PASSES} x {len(D)} frames in {time.perf_counter() - t0:.1f} s on {B.NT} threads: "
              f"blocks {len(dump['keys'])}, observed voxels {int((w > 0).sum())}, max weight {w.max():.0f}, "
              f"vertices {len(mesh['vertices'])}, triangles {len(mesh['triangles'])}")
    return _refs[name]


@pytest.fixture(scope="module", autouse=True)
def _release_host_memory():
    """the references and bench frames hold several GB of host memory: drop them when the module ends"""
    yield
    _refs.clear()
    B.release_frames()


@pytest.fixture(scope="module", params=["C3", "C4", "C5"])
def bench(request):
    return _reference(request.param)


def _integrated(ref, **kw):
    v = _vol(ref["cfg"], kw.pop("cap", ref["cap"]), **kw)
    v.set_group_size(GROUP)
    for _ in range(B.PASSES):
        v.integrate_batch(ref["D"], ref["C"], ref["cfg"].K, ref["T"])
    v.synchronize()
    return v


# ---------------------------------------------------------------------------------------------------------------------
# bench scale: fused = un-fused = twin; mesh and point cloud
# ---------------------------------------------------------------------------------------------------------------------

def test_bench_scale_fused_and_unfused_equal_the_twin(bench):
    cfg, ref = bench["cfg"], bench["dump"]
    w = ref["vox"][:, 1]
    nb_min, w_min = REACH[cfg.name]
    assert len(ref["keys"]) >= nb_min and w.max() >= w_min
    assert w[w > 0].min() == B.PASSES                  # every observed voxel took both passes
    fused = _integrated(bench)
    _same_as(fused.dump_blocks(), ref)
    updates = fused.counters()[0]
    fused.close()
    plain = _vol(cfg, bench["cap"])
    plain.set_fusion(False)
    for _ in range(B.PASSES):
        plain.integrate_batch(bench["D"], bench["C"], cfg.K, bench["T"])
    plain.synchronize()
    _same_as(plain.dump_blocks(), ref)
    assert plain.counters()[0] == updates               # the same (block, frame) updates
    plain.close()


def test_bench_scale_mesh_and_point_cloud_equal_the_twin(bench):
    cfg = bench["cfg"]
    vol = _integrated(bench)
    assert vol.num_blocks() > 4 * 1024                  # the mesher's block scan runs over several 1024-block chunks
    m = vol.extract_mesh()
    a, b = B.canon(m), bench["mesh"]
    assert len(a["triangles"]) > 1_000_000
    for k in ("edges", "triangles"):
        assert np.array_equal(a[k], b[k]), k
    for k in ("vertices", "colors"):
        assert np.array_equal(a[k].view(np.uint64), b[k].view(np.uint64)), k
    n = _check_points(vol, cfg.voxel_size, 16, m)
    print(f"\n[{cfg.name} mesh] blocks {vol.num_blocks()}, vertices {len(a['vertices'])}, "
          f"triangles {len(a['triangles'])}, points {n}")
    vol.close()


# ---------------------------------------------------------------------------------------------------------------------
# far and consecutive runs against the Open3D-order restatement
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("run", [B.FAR_C5, B.RUN_C4], ids=["C5-far", "C4-run"])
def test_consecutive_frames_equal_the_open3d_order_oracle(run):
    cfg, D, C, T = B.consecutive(*run)
    n = len(D)
    o3, units = B.open3d_order(cfg, D, C, T)
    want = o3.dump_blocks()
    want_mesh = B.canon(o3.extract_triangle_mesh())
    cap = _capacity(len(want["keys"]))
    # one fused group of all frames, and frame by frame (each frame's touched blocks: the sub-blocks of its units)
    fused = _vol(cfg, cap)
    fused.set_group_size(n)
    fused.integrate_batch(D, C, cfg.K, T)
    frames = _vol(cfg, cap)
    for i in range(n):
        frames.integrate(D[i], C[i], cfg.K, T[i])
        assert np.array_equal(sorted_keys(frames.last_touched_keys()), B.unit_blocks(units[i])), i
    for v in (fused, frames):
        n_obs, wmax = B.equal_to_open3d_order(v.dump_blocks(), want)
        m = B.canon(v.extract_mesh())
        B.same_topology_and_vertices(m, want_mesh)
        assert np.abs(m["colors"] - want_mesh["colors"]).max() < 1e-5
        v.close()
    assert wmax >= 8 and n_obs > 100_000 and len(want_mesh["triangles"]) > 20_000
    if cfg.name == "C5":
        assert np.abs(want_mesh["vertices"][:, 2]).min() > 1900.0
    # float64 colour: voxel and mesh colours equal Open3D's bit for bit
    c64 = _vol(cfg, cap, color_float64=True)
    c64.set_group_size(n)
    c64.integrate_batch(D, C, cfg.K, T)
    a, b = sort_dump(c64.dump_blocks()), sort_dump(want)
    assert np.array_equal(a["keys"], b["keys"])
    assert np.array_equal(a["vox"][:, :2].astype(np.float64), b["vox"][:, :2])
    assert np.array_equal(a["rgb64"].view(np.uint64), b["vox"][:, 2:].view(np.uint64))
    m = B.canon(c64.extract_mesh())
    B.same_topology_and_vertices(m, want_mesh)
    assert np.array_equal(m["colors"].view(np.uint64), want_mesh["colors"].view(np.uint64))
    c64.close()
    print(f"\n[{cfg.name} frames {run[1]}..{run[1] + n - 1}] blocks {len(want['keys'])}, observed voxels {n_obs}, "
          f"max weight {wmax:.0f}, vertices {len(want_mesh['vertices'])}, triangles {len(want_mesh['triangles'])}")


# ---------------------------------------------------------------------------------------------------------------------
# C5 in hash shards, C4's raw-depth leg, C5 growth
# ---------------------------------------------------------------------------------------------------------------------

def _pack(k):
    k = np.asarray(k, np.int64) + (1 << 20)
    return (k[..., 0] << 42) | (k[..., 1] << 21) | k[..., 2]


def _triangle_roots_ok(edges, triangles, owned_keys):
    """tests/_halo_oracle.triangle_roots_ok vectorised: every triangle lies in the 9^3 tile of an owned block."""
    P = np.asarray(edges)[:, :3].astype(np.int64)[np.asarray(triangles, np.int64)]
    lo, hi = P.min(1), P.max(1)
    owned = np.unique(_pack(owned_keys))
    ok = np.zeros(len(P), bool)
    for off in [(0, 0, 0)] + H.OFFSETS:
        b = (lo >> 3) - np.array(off)
        ok |= np.isin(_pack(b), owned) & np.all(lo >= 8 * b, axis=1) & np.all(hi <= 8 * b + 8, axis=1)
    return bool(ok.all())


def _sharded_extraction(single, shards):
    """tests/test_gpu_sharded_extract.py's _check at bench scale: the mesh pieces partition the triangles and weld to
    the unsharded mesh (and to their numpy weld), the point pieces are disjoint and together the unsharded cloud, the
    shards are left untouched.  (The per-record numpy restatement of the halo is checked there on smaller maps.)"""
    world = len(shards)
    before = [v.dump_blocks() for v in shards]
    recs = [sharding.halo_records(v, world) for v in shards]
    mesh = [sharding.mesh_piece(v, [recs[s][r] for s in range(world)]) for r, v in enumerate(shards)]
    pts = [sharding.point_piece(v, [recs[s][r] for s in range(world)]) for r, v in enumerate(shards)]
    full = single.extract_mesh()
    assert sum(len(m.triangles) for m in mesh) == len(full.triangles)
    for r, m in enumerate(mesh):
        assert _triangle_roots_ok(m.edge_ids, m.triangles, before[r]["keys"]), r
    welded = sharding.weld(mesh, device=shards[0].device)
    a, b = B.canon(welded), B.canon(full)
    for k in b:
        assert np.array_equal(a[k], b[k]), k
    nw = H.numpy_weld([dict(vertices=m.vertices, colors=m.vertex_colors, edges=m.edge_ids, triangles=m.triangles)
                       for m in mesh])
    assert np.array_equal(welded.edge_ids, nw["edges"]) and np.array_equal(welded.triangles, nw["triangles"])
    assert np.array_equal(welded.vertices, nw["vertices"]) and np.array_equal(welded.vertex_colors, nw["colors"])
    fpc = single.extract_point_cloud()
    fe = np.asarray(single.extract_point_cloud_with_halo(np.zeros((0, 4), np.int32), np.zeros((0, 5), np.float32))
                    .edge_ids)
    assert len(fe) == len(fpc.points)
    ge = np.concatenate([p.edge_ids for p in pts])
    gp = np.concatenate([p.points for p in pts])
    gc = np.concatenate([p.colors for p in pts])
    assert len(np.unique(ge, axis=0)) == len(ge) == len(fe)
    o1, o2 = np.lexsort(ge.T[::-1]), np.lexsort(fe.T[::-1])
    assert np.array_equal(ge[o1], fe[o2])
    assert np.array_equal(gp[o1], fpc.points[o2]) and np.array_equal(gc[o1], fpc.colors[o2])
    for v, d in zip(shards, before):
        after = v.dump_blocks()
        assert all(np.array_equal(after[k], d[k]) for k in d)
    return len(b["triangles"]), len(fe)


@pytest.mark.parametrize("world", [8, 3])
def test_c5_hash_shards_equal_the_unsharded_volume(world):
    ref = _reference("C5")
    single = _integrated(ref)
    _same_as(single.dump_blocks(), ref["dump"])
    shards = [_integrated(ref, cap=_capacity(len(ref["dump"]["keys"]) / world), shard_rank=r, shard_count=world)
              for r in range(world)]
    parts = []
    for r, s in enumerate(shards):
        p = s.dump_blocks()
        assert len(p["keys"]) > 0 and np.all(p["hashes"] % np.uint64(world) == r)
        parts.append(p)
    _same_as({k: np.concatenate([p[k] for p in parts]) for k in ("keys", "hashes", "vox")}, ref["dump"])
    del parts
    nt, npts = _sharded_extraction(single, shards)
    assert nt > 1_000_000 and npts > 1_000_000
    print(f"\n[C5 x {world} shards] blocks {len(ref['dump']['keys'])}, triangles {nt}, points {npts}")
    for v in shards + [single]:
        v.close()


def test_c4_raw_uint16_depth_leg():
    """bench.py's e2e_u16 leg: the C4 frames rounded to uint16 at 5000 units per metre, pinned, through FrameIngest
    with depth_scale = float32(1/5000); equal to the same depths widened on the host and to the twin."""
    cfg, D, C, T = B.bench_frames("C4")
    scale = np.float32(1.0 / 5000.0)
    assert float(D.max()) * 5000.0 < 65535.0
    raw = np.round(D * 5000.0).astype(np.uint16)
    Df = raw.astype(np.float32) * scale
    assert not np.array_equal(Df, D)                    # the rounding changes the depths
    cap = _capacity(150_000)
    a = _vol(cfg, cap)
    a.set_group_size(GROUP)
    ingest = FrameIngest(a, chunk_frames=64)
    ingest.integrate_batch(torch.from_numpy(raw).pin_memory(), torch.from_numpy(C).pin_memory(), cfg.K, T,
                           depth_scale=scale)
    ingest.synchronize()
    got = sort_dump(a.dump_blocks())
    a.close()
    b = _vol(cfg, cap)
    b.set_group_size(GROUP)
    b.integrate_batch(Df, C, cfg.K, T)
    _same_as(b.dump_blocks(), got)
    b.close()
    _same_as(B.twin(cfg, Df, C, T).dump_blocks(), got)
    assert len(got["keys"]) > 100_000


def test_c5_growth_from_1024_blocks_equals_the_fixed_volume():
    """The street keeps finding new space: a pool of 1024 blocks grows to hold the bench frames' 240k."""
    ref = _reference("C5")
    fixed = _integrated(ref)
    grown = _integrated(ref, cap=1024, max_capacity_blocks=ref["cap"])
    capacity, growths = grown.capacity()
    nb = len(ref["dump"]["keys"])
    assert growths >= 2 and nb <= capacity <= ref["cap"]
    _same_as(grown.dump_blocks(), ref["dump"])
    _same_as(fixed.dump_blocks(), ref["dump"])
    assert grown.counters()[0] == fixed.counters()[0]
    a, b = B.canon(grown.extract_mesh()), ref["mesh"]
    for k in b:
        assert np.array_equal(a[k], b[k]), k
    print(f"\n[C5 growth] 1024 -> {capacity} blocks in {growths} growths, {nb} blocks held")
    fixed.close()
    grown.close()
