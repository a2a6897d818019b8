"""Growable TSDF volume (max_capacity_blocks): a volume that grew holds, block for block and bit for bit, what a volume
big enough from the start holds - the twin's dump, the fixed volume's mesh and its (block, frame) update count - in
every integration mode and at the edges of the pipeline: groups that overflow the pool are skipped, the pool grows,
and the skipped groups are replayed in order.  The last test (CPU) checks the ctypes mirror of b2v_config."""

import os
import shutil
import subprocess

import numpy as np
import pytest

import oracle
from pyslam_b200 import B200TsdfVolume
from pyslam_b200 import synthetic as S
from tests._util import GOLDEN, ROOT, sort_dump

START, MAX = 64, 1 << 16


def _volume(cfg, capacity, max_capacity=None, **kw):
    return B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=capacity,
                          max_capacity_blocks=max_capacity, **kw)


def _same(a, b):
    a, b = sort_dump(a), sort_dump(b)
    for name in ("keys", "hashes", "vox"):
        assert np.array_equal(a[name], b[name]), name


def _mesh(vol):
    m = vol.extract_mesh()
    return oracle.canonical_mesh(m.vertices, m.vertex_colors, m.edge_ids, m.triangles)


def _same_mesh(a, b):
    for name in ("edges", "triangles", "vertices", "colors"):
        assert np.array_equal(a[name], b[name]), name


_frames_cache, _twin_cache = {}, {}


def _frames(name):
    if name not in _frames_cache:
        cfg = S.CONFIGS[name]
        fr = [S.render_frame(cfg, i) for i in range(cfg.n_frames)]
        _frames_cache[name] = tuple(np.stack([f[k] for f in fr]) for k in range(3))
    return _frames_cache[name]


def _twin(name):
    if name not in _twin_cache:
        cfg = S.CONFIGS[name]
        tw = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc)
        D, C, T = _frames(name)
        for i in range(len(D)):
            tw.integrate(D[i], C[i], cfg.K, T[i], nthreads=8)
        _twin_cache[name] = tw.dump_blocks()
    return _twin_cache[name]


MODES = ["frames", "group1", "group3", "group16", "group32", "fusion_off", "overlap_off"]


def _integrate(vol, mode, D, C, T, K):
    """The frames in `mode`.  Batches go in two calls with a synchronising call between them, so that even 32-frame
    groups overflow the pool twice."""
    if mode == "frames":
        for i in range(len(D)):
            vol.integrate(D[i], C[i], K, T[i])
        return
    if mode.startswith("group"):
        vol.set_group_size(int(mode[5:]))
    elif mode == "fusion_off":
        vol.set_fusion(False)
    elif mode == "overlap_off":
        vol.set_overlap(False)
    h = len(D) // 2
    vol.integrate_batch(D[:h], C[:h], K, T[:h])
    vol.capacity()
    vol.integrate_batch(D[h:], C[h:], K, T[h:])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C1", "T0"])
@pytest.mark.parametrize("mode", MODES)
def test_grown_volume_equals_twin_and_fixed_volume(name, mode):
    cfg = S.CONFIGS[name]
    D, C, T = _frames(name)
    out = {}
    for label, cap, mx in (("fixed", MAX, None), ("grown", START, MAX)):
        vol = _volume(cfg, cap, mx)
        _integrate(vol, mode, D, C, T, cfg.K)
        vol.synchronize()
        out[label] = (vol.dump_blocks(), _mesh(vol), vol.counters()[0], vol.capacity())
        vol.close()
    dump, mesh, updates, (capacity, growths) = out["grown"]
    _same(dump, _twin(name))
    _same_mesh(mesh, out["fixed"][1])
    assert updates == out["fixed"][2]
    assert growths >= 2 and START < capacity <= MAX and capacity >= len(dump["keys"])
    assert out["fixed"][3] == (MAX, 0)


def _pair(cfg, run, **kw):
    """run(volume) on a fixed volume of MAX blocks and on a growable one from START: equal dumps and update counts."""
    res = []
    for cap, mx in ((MAX, None), (START, MAX)):
        vol = _volume(cfg, cap, mx, **kw)
        run(vol)
        vol.synchronize()
        res.append((vol.dump_blocks(), vol.counters()[0], vol.capacity()[1]))
        vol.close()
    _same(res[0][0], res[1][0])
    assert res[0][1] == res[1][1]
    assert res[1][2] >= 1
    return res[1][0]


@pytest.mark.gpu
def test_device_frames_on_a_caller_stream():
    import torch
    cfg = S.CONFIGS["C1"]
    D, C, T = _frames("C1")
    d, c = torch.from_numpy(D).cuda(), torch.from_numpy(C).cuda()
    s = torch.cuda.Stream()

    def run(vol):
        with torch.cuda.stream(s):
            vol.integrate_batch(d[:60], c[:60], cfg.K, T[:60], stream=s.cuda_stream)
            for i in range(60, 70):
                vol.integrate(d[i], c[i], cfg.K, T[i], stream=s.cuda_stream)
        s.synchronize()

    _pair(cfg, run)


@pytest.mark.gpu
def test_frame_ingest_with_input_event():
    from pyslam_b200.sharding import FrameIngest
    cfg = S.CONFIGS["C1"]
    D, C, T = _frames("C1")

    def run(vol):
        FrameIngest(vol, chunk_frames=24).integrate_batch(D, C, cfg.K, T)

    _same(_pair(cfg, run), _twin("C1"))


@pytest.mark.gpu
def test_raw_uint16_depth():
    cfg = S.CONFIGS["C1"]
    D, C, T = _frames("C1")
    D16 = np.round(D[:50] * 1000.0).astype(np.uint16)

    def run(vol):
        vol.integrate_batch(D16[:40], C[:40], cfg.K, T[:40], depth_scale=1e-3)
        for i in range(40, 50):
            vol.integrate(D16[i], C[i], cfg.K, T[i], depth_scale=1e-3)

    _pair(cfg, run)


@pytest.mark.gpu
def test_gpu_rectification():
    g = np.load(os.path.join(GOLDEN, "remap_T0.npz"))
    cfg = S.CONFIGS["T0"]
    K = (float(g["new_K"][0, 0]), float(g["new_K"][1, 1]), float(g["new_K"][0, 2]), float(g["new_K"][1, 2]))
    D, C, T = _frames("T0")
    bgr = np.ascontiguousarray(C[..., ::-1])

    def run(vol):
        vol.set_rectification(g["map1"], g["map2"], swap_rb=True)
        vol.integrate_batch(D, bgr, K, T)

    _pair(cfg, run)


@pytest.mark.gpu
def test_new_intrinsics_and_larger_frames_right_after_an_overflow():
    """The lambda image and the texel images are rewritten only after the skipped groups were replayed with them."""
    cfg, big = S.CONFIGS["T0"], S.CONFIGS["C1"]
    D, C, T = _frames("T0")
    Db, Cb, Tb = _frames("C1")
    K2 = (cfg.fx * 1.1, cfg.fy * 1.1, cfg.cx, cfg.cy)

    def run(vol):
        vol.integrate_batch(D[:12], C[:12], cfg.K, T[:12])   # overflows the 64 blocks at once
        vol.integrate_batch(D[12:], C[12:], K2, T[12:])      # new intrinsics
        vol.integrate_batch(Db[:8], Cb[:8], big.K, Tb[:8])   # larger frames: new staging
        for i in range(8, 12):
            vol.integrate(Db[i], Cb[i], big.K, Tb[i])

    _pair(cfg, run)


@pytest.mark.gpu
def test_overflow_in_the_last_group_only():
    """The pool fills in the last group of the call; synchronize() grows it and replays that group."""
    cfg = S.CONFIGS["C1"]
    D, C, T = _frames("C1")
    probe = _volume(cfg, MAX)
    probe.set_group_size(8)
    probe.integrate_batch(D[:24], C[:24], cfg.K, T[:24])
    n24 = probe.num_blocks()
    probe.close()
    res = []
    for cap, mx in ((MAX, None), (n24, MAX)):
        vol = _volume(cfg, cap, mx)
        vol.set_group_size(8)
        vol.integrate_batch(D[:32], C[:32], cfg.K, T[:32])
        vol.synchronize()
        res.append((vol.dump_blocks(), vol.counters()[0], vol.capacity()[1]))
        vol.close()
    _same(res[0][0], res[1][0])
    assert res[0][1] == res[1][1] and res[1][2] == 1


@pytest.mark.gpu
def test_two_hash_shards_equal_the_unsharded_twin():
    cfg = S.CONFIGS["T0"]
    D, C, T = _frames("T0")
    parts = []
    for r in range(2):
        vol = _volume(cfg, START, MAX, shard_rank=r, shard_count=2)
        vol.integrate_batch(D, C, cfg.K, T)
        vol.synchronize()
        assert vol.capacity()[1] >= 1
        parts.append(vol.dump_blocks())
        vol.close()
    merged = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    _same(merged, _twin("T0"))


@pytest.mark.gpu
def test_ceiling_one_block_short_raises_and_exact_ceiling_does_not():
    cfg = S.CONFIGS["T0"]
    D, C, T = _frames("T0")
    ref = _twin("T0")
    n = len(ref["keys"])
    short = _volume(cfg, START, n - 1)
    short.integrate_batch(D, C, cfg.K, T)
    with pytest.raises(RuntimeError, match="block pool full"):
        short.synchronize()
    short.close()
    exact = _volume(cfg, START, n)
    exact.integrate_batch(D, C, cfg.K, T)
    exact.synchronize()
    _same(exact.dump_blocks(), ref)
    assert exact.capacity()[0] == n
    exact.close()
    fixed = _volume(cfg, n - 1)   # growth off: the pool-full error, as for any fixed pool
    fixed.integrate_batch(D, C, cfg.K, T)
    with pytest.raises(RuntimeError, match="block pool full"):
        fixed.synchronize()
    assert fixed.num_blocks() == n - 1
    fixed.close()


@pytest.mark.gpu
def test_upload_and_import_grow_the_pool():
    import torch
    cfg = S.CONFIGS["T0"]
    ref = sort_dump(_twin("T0"))
    vol = _volume(cfg, START, MAX)
    vol.upload_blocks(ref["keys"][:1000], ref["vox"][:1000])
    assert vol.capacity()[0] >= 1000
    keys4 = torch.zeros((len(ref["keys"]) - 1000, 4), dtype=torch.int32)
    keys4[:, :3] = torch.from_numpy(ref["keys"][1000:])
    vol.import_blocks_torch(keys4.cuda(), torch.from_numpy(np.ascontiguousarray(ref["vox"][1000:])).cuda())
    _same(vol.dump_blocks(), ref)
    assert vol.capacity()[0] >= len(ref["keys"]) and vol.capacity()[1] >= 2
    vol.close()


@pytest.mark.gpu
def test_reset_keeps_the_capacity():
    cfg = S.CONFIGS["T0"]
    D, C, T = _frames("T0")
    vol = _volume(cfg, START, MAX)
    vol.integrate_batch(D, C, cfg.K, T)
    vol.synchronize()
    grown = vol.capacity()
    vol.integrate_batch(D[:4], C[:4], cfg.K, T[:4])   # pending work at the reset is discarded
    vol.reset()
    assert vol.num_blocks() == 0 and vol.capacity() == grown
    vol.integrate_batch(D, C, cfg.K, T)
    vol.synchronize()
    _same(vol.dump_blocks(), _twin("T0"))
    assert vol.capacity() == grown
    vol.close()


@pytest.mark.gpu
def test_plugin_with_a_growable_pool_emits_the_large_pool_mesh():
    from tests import plugin_standins as P
    from tests.test_plugin import _camera
    cfg = S.CONFIGS["T0"]
    D, C, T = _frames("T0")
    meshes = []
    for kw in (dict(kVolumetricIntegrationB200CapacityBlocks=MAX),
               dict(kVolumetricIntegrationB200CapacityBlocks=256, kVolumetricIntegrationB200MaxCapacityBlocks=MAX)):
        integ = P.standalone_integrator_class()(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF",
                                                kVolumetricIntegrationVoxelLength=cfg.voxel_size,
                                                kVolumetricIntegrationTSdfTrunc=cfg.sdf_trunc, **kw)
        for i in range(len(D)):
            integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(
                id=i, pose=T[i], img=np.ascontiguousarray(C[i][..., ::-1]), depth=D[i]))
        integ.run_pending()
        integ.add_update_output_task()
        integ.step()
        out = None
        while (o := integ.pop_output()) is not None:
            out = o
        V, Cc, Tr = (np.asarray(a) for a in (out.mesh.vertices, out.mesh.vertex_colors, out.mesh.triangles))
        vc = np.hstack([V, Cc])
        tri = V[Tr].reshape(len(Tr), 9)   # triangles by their vertices' positions: pool order drops out
        meshes.append(dict(vertices=vc[np.lexsort(vc.T[::-1])], triangles=tri[np.lexsort(tri.T[::-1])]))
        if "kVolumetricIntegrationB200MaxCapacityBlocks" in kw:
            assert integ.volume.capacity()[1] >= 1
        integ.quit()
    for name in ("vertices", "triangles"):
        assert np.array_equal(meshes[0][name], meshes[1][name]), name


def test_config_struct_layout_matches_the_header(tmp_path):
    """CPU: b2v_config's offsets and size as a C compiler lays them out equal the ctypes mirror's."""
    import ctypes
    from pyslam_b200._lib import B2VConfig
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    if not gcc:
        pytest.skip("gcc not available")
    names = [f[0] for f in B2VConfig._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b2v.h"\nint main(void) {\n'
                   + "".join(f'    printf("%zu\\n", offsetof(b2v_config, {n}));\n' for n in names)
                   + '    printf("%zu\\n", sizeof(b2v_config));\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    r = subprocess.run([gcc, "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    assert got == [getattr(B2VConfig, n).offset for n in names] + [ctypes.sizeof(B2VConfig)]
    assert names[-1] == "max_capacity_blocks"
