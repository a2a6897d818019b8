"""GPU: the three plugins with kVolumetricIntegrationB200Devices, a map hash-sharded over 2 and 3 ranks (worker
processes), against the single-GPU plugin fed the same tasks.  On one GPU the ranks share device 0 and talk over gloo;
the NCCL test needs two GPUs and skips below."""

import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import oracle
from pyslam_b200 import B200TsdfVolume, map_state, shard_plugin
from pyslam_b200 import synthetic as S
from tests import plugin_standins as P

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _close_groups(monkeypatch):
    """A failing test still stops its workers and frees the process's default process group for the next test."""
    groups = []
    init = shard_plugin.ShardGroup.__init__

    def recorded(self, *a, **k):
        groups.append(self)
        init(self, *a, **k)

    monkeypatch.setattr(shard_plugin.ShardGroup, "__init__", recorded)
    yield
    for g in groups:
        if hasattr(g, "_closed"):
            g.close()


def _canon(m):
    return oracle.canonical_mesh(m.vertices, m.vertex_colors, m.edge_ids, m.triangles)


def _rows(*cols):
    a = np.concatenate([np.asarray(c, np.float64).reshape(len(c), -1) for c in cols], axis=1)
    return a[np.lexsort(a.T[::-1])] if len(a) else a


def _camera(cfg, **kw):
    return SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None, **kw)


def _identity_maps(cfg):
    y, x = np.mgrid[:cfg.height, :cfg.width].astype(np.float32)
    return x, y


def _last_output(integ):
    integ.add_update_output_task()
    integ.step()
    out = None
    while (o := integ.pop_output()) is not None:
        out = o
    return out


def _snap(integ, mesh=True):
    """The map's output now: the welded mesh with its edge ids (the op the plugin's mesh output runs, checked against
    that output), or the output point cloud."""
    out = _last_output(integ)
    if not mesh:
        return out.point_cloud
    m = integ._map_call("mesh")
    assert len(m.triangles) == len(out.mesh.triangles) and np.array_equal(np.sort(m.vertices, 0),
                                                                           np.sort(out.mesh.vertices, 0))
    return m


def _pids(integ):
    return [p.pid for p in integ._shards.procs] if integ._shards is not None else []


def _gone(pids):
    for p in pids:
        try:
            os.kill(p, 0)
        except ProcessLookupError:
            continue
        return False
    return True


def _pair(make, world, devices=None, **kw):
    """(single plugin, sharded plugin) of the same configuration."""
    return make(**kw), make(kVolumetricIntegrationB200Devices=devices or [0] * world, **kw)


# ---- TSDF ------------------------------------------------------------------------------------------------------------

def _tsdf(cfg, raw16=False, gpu_rect=True, **kw):
    api = SimpleNamespace(**{**vars(P.API), "USE_CPP": raw16})
    from pyslam_b200.integrator import make_integrator_class
    Cls = make_integrator_class(P.StandaloneIntegratorBase, api)
    extra = dict(calib_maps=_identity_maps(cfg)) if gpu_rect else {}
    return lambda **k: Cls(_camera(cfg, depth_factor=1.0 / 5000.0), P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF",
                           kVolumetricIntegrationVoxelLength=cfg.voxel_size, kVolumetricIntegrationTSdfTrunc=cfg.sdf_trunc,
                           kVolumetricIntegrationB200CapacityBlocks=1 << 15, **extra, **kw, **k)


def _tsdf_kd(cfg, i, raw16):
    d, c, T = S.render_frame(cfg, i % cfg.n_frames)
    depth = np.round(d * 5000.0).astype(np.uint16) if raw16 else d
    return P.VolumetricIntegrationKeyframeData(id=i, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=depth)


def _same_output(a, b, mesh):
    if mesh:
        ca, cb = _canon(a), _canon(b)
        assert len(a.triangles) > 100
        for k in ("vertices", "triangles", "edges"):
            assert np.array_equal(ca[k], cb[k]), k
    else:
        assert len(a.points) > 100
        assert np.array_equal(_rows(a.points, a.colors), _rows(b.points, b.colors))


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("mesh", [True, False])
def test_tsdf_backlog_reset_and_outputs_T0(world, mesh):
    """40 queued INTEGRATE tasks drained in fused batches, then a RESET between frames."""
    cfg = S.CONFIGS["T0"]
    one, many = _pair(_tsdf(cfg), world, kVolumetricIntegrationB200MaxBatch=16,
                      kVolumetricIntegrationTsdfExtractMesh=mesh)
    pids = _pids(many)
    outs = []
    for integ in (one, many):
        for i in range(40):
            integ.add_keyframe_data(_tsdf_kd(cfg, i, False))
        integ.run_pending()
        first = _snap(integ, mesh)
        integ.reset()
        for i in range(3):
            integ.add_keyframe_data(_tsdf_kd(cfg, 7 + i, False))
            integ.step()
        outs.append((first, _snap(integ, mesh)))
    assert many.integrated_frames == one.integrated_frames == 43
    for a, b in zip(*outs):
        _same_output(a, b, mesh)
    one.quit()
    many.quit()
    assert _gone(pids)


@pytest.mark.parametrize("raw16,gpu_rect", [(True, True), (False, True), (False, False)])
def test_tsdf_C2_raw_depth_rectified_and_host_path(raw16, gpu_rect):
    cfg = S.CONFIGS["C2"]
    one, many = _pair(_tsdf(cfg, raw16, gpu_rect), 2, kVolumetricIntegrationB200MaxBatch=4)
    outs = []
    for integ in (one, many):
        for i in range(6):
            integ.add_keyframe_data(_tsdf_kd(cfg, i, raw16))
        integ.run_pending()
        outs.append(_snap(integ))
    _same_output(outs[0], outs[1], True)
    one.quit()
    many.quit()


def _dump_state(paths, cfg):
    v = B200TsdfVolume(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, capacity_blocks=1 << 15)
    v.load_state(paths)
    d = v.dump_blocks()
    v.close()
    o = np.lexsort(d["keys"].T[::-1])
    return {k: x[o] for k, x in d.items()}


def test_tsdf_save_on_2_ranks_load_into_3_and_into_one(tmp_path):
    cfg = S.CONFIGS["T0"]
    make = _tsdf(cfg, kVolumetricIntegrationB200SaveMapState=True)
    saver = make(kVolumetricIntegrationB200Devices=[0, 0])
    ref = make()
    for integ in (saver, ref):
        for i in range(8):
            integ.add_keyframe_data(_tsdf_kd(cfg, i, False))
        integ.run_pending()
    for name in ("two", "ref", "three", "single"):
        (tmp_path / name).mkdir()
    saver.save(str(tmp_path / "two"))
    ref.save(str(tmp_path / "ref"))
    for integ in (saver, ref):
        integ.step()
        assert integ.save_request_completed.value == 1
    saver.quit()
    saved = _dump_state(map_state.state_files(str(tmp_path / "two" / "dense_map.ply")), cfg)
    assert len(saved["keys"]) > 20
    want = _dump_state(str(tmp_path / "ref" / "dense_map.state.npz"), cfg)
    for k in want:
        assert np.array_equal(saved[k], want[k]), k
    three, single = make(kVolumetricIntegrationB200Devices=[0, 0, 0]), make()
    for integ, name in ((three, "three"), (single, "single")):
        integ.load(str(tmp_path / "two"))
        integ.step()
        assert integ.load_request_completed.value == 1
        integ.save(str(tmp_path / name))      # the loaded map, block for block
        integ.step()
        got = _dump_state(map_state.state_files(str(tmp_path / name / "dense_map.ply")), cfg)
        for k in want:
            assert np.array_equal(got[k], want[k]), (name, k)
    outs = []
    for integ in (three, single, ref):      # later integration continues identically
        for i in range(8, 12):
            integ.add_keyframe_data(_tsdf_kd(cfg, i, False))
        integ.run_pending()
        outs.append(_snap(integ))
    _same_output(outs[0], outs[2], True)
    _same_output(outs[1], outs[2], True)
    for integ in (three, single, ref):
        integ.quit()


# ---- voxel grids -------------------------------------------------------------------------------------------------------

def test_voxel_grid_input_order_sums_bit_for_bit():
    cfg = S.CONFIGS["T0"]
    Cls = P.standalone_voxel_grid_integrator_class()

    def make(**k):
        return Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_VOXEL_GRID",
                   kVolumetricIntegrationVoxelLength=0.03, kVolumetricIntegrationVoxelGridUseCarving=True,
                   kVolumetricIntegrationB200CapacityBlocks=4096, kVolumetricIntegrationB200InputOrderSums=True,
                   calib_maps=_identity_maps(cfg), **k)

    for world in (2, 3):
        one, many = _pair(make, world)
        pids = _pids(many)
        for integ in (one, many):
            for i in range(5):
                integ.add_keyframe_data(_tsdf_kd(cfg, i, False))
                integ.step()
        a, b = (x._map_call("voxels", dict(min_count=1)) for x in (one, many))
        assert len(a.points) > 1000
        assert np.array_equal(_rows(a.points, a.colors), _rows(b.points, b.colors))
        assert len(_last_output(many).point_cloud.points) == len(_last_output(one).point_cloud.points)
        one.quit()
        many.quit()
        assert _gone(pids)


def _c3_kds(n):
    cfg = S.CONFIGS["C3"]
    out = []
    for i in range(n):
        d, c, Tcw = S.render_frame(cfg, 12 * i)
        cls = S.render_class_ids(cfg, 12 * i).astype(np.int32)
        inst = np.where(cls % 3 == 0, -1, cls * 7 + (np.arange(cls.shape[1])[None, :] // 400) + i % 2)
        inst[:40] = 0
        out.append(P.VolumetricIntegrationKeyframeData(id=i, pose=Tcw, img=np.ascontiguousarray(c[..., ::-1]),
                                                       depth=d, semantic_img=cls,
                                                       semantic_instances_img=inst.astype(np.int32)))
    return cfg, out


def _same_objects(a, b):
    la = sorted(a.objects.object_list, key=lambda o: o.object_id)
    lb = sorted(b.objects.object_list, key=lambda o: o.object_id)
    assert len(la) == len(lb) == a.objects.num_objects == b.objects.num_objects > 0
    for x, y in zip(la, lb):
        assert (x.object_id, x.class_id) == (y.object_id, y.class_id)
        assert np.array_equal(_rows(x.points, x.colors), _rows(y.points, y.colors))
        assert (x.confidence_min, x.confidence_max) == (y.confidence_min, y.confidence_max)
        assert np.allclose(x.box_matrix, y.box_matrix, atol=1e-9) and np.allclose(x.box_size, y.box_size, atol=1e-9)


@pytest.mark.parametrize("prob", [False, True])
def test_semantic_objects_and_point_cloud_C3(prob):
    cfg, kds = _c3_kds(4)
    Cls = P.standalone_semantic_integrator_class()

    def make(**k):
        return Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_SEMANTIC",
                   kVolumetricIntegrationVoxelLength=0.015, kVolumetricIntegrationVoxelGridUseCarving=True,
                   kVolumetricIntegrationB200CapacityBlocks=1 << 12, kVolumetricIntegrationB200MaxCapacityBlocks=1 << 17,
                   use_semantic_probabilistic=prob, calib_maps=_identity_maps(cfg), **k)

    for world, objects in ((2, True), (3, True), (2, False)):
        one, many = _pair(make, world, kVolumetricIntegrationB200GenerateObjects=objects)
        outs = []
        for integ in (one, many):
            for kd in kds:
                integ.add_keyframe_data(kd)
                integ.step()
            assert integ.last_instance_map
            outs.append(_last_output(integ))
        assert many.last_instance_map == one.last_instance_map
        if objects:
            _same_objects(*outs)
        else:
            a, b = (o.point_cloud for o in outs)
            assert len(a.points) > 1000
            assert np.array_equal(_rows(a.points, a.colors, a.semantics, a.object_ids),
                                  _rows(b.points, b.colors, b.semantics, b.object_ids))
        one.quit()
        many.quit()


def test_bad_keyframe_is_logged_and_the_loop_goes_on():
    cfg, kds = _c3_kds(2)
    log = []

    class Base(P.StandaloneIntegratorBase):
        print = staticmethod(lambda *a, **k: log.append(" ".join(map(str, a))))

    from pyslam_b200.integrator_semantic import make_semantic_integrator_class
    Cls = make_semantic_integrator_class(Base, P.API)
    integ = Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_SEMANTIC",
                kVolumetricIntegrationB200CapacityBlocks=1 << 12, kVolumetricIntegrationB200MaxCapacityBlocks=1 << 17,
                calib_maps=_identity_maps(cfg), kVolumetricIntegrationB200Devices=[0, 0])
    pids = _pids(integ)
    bad = kds[0]
    integ.add_keyframe_data(P.VolumetricIntegrationKeyframeData(id=9, pose=bad.pose, img=bad.img[:, :-1],
                                                                depth=bad.depth, semantic_img=bad.semantic_img,
                                                                semantic_instances_img=bad.semantic_instances_img))
    integ.step()
    assert any("rank 0" in m and "color" in m for m in log) and integ.is_running.value == 1
    integ.add_keyframe_data(kds[1])
    integ.step()
    assert integ.last_integrated_id == 1 and len(_last_output(integ).objects.object_list) > 0
    integ.quit()
    assert _gone(pids)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_nccl_two_gpus():
    cfg = S.CONFIGS["T0"]
    one, many = _pair(_tsdf(cfg, True, True), 2, devices=[0, 1], kVolumetricIntegrationB200MaxBatch=8)
    assert many._shards.backend == "nccl"
    outs = []
    for integ in (one, many):
        for i in range(20):
            integ.add_keyframe_data(_tsdf_kd(cfg, i, True))
        integ.run_pending()
        outs.append(_snap(integ))
    _same_output(outs[0], outs[1], True)
    one.quit()
    many.quit()
    cfg, kds = _c3_kds(3)
    Cls = P.standalone_semantic_integrator_class()

    def make(**k):
        return Cls(_camera(cfg), P.DatasetEnvironmentType.INDOOR, None, "B200_SEMANTIC",
                   kVolumetricIntegrationB200CapacityBlocks=1 << 12, kVolumetricIntegrationB200MaxCapacityBlocks=1 << 17,
                   use_semantic_probabilistic=True, calib_maps=_identity_maps(cfg), **k)

    one, many = _pair(make, 2, devices=[0, 1])
    outs = []
    for integ in (one, many):
        for kd in kds:
            integ.add_keyframe_data(kd)
            integ.step()
        outs.append(_last_output(integ))
    _same_objects(*outs)
    one.quit()
    many.quit()
