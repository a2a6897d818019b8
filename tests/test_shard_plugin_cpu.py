"""The multi-process plugin protocol (`shard_plugin`) on the CPU: real worker processes over gloo, every rank's map a
recording stand-in.  Every rank must see the calls a single map sees; errors come back to rank 0 and the loop goes on;
no worker outlives the plugin, a failed init() or rank 0."""

import os
import pickle
import signal
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import pytest

from pyslam_b200 import integrator as I
from pyslam_b200 import map_state, shard_plugin, sharding
from pyslam_b200 import synthetic as S
from tests import plugin_standins as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_DIR = "B200_SHARD_TEST_DIR"


class _RecVolume:
    """Stands in for B200TsdfVolume in every rank; appends each call to <dir>/calls.<rank>.pkl."""

    def __init__(self, **kw):
        self.kw, self.rank = kw, kw.get("shard_rank", "single")
        self.calls = [("pid", os.getpid())]
        if os.environ.get("B200_SHARD_TEST_FAIL_CREATE") == str(self.rank):
            self._log()
            raise RuntimeError(f"no room on rank {self.rank}")
        self._log()

    def _log(self):
        with open(os.path.join(os.environ[_DIR], f"calls.{self.rank}.pkl"), "wb") as f:
            pickle.dump(self.calls, f)

    def _rec(self, *call):
        self.calls.append(call)
        self._log()

    def integrate_batch(self, depths, colors, K, poses, depth_scale=None):
        poses = np.asarray(poses, np.float64).reshape(-1, 4, 4)
        if self.rank == 1 and poses[0, 0, 3] == 99.0:
            raise RuntimeError("poisoned frame on rank 1")
        self._rec("integrate_batch", tuple(float(k) for k in K), poses.copy(), np.asarray(depths).dtype.str,
                  float(np.asarray(depths, np.float64).sum()), int(np.asarray(colors, np.int64).sum()),
                  None if depth_scale is None else float(depth_scale))

    def reset(self):
        self._rec("reset")

    def extract_triangle_mesh(self):
        self._rec("mesh")
        return SimpleNamespace(vertices=np.zeros((3, 3)), triangles=np.array([[0, 1, 2]], np.int32),
                               vertex_colors=np.zeros((3, 3)), vertex_normals=np.zeros((0, 3)))

    def save_state(self, path):
        self._rec("save_state", os.path.basename(path))
        open(path, "wb").close()

    def load_state(self, paths):
        self._rec("load_state", [os.path.basename(p) for p in ([paths] if isinstance(paths, str) else paths)])

    def close(self):
        self._rec("close")


def _mesh_sharded(volume):
    m = volume.extract_triangle_mesh()
    return m if volume.rank == 0 else None


def _install_fakes():
    I.B200TsdfVolume = _RecVolume
    sharding.extract_mesh_sharded = _mesh_sharded


def _fake_worker_plugin(spec, side):
    """WORKER_FACTORY of these tests: the worker's plugin with the recording map."""
    _install_fakes()
    return shard_plugin.worker_plugin(spec, side)


@pytest.fixture
def fakes(monkeypatch, tmp_path):
    monkeypatch.setenv(_DIR, str(tmp_path))
    monkeypatch.setattr(I, "B200TsdfVolume", _RecVolume)
    monkeypatch.setattr(sharding, "extract_mesh_sharded", _mesh_sharded)
    monkeypatch.setattr(shard_plugin, "WORKER_FACTORY", "tests.test_shard_plugin_cpu:_fake_worker_plugin")
    monkeypatch.setattr(shard_plugin, "device_count", lambda: 2)
    monkeypatch.setattr(shard_plugin, "TIMEOUT_S", 30.0)
    monkeypatch.setattr(shard_plugin, "JOIN_TIMEOUT_S", 10.0)
    return tmp_path


def _calls(folder, rank):
    with open(os.path.join(folder, f"calls.{rank}.pkl"), "rb") as f:
        return pickle.load(f)


def _alive(pid):
    try:
        os.kill(pid, 0)
    except ProcessLookupError:
        return False
    try:   # a zombie child of this process is gone for every purpose but its pid
        return os.waitpid(pid, os.WNOHANG) == (0, 0)
    except ChildProcessError:
        return True


def _gone(pids, within=15.0):
    end = time.monotonic() + within
    while time.monotonic() < end and any(_alive(p) for p in pids):
        time.sleep(0.1)
    return not any(_alive(p) for p in pids)


def _camera():
    cfg = S.CONFIGS["T0"]
    return SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)


def _plugin(base=P.StandaloneIntegratorBase, **kw):
    Cls = I.make_integrator_class(base, P.API)
    return Cls(_camera(), P.DatasetEnvironmentType.INDOOR, None, "B200_TSDF", **kw)


def _kd(i, x=None):
    d, c, T = S.render_frame(S.CONFIGS["T0"], i % 3)
    T = T.copy()
    T[0, 3] += 0.01 * i if x is None else x - T[0, 3]
    return P.VolumetricIntegrationKeyframeData(id=i, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=d)


def _feed(integ, folder):
    """A task sequence through the plugin: a drained backlog (fused batches and a single frame), an output, a RESET,
    one more frame and SAVE with the map state."""
    for i in range(5):
        integ.add_keyframe_data(_kd(i))
    integ.run_pending()
    integ.add_update_output_task()
    integ.step()
    integ.reset()
    integ.add_keyframe_data(_kd(5))
    integ.step()
    integ.save(str(folder))
    integ.step()
    assert integ.save_request_completed.value == 1


@pytest.mark.parametrize("world", [2, 3])
def test_every_rank_makes_the_single_maps_calls(fakes, world):
    single_dir, shard_dir = fakes / "single", fakes / "sharded"
    single_dir.mkdir()
    shard_dir.mkdir()
    one = _plugin(kVolumetricIntegrationB200MaxBatch=4, kVolumetricIntegrationB200SaveMapState=True)
    _feed(one, single_dir)
    one.quit()
    want = _calls(fakes, "single")[1:]
    integ = _plugin(kVolumetricIntegrationB200MaxBatch=4, kVolumetricIntegrationB200SaveMapState=True,
                    kVolumetricIntegrationB200Devices=[0] * world)
    assert integ._shards.backend == "gloo" and integ._shards.world == world
    pids = [p.pid for p in integ._shards.procs]
    _feed(integ, shard_dir)
    integ.quit()
    assert _gone(pids)
    for r in range(world):
        got = _calls(fakes, r)
        assert got[0][1] == (os.getpid() if r == 0 else pids[r - 1])
        got = got[1:]
        assert len(got) == len(want), (r, [c[0] for c in got], [c[0] for c in want])
        for g, w in zip(got, want):
            if g[0] == "save_state":
                assert g[1] == f"dense_map.state.{r}-of-{world}.npz" and w[1] == "dense_map.state.npz"
                continue
            assert g[0] == w[0]
            for a, b in zip(g[1:], w[1:]):
                assert np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b, (r, g[0])
    names = [c[0] for c in want]
    assert names.count("integrate_batch") == 3 and names.index("reset") > names.index("mesh")
    assert sorted(os.listdir(shard_dir)) == sorted(["dense_map.ply"] + [f"dense_map.state.{r}-of-{world}.npz"
                                                                         for r in range(world)])


def test_load_reads_shard_files_on_every_rank(fakes):
    for r in range(2):
        open(fakes / f"dense_map.state.{r}-of-2.npz", "wb").close()
    integ = _plugin(kVolumetricIntegrationB200Devices=[0, 0, 0])
    pids = [p.pid for p in integ._shards.procs]
    integ.load(str(fakes))
    integ.step()
    assert integ.load_request_completed.value == 1
    integ.quit()
    assert _gone(pids)
    for r in range(3):
        assert ("load_state", ["dense_map.state.0-of-2.npz", "dense_map.state.1-of-2.npz"]) in _calls(fakes, r)


class _LoggingBase(P.StandaloneIntegratorBase):
    log = []
    print = staticmethod(lambda *a, **k: _LoggingBase.log.append(" ".join(map(str, a))))


def test_a_worker_error_reaches_rank_0_and_the_loop_goes_on(fakes):
    _LoggingBase.log.clear()
    integ = _plugin(_LoggingBase, kVolumetricIntegrationB200Devices=[0, 0])
    pids = [p.pid for p in integ._shards.procs]
    integ.add_keyframe_data(_kd(0, x=99.0))
    integ.step()
    assert any("rank 1: RuntimeError: poisoned frame on rank 1" in m for m in _LoggingBase.log)
    assert integ.is_running.value == 1
    integ.add_keyframe_data(_kd(1))
    integ.step()
    assert [c[0] for c in _calls(fakes, 1)].count("integrate_batch") == 1
    assert [c[0] for c in _calls(fakes, 0)].count("integrate_batch") == 2
    integ.quit()
    assert _gone(pids)


def test_a_killed_worker_fails_the_next_op_instead_of_hanging(fakes):
    _LoggingBase.log.clear()
    integ = _plugin(_LoggingBase, kVolumetricIntegrationB200Devices=[0, 0, 0])
    pids = [p.pid for p in integ._shards.procs]
    os.kill(pids[0], signal.SIGKILL)
    t0 = time.monotonic()
    integ.add_keyframe_data(_kd(0))
    integ.step()
    assert time.monotonic() - t0 < shard_plugin.TIMEOUT_S
    assert any("shard group is down" in m for m in _LoggingBase.log)
    assert _gone(pids)
    integ.add_update_output_task()
    integ.step()                      # every later op fails at once
    assert integ.is_running.value == 1
    integ.quit()


def test_a_failed_init_leaves_no_worker(fakes, monkeypatch):
    monkeypatch.setenv("B200_SHARD_TEST_FAIL_CREATE", "2")
    with pytest.raises(RuntimeError, match="rank 2: RuntimeError: no room on rank 2"):
        _plugin(kVolumetricIntegrationB200Devices=[0, 0, 0])
    pids = [_calls(fakes, r)[0][1] for r in (1, 2)]
    assert _gone(pids)


def _orphan_main(folder):
    """Rank 0 that dies without shutting its workers down (run in a child process by the next test)."""
    os.environ[_DIR] = folder
    _install_fakes()
    shard_plugin.WORKER_FACTORY = "tests.test_shard_plugin_cpu:_fake_worker_plugin"
    shard_plugin.device_count = lambda: 1
    integ = _plugin(kVolumetricIntegrationB200Devices=[0, 0, 0])
    print(" ".join(str(p.pid) for p in integ._shards.procs), flush=True)
    os._exit(1)


def test_workers_exit_with_rank_0(fakes):
    code = f"import tests.test_shard_plugin_cpu as t; t._orphan_main({str(fakes)!r})"
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=300)
    pids = [int(p) for p in out.stdout.split()]
    assert len(pids) == 2, out.stderr
    assert _gone(pids)


def test_device_list_validation_and_backend_rule(monkeypatch):
    monkeypatch.setattr(shard_plugin, "device_count", lambda: 2)
    assert shard_plugin.parse_devices([]) == [] and shard_plugin.parse_devices([1, 0]) == [1, 0]
    for bad in ((0, 1), "0,1", 3, None, [0, 2], [-1], [0, 1.0], [True]):
        with pytest.raises(RuntimeError, match="kVolumetricIntegrationB200Devices"):
            shard_plugin.parse_devices(bad)
    assert shard_plugin.backend_for([0, 1]) == "nccl" and shard_plugin.backend_for([1, 0, 2]) == "nccl"
    assert shard_plugin.backend_for([0, 0]) == "gloo" and shard_plugin.backend_for([0, 1, 1]) == "gloo"
    monkeypatch.setattr(I, "B200TsdfVolume", _RecVolume)
    monkeypatch.setenv(_DIR, "/nonexistent")
    with pytest.raises(RuntimeError, match=r"outside \[0, 2\)"):
        _plugin(kVolumetricIntegrationB200Devices=[0, 5])


def test_no_process_for_an_empty_or_one_entry_list(fakes, monkeypatch):
    def no_group(*a, **k):
        raise AssertionError("a shard group was started")

    monkeypatch.setattr(shard_plugin, "ShardGroup", no_group)
    _LoggingBase.log.clear()
    a = _plugin(_LoggingBase)
    assert a._shards is None and a.volume.kw["device"] == 0 and not _LoggingBase.log
    b = _plugin(_LoggingBase, kVolumetricIntegrationB200Devices=[1], kVolumetricIntegrationB200Device=0)
    assert b._shards is None and b.volume.kw["device"] == 1 and "shard_rank" not in b.volume.kw
    assert any("kVolumetricIntegrationB200Device ignored" in m for m in _LoggingBase.log)


def test_state_files_single_or_shard_set(tmp_path):
    ply = str(tmp_path / "dense_map.ply")
    assert map_state.state_files(ply) == map_state.state_path(ply)      # nothing saved: the single path
    for r in range(3):
        open(map_state.shard_state_path(ply, r, 3), "wb").close()
    assert map_state.state_files(ply) == [str(tmp_path / f"dense_map.state.{r}-of-3.npz") for r in range(3)]
    open(map_state.shard_state_path(ply, 0, 2), "wb").close()            # an incomplete set beside a complete one
    assert len(map_state.state_files(ply)) == 3
    open(map_state.shard_state_path(ply, 1, 2), "wb").close()
    with pytest.raises(ValueError, match="more than one set"):
        map_state.state_files(ply)
    map_state.remove_other_states(ply, 2)
    assert len(map_state.state_files(ply)) == 2
    open(map_state.state_path(ply), "wb").close()                        # the single file wins
    assert map_state.state_files(ply) == map_state.state_path(ply)
    map_state.remove_other_states(ply, 2)
    os.remove(map_state.shard_state_path(ply, 1, 2))
    with pytest.raises(ValueError, match="no complete set"):
        map_state.state_files(ply)
