"""Map state files without a GPU: the validation of `map_state.read` (every malformed or mismatched input raises
ValueError), the ownership filter of a re-sharding load, and the plugins' SAVE / LOAD task flow with a fake volume."""

import os

import numpy as np
import pytest

from pyslam_b200 import integrator as I
from pyslam_b200 import map_state, sharding
from tests import plugin_standins as P
from pyslam_b200 import synthetic as S

CONFIG = dict(voxel_size=np.float64(0.05), block_size=np.int32(8))
SETTINGS = dict(depth_threshold=np.float32(5.0), depth_decay_rate=np.float32(0.07), next_object_id=np.int32(12))
SPEC = dict(keys=(np.int32, (3,)), count=(np.int32, (512,)), counter=(np.int32, (512,)),
            lab=(np.float32, (512, 8)))
BOUNDS = {"count": (0, None), "counter": (0, 8)}


def _blocks(keys, seed=0):
    rng = np.random.default_rng(seed)
    n = len(keys)
    return dict(keys=np.asarray(keys, np.int32).reshape(n, 3), count=rng.integers(0, 9, (n, 512)).astype(np.int32),
                counter=rng.integers(0, 9, (n, 512)).astype(np.int32),
                lab=rng.standard_normal((n, 512, 8)).astype(np.float32))


def _keys(n, seed=1):
    return np.unique(np.random.default_rng(seed).integers(-50, 50, (3 * n, 3)), axis=0)[:n].astype(np.int32)


def _write(path, blocks, rank=0, count=1, config=CONFIG, settings=SETTINGS, kind="semantic", sk=1):
    map_state.write(str(path), kind, sk, config, settings, rank, count, blocks)
    return str(path)


def _read(paths, rank=0, count=1, max_blocks=1 << 20, config=CONFIG):
    return map_state.read(paths, "semantic", 1, config, {k: v.dtype for k, v in SETTINGS.items()}, SPEC, rank, count,
                          max_blocks, BOUNDS)


def _rewrite(src, dst, **changes):
    with np.load(src) as z:
        d = {k: z[k] for k in z.files}
    for k, v in changes.items():
        if v is None:
            d.pop(k)
        else:
            d[k] = v
    with open(dst, "wb") as f:
        np.savez(f, **d)
    return str(dst)


def test_roundtrip_of_the_file_and_its_settings(tmp_path):
    b = _blocks(_keys(40))
    path = _write(tmp_path / "a.npz", b)
    settings, got = _read(path)
    assert settings == SETTINGS and all(type(settings[k]) is type(SETTINGS[k]) for k in SETTINGS)
    for k in SPEC:
        assert got[k].dtype == b[k].dtype and np.array_equal(got[k], b[k]), k
    with np.load(path, allow_pickle=False) as z:   # no pickled object anywhere
        assert all(z[k].dtype != object for k in z.files)
    settings, got = _read(_write(tmp_path / "e.npz", _blocks(np.zeros((0, 3)))))
    assert len(got["keys"]) == 0 and got["lab"].shape == (0, 512, 8)


@pytest.mark.parametrize("saved,loaded", [(1, 3), (3, 1), (3, 2), (2, 4), (4, 4)])
def test_resharding_keeps_exactly_the_owned_blocks(saved, loaded, tmp_path):
    keys = _keys(300)
    whole = _blocks(keys)
    own = sharding.owner_of(keys, saved)
    files = [_write(tmp_path / f"s{r}.npz", {k: v[own == r] for k, v in whole.items()}, r, saved) for r in range(saved)]
    seen = []
    for r in range(loaded):
        _, got = _read(files, r, loaded)
        assert (sharding.owner_of(got["keys"], loaded) == r).all()
        seen.append(got)
    keys_all = np.concatenate([g["keys"] for g in seen])
    assert len(keys_all) == len(keys)
    merged = sharding.merge_dumps(seen)
    ref = sharding.merge_dumps([whole])
    for k in SPEC:
        assert np.array_equal(merged[k], ref[k]), k


def _bad_cases(tmp_path):
    b = _blocks(_keys(20))
    good = _write(tmp_path / "good.npz", b)
    cnt, ctr = b["count"].copy(), b["counter"].copy()
    cnt[3, 7], ctr[5, 1] = -1, 9
    dup = b["keys"].copy()
    dup[4] = dup[11]
    r = lambda name, **c: _rewrite(good, tmp_path / name, **c)   # noqa: E731
    half = _blocks(_keys(20)[:10])
    return good, {
        "version": r("v.npz", format_version=np.int32(2)),
        "version dtype": r("vd.npz", format_version=np.int64(1)),
        "kind": r("k.npz", kind=np.str_("tsdf")),
        "kind not a string": r("kn.npz", kind=np.int32(3)),
        "semantic kind": r("sk.npz", semantic_kind=np.int32(0)),
        "config value": r("c.npz", voxel_size=np.float64(0.05000001)),
        "config dtype": r("cd.npz", voxel_size=np.float32(0.05)),
        "config missing": r("cm.npz", block_size=None),
        "setting missing": r("sm.npz", next_object_id=None),
        "setting dtype": r("sd.npz", next_object_id=np.int64(12)),
        "shard setting": r("sh.npz", shard_rank=np.int32(2), shard_count=np.int32(2)),
        "array missing": r("am.npz", blocks_lab=None),
        "array unexpected": r("au.npz", blocks_extra=np.zeros(3)),
        "array dtype": r("ad.npz", blocks_count=b["count"].astype(np.int64)),
        "array shape": r("as.npz", blocks_lab=b["lab"][:, :, :4].copy()),
        "array length": r("al.npz", blocks_count=b["count"][:5].copy()),
        "keys shape": r("ks.npz", blocks_keys=b["keys"][:, :2].copy()),
        "negative count": r("nc.npz", blocks_count=cnt),
        "counter above 8": r("ca.npz", blocks_counter=ctr),
        "duplicate keys": r("dk.npz", blocks_keys=dup),
        "a block the saver does not own": _write(tmp_path / "own.npz", b, 0, 2),
        "duplicate across files": [good, _write(tmp_path / "half.npz", half)],
        "settings disagree": [good, _write(tmp_path / "o.npz", _blocks(_keys(5, seed=9) + 1000),
                                           settings=dict(SETTINGS, next_object_id=np.int32(13)))],
        "missing file": str(tmp_path / "nothing.npz"),
        "not an npz": _not_npz(tmp_path),
        "a bare array": _bare(tmp_path),
        "no files": [],
    }


def _not_npz(tmp_path):
    p = tmp_path / "text.npz"
    p.write_text("not a state file")
    return str(p)


def _bare(tmp_path):
    p = tmp_path / "bare.npy"
    np.save(p, np.zeros(3))
    return str(p)


def test_every_malformed_input_is_a_value_error(tmp_path):
    good, cases = _bad_cases(tmp_path)
    _read(good)
    for name, paths in cases.items():
        with pytest.raises(ValueError):
            _read(paths)
            pytest.fail(f"accepted: {name}")


def test_capacity_counts_the_owned_blocks_only(tmp_path):
    keys = _keys(200)
    path = _write(tmp_path / "a.npz", _blocks(keys))
    n0 = int((sharding.owner_of(keys, 2) == 0).sum())
    _read(path, 0, 2, max_blocks=n0)
    with pytest.raises(ValueError):
        _read(path, 0, 2, max_blocks=n0 - 1)
    with pytest.raises(ValueError):
        _read(path, max_blocks=len(keys) - 1)


def test_chunks_bound_the_upload():
    assert map_state.chunks(0, 10240) == [(0, 0)]
    c = map_state.chunks(100000, 10240)
    assert c[0][0] == 0 and c[-1][1] == 100000 and all(b - a <= map_state.CHUNK_BYTES // 10240 for a, b in c)
    assert all(c[i][1] == c[i + 1][0] for i in range(len(c) - 1))
    assert map_state.state_path("/x/dense_map.ply") == "/x/dense_map.state.npz"


# ---- plugins: SAVE writes the state with the parameter on, LOAD restores it and signals -----------------------------

class _StateVolume:
    """A fake volume with save_state / load_state (the state is a small array)."""

    def __init__(self, **kw):
        self.value = np.zeros(3)

    def integrate_batch(self, depths, colors, K, poses, depth_scale=None):
        self.value = self.value + len(depths)

    def reset(self):
        self.value = np.zeros(3)

    def save_state(self, path):
        with open(path, "wb") as f:
            np.save(f, self.value)

    def load_state(self, path):
        if not os.path.exists(path):
            raise ValueError(f"{path}: not a map state file")
        self.value = np.load(path)

    def extract_triangle_mesh(self):
        from types import SimpleNamespace
        v = np.array([self.value, self.value + 1, self.value + 2])
        return SimpleNamespace(vertices=v, triangles=np.array([[0, 1, 2]], np.int32), vertex_colors=np.ones((3, 3)),
                               vertex_normals=np.zeros((0, 3)))

    def close(self):
        pass


def test_plugin_save_and_load_task_flow(monkeypatch, tmp_path):
    monkeypatch.setattr(I, "B200TsdfVolume", _StateVolume)
    Cls = P.standalone_integrator_class()
    cfg = S.CONFIGS["T0"]
    from types import SimpleNamespace
    camera = SimpleNamespace(fx=cfg.fx, fy=cfg.fy, cx=cfg.cx, cy=cfg.cy, width=cfg.width, height=cfg.height, D=None)
    d, c, T = S.render_frame(cfg, 0)
    kd = P.VolumetricIntegrationKeyframeData(id=1, pose=T, img=np.ascontiguousarray(c[..., ::-1]), depth=d)
    one = Cls(camera, P.DatasetEnvironmentType.INDOOR, None, "B200", kVolumetricIntegrationB200SaveMapState=True)
    for _ in range(3):
        one.add_keyframe_data(kd)
    one.run_pending()
    one.save(str(tmp_path))
    one.run_pending()
    assert one.save_request_completed.value == 1
    assert (tmp_path / "dense_map.ply").exists() and (tmp_path / "dense_map.state.npz").exists()
    two = Cls(camera, P.DatasetEnvironmentType.INDOOR, None, "B200")
    notified = []
    orig = two.load_request_condition.notify_all
    two.load_request_condition.notify_all = lambda: (notified.append(two.load_request_completed.value), orig())
    two.load(str(tmp_path / "absent"))
    assert two.load_request_completed.value == 0
    two.run_pending()
    assert notified == [0] and two.load_request_completed.value == 0 and two.is_running.value == 1
    two.load(str(tmp_path))
    two.run_pending()
    assert notified == [0, 1] and two.load_request_completed.value == 1
    assert np.array_equal(two.volume.value, one.volume.value)
    # parameter off (the default): SAVE writes the .ply alone
    off = tmp_path / "off"
    off.mkdir()
    two.save(str(off))
    two.run_pending()
    assert (off / "dense_map.ply").exists() and not (off / "dense_map.state.npz").exists()
