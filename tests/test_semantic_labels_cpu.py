"""CPU: the unbounded label map of tests/_semantic_labels.py, the oracle of the Bayesian grid with an overflow label
store.  It equals the 8-slot oracle where no voxel passes 8 pairs (the committed reference run), equals the compiled
reference live on scenes with 9, 17 and 40 pairs per voxel (when oracle/_ref is built), and the scenes reach what the
GPU tests rely on: more than 8 pairs, chains of 3 chunks and more, chunks released and needed again, and more chunks
than one."""

import os

import numpy as np
import pytest

import oracle
from tests import _grid_prep_scenes as E
from tests import _semantic_labels as SL
from tests import _semantic_scenes as SC
from tests._util import GOLDEN, sort_dump

FIELDS = ("keys", "count", "pos_sum", "col_sum", "object_id", "class_id", "aux", "lab_obj", "lab_cls", "lab_logp",
          "confidence")


def test_unbounded_map_equals_the_8_slot_oracle_on_the_reference_run():
    g = np.load(os.path.join(GOLDEN, "semantic_T0.npz"))
    grids = [oracle.numpy_semantic_grid(float(g["voxel_size"]), "probabilistic"),
             SL.UnboundedSemanticGrid(float(g["voxel_size"]))]
    for G in grids:
        G.set_depth_threshold(float(g["prob_depth_threshold"]))
        G.set_depth_decay_rate(float(g["prob_depth_decay_rate"]))
        for i in range(int(g["n_frames"])):
            G.integrate(*[g[f"prob_{n}_{i}"] for n in ("points", "colors", "cls", "inst", "depths")])
    a, b = grids[0].dump(), grids[1].dump()
    assert grids[1].max_pairs() <= 8 and grids[0].label_overflows == 0
    for k in FIELDS:
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("n", [9, 17, 40])
def test_scene_census(n):
    most, chain, used, reuse = SL.census(SL.scene_many_pairs(n))
    assert most >= n
    assert chain == SL.chunks_of(most) and chain >= (1 if n < 33 else 3)
    assert reuse, "an edit released chunks that a later call needed again"
    assert max(used) > 1, "the store must grow past one chunk"


def test_churn_census():
    T0, _ = E.cam_poses()
    most, chain, used, reuse = SL.census(SL.scene_churn(T0))
    assert most > 8 and max(used) > 100 and reuse


def test_unbounded_map_without_chains_is_the_8_slot_oracle():
    """Every scene of tests/_semantic_scenes.py whose voxels stay within 8 pairs gives the same dump both ways."""
    for name, sc in SC.scenes().items():
        if name.startswith("eviction"):
            continue
        G8 = oracle.numpy_semantic_grid(SC.VS, "probabilistic")
        GU = SL.UnboundedSemanticGrid(SC.VS)
        for t in (G8, GU):
            t.set_depth_threshold(sc.get("depth_threshold", 5.0))
            t.set_depth_decay_rate(sc.get("depth_decay_rate", 0.07))
        for op, kw in sc["steps"]:
            SC.apply(G8, "oracle", op, kw)
            SC.apply(GU, "oracle", op, kw)
        a, b = G8.dump(), GU.dump(8)
        for k in FIELDS:
            assert np.array_equal(a[k], b[k]), (name, k)


@pytest.mark.skipif(not oracle.have_ref_semantic(), reason="compiled reference (oracle/_ref) not built")
@pytest.mark.parametrize("n", [9, 17, 40])
def test_unbounded_map_equals_the_compiled_reference(n):
    sc = SL.scene_many_pairs(n)
    sc = dict(sc, steps=[s for s in sc["steps"] if s[0] != "clear"])
    G = SL.UnboundedSemanticGrid(SC.VS)
    R = oracle.RefSemanticGrid(SC.VS, "probabilistic")
    for t in (G, R):
        t.set_depth_threshold(sc["depth_threshold"])
        t.set_depth_decay_rate(sc["depth_decay_rate"])
    for i, (op, kw) in enumerate(sc["steps"]):
        SC.apply(G, "oracle", op, kw)
        SC.apply(R, "ref", op, kw)
        K = max(8, G.max_pairs())
        a, b = G.dump(K), sort_dump(R.dump_blocks(K))
        for k in ("keys", "count", "pos_sum", "col_sum", "object_id", "class_id", "aux", "lab_obj", "lab_cls"):
            assert np.array_equal(a[k], b[k]), (n, i, op, k)
        fin = np.isfinite(b["lab_logp"])
        assert np.array_equal(np.isfinite(a["lab_logp"]), fin), (n, i)
        assert np.allclose(a["lab_logp"][fin], b["lab_logp"][fin], rtol=1e-6, atol=0), (n, i, op)
        assert np.allclose(a["confidence"], b["confidence"], rtol=2e-6, atol=1e-9), (n, i, op)


# ---- overflow label pairs in the map state file ----------------------------------------------------------------------

def _state(tmp_path, labels, name="s.npz", counter=None):
    """A one-block Bayesian state file whose voxels 3 and 9 hold 2 and 9 overflow pairs."""
    from pyslam_b200 import map_state
    V = 512
    cnt = np.zeros((1, V), np.int32)
    cnt[0, 3], cnt[0, 9] = 2, 9
    ctr = np.where(cnt > 0, 8 + cnt, 1).astype(np.int32) if counter is None else counter
    arrays = dict(keys=np.zeros((1, 3), np.int32), counter=ctr)
    lab = dict(count=cnt, obj=np.arange(11, dtype=np.int32), cls=np.arange(11, dtype=np.int32),
               logp=np.full(11, 0.25, np.float32))
    lab.update(labels)
    path = str(tmp_path / name)
    map_state.write(path, "semantic", 1, {}, {}, 0, 1, arrays, lab)
    return path


def _read_state(path, labels=True):
    from pyslam_b200 import map_state
    spec = dict(keys=(np.int32, (3,)), counter=(np.int32, (512,)))
    return map_state.read(path, "semantic", 1, {}, {}, spec, 0, 1, 16, {"counter": (0, 8)}, labels=labels)


def test_state_file_label_arrays_round_trip_and_validation(tmp_path):
    from pyslam_b200 import map_state
    _, blocks, lab = _read_state(_state(tmp_path, {}))
    assert lab["count"][0, 9] == 9 and len(lab["obj"]) == 11 and blocks["counter"][0, 9] == 17
    s = map_state.label_slice(lab, 0, 1)
    assert np.array_equal(s["logp"], lab["logp"])
    imin = np.iinfo(np.int32).min
    bad = [dict(count=np.full((1, 512), -1, np.int32)), dict(obj=np.arange(10, dtype=np.int32)),
           dict(obj=np.full(11, imin, np.int32)), dict(cls=np.full(11, imin, np.int32)),
           dict(logp=np.full(11, np.nan, np.float32)), dict(logp=np.full(11, -1.0, np.float32)),
           dict(logp=np.zeros(11, np.float64))]
    for i, b in enumerate(bad):
        with pytest.raises(ValueError):
            _read_state(_state(tmp_path, b, f"b{i}.npz"))
    wrong_counter = np.ones((1, 512), np.int32)
    wrong_counter[0, 3] = 10
    with pytest.raises(ValueError):      # voxel 9 has overflow pairs but not 8 + 9 pairs
        _read_state(_state(tmp_path, {}, "c.npz", counter=wrong_counter))
    with pytest.raises(ValueError):      # a map that takes no label pairs
        _read_state(_state(tmp_path, {}, "d.npz"), labels=False)
