"""CPU: pin `oracle.numpy_semantic_grid`, the plain per-voxel restatement that tests/test_gpu_semantic_edges.py judges
the kernels of b2v_semantic.cu with, to the reference rather than to those kernels:

(1) the committed dumps of the UNMODIFIED compiled reference (tests/golden/semantic_T0.npz, semantic_assoc_T0.npz),
    field by field, with the bounds tests/test_gpu_semantic.py uses for the same comparison;
(2) the reference's own known-answer tests (cpp/test_volumetric_voxel_semantic.py:20-229);
(3) the census of the edge scenes: each reaches the case it is built for;
(4) when oracle/_ref/libref_semantic.so is built: the oracle against the compiled reference, live, after every step
    of every edge scene the reference's harness can express, edits and read-outs included.

Limits.  No committed golden contains an edit (merge_segments, remove_*), so without the compiled reference those
rules are tied to it only by the header lines the oracle's docstring cites; (4) is where they meet the reference
itself.  The 8-slot eviction is the kernel's own rule: the reference keeps every label, so scenes with more than 8
labels in a voxel are compared with the reference up to the first eviction only (the overflow count says when)."""

import inspect
import os

import numpy as np
import pytest

import oracle
from tests import _semantic_scenes as SC
from tests._util import GOLDEN, sort_dump

KINDS = {"vote": "voting", "prob": "probabilistic"}
DUMP_FIELDS = ("keys", "count", "pos_sum", "col_sum", "object_id", "class_id", "aux", "lab_obj", "lab_cls")


def _replay_T0(tag):
    g = np.load(os.path.join(GOLDEN, "semantic_T0.npz"))
    G = oracle.numpy_semantic_grid(float(g["voxel_size"]), KINDS[tag])
    G.set_depth_threshold(float(g[f"{tag}_depth_threshold"]))
    G.set_depth_decay_rate(float(g[f"{tag}_depth_decay_rate"]))
    for i in range(int(g["n_frames"])):
        G.integrate(*[g[f"{tag}_{n}_{i}"] for n in ("points", "colors", "cls", "inst", "depths")])
    return g, G


def _rows(v):
    a = np.concatenate([v["points"], v["colors"].astype(np.float64), v["class_ids"][:, None].astype(np.float64),
                        v["object_ids"][:, None].astype(np.float64), v["confidences"][:, None].astype(np.float64)], 1)
    return a[np.lexsort((a[:, 2], a[:, 1], a[:, 0]))]


@pytest.mark.parametrize("tag", ["vote", "prob"])
def test_oracle_reproduces_the_reference_dump_and_read_out(tag, capsys):
    g, G = _replay_T0(tag)
    d = G.dump()
    for k in DUMP_FIELDS[:7 if tag == "vote" else 9]:      # a voting voxel has no label slots
        assert np.array_equal(d[k], g[f"{tag}_{k}"]), k
    assert G.label_overflows == 0
    ref_lp, ref_conf = g[f"{tag}_lab_logp"], g[f"{tag}_confidence"]
    if tag == "vote":
        assert np.array_equal(d["confidence"], ref_conf)
    else:
        # evidence: bit-exact except where glibc's expf (not correctly rounded) and the float64-rounded exp disagree by
        # one ulp on a depth-decay weight - a handful of the ~10^5 observations (as tests/test_gpu_semantic.py)
        fin = np.isfinite(ref_lp)
        assert np.array_equal(np.isfinite(d["lab_logp"]), fin)
        ndiff = int((d["lab_logp"][fin] != ref_lp[fin]).sum())
        assert ndiff <= max(2, fin.sum() // 1000), ndiff
        assert np.allclose(d["lab_logp"][fin], ref_lp[fin], rtol=1e-6, atol=0)
        assert np.allclose(d["confidence"], ref_conf, rtol=2e-6, atol=1e-9)
        with capsys.disabled():
            print(f"\n  oracle vs reference (Bayesian): {ndiff} of {int(fin.sum())} evidences and "
                  f"{int((d['confidence'] != ref_conf).sum())} of {int((g['prob_count'] > 0).sum())} confidences "
                  "differ in the last bit")
    v = G.get_voxels(2, 0.4)
    ref = {k: g[f"{tag}_voxels_{k}"] for k in ("points", "colors", "class_ids", "object_ids", "confidences")}
    # a Bayesian voxel whose confidence sits within float rounding of 0.4 may flip (as tests/test_gpu_semantic.py)
    if len(v["points"]) == len(ref["points"]):
        a, b = _rows(v), _rows(ref)
        assert np.array_equal(a[:, :8], b[:, :8])
        assert np.allclose(a[:, 8], b[:, 8], rtol=2e-6, atol=0)
        assert tag == "prob" or np.array_equal(a[:, 8], b[:, 8])
    else:
        assert tag == "prob" and abs(len(v["points"]) - len(ref["points"])) <= 2


@pytest.mark.parametrize("tag", ["vote", "prob"])
def test_oracle_reproduces_the_reference_association(tag):
    """The integrator's loop body (associate with carving -> remap -> integrate) over the 4 frames of
    tests/golden/semantic_assoc_T0.npz.  New object ids are handed out in ascending instance order here and in
    block-iteration order in the reference, so ids are compared through the bijection the maps define."""
    from pyslam_b200 import remap_instance_ids
    from pyslam_b200 import synthetic as S
    g = np.load(os.path.join(GOLDEN, "semantic_assoc_T0.npz"))
    G = oracle.numpy_semantic_grid(float(g["voxel_size"]), KINDS[tag])
    G.set_depth_threshold(10.0)
    K = g["K"]
    phi = {-1: -1, 0: 0}
    for i in range(int(g["n_frames"])):
        d, c, T = g[f"depth_{i}"], g[f"color_{i}"], g[f"Tcw_{i}"]
        cls_img, inst_img = g[f"class_image_{i}"], g[f"instance_image_{i}"]
        h, w = d.shape
        m = G.assign_object_ids_to_instance_ids(K, w, h, T, float(g["param_depth_max"]), float(g["param_depth_min"]),
                                                cls_img, inst_img, d, float(g["param_depth_threshold"]),
                                                bool(g["param_do_carving"]), float(g["param_min_vote_ratio"]),
                                                int(g["param_min_votes"]))
        ref = dict(zip(g[f"{tag}_map_inst_{i}"].tolist(), g[f"{tag}_map_obj_{i}"].tolist()))
        assert sorted(m) == sorted(ref), (i, m, ref)
        for k, ro in ref.items():
            assert phi.setdefault(ro, m[k]) == m[k], (i, k, ro, m[k], phi)
        obj_img = remap_instance_ids(inst_img, m)
        Twc = S.inv_T(T)
        valid = (d > 0) & (d < float(g["max_depth"]))
        z = d[valid].astype(np.float64)
        rows, cols = np.where(valid)
        x, y = (cols - K[2]) * z * (1.0 / K[0]), (rows - K[3]) * z * (1.0 / K[1])
        pw = np.stack([x * Twc[r, 0] + y * Twc[r, 1] + z * Twc[r, 2] + Twc[r, 3] for r in range(3)],
                      axis=1).astype(np.float32)
        G.integrate(pw, (c[valid] / 255.0).astype(np.float32), cls_img[valid], obj_img[valid], d[valid])
    assert len(set(phi.values())) == len(phi)
    assert G.next_object_id == int(g[f"{tag}_next_object_id"])
    dmp = G.dump()
    assert np.array_equal(dmp["keys"], g[f"{tag}_keys"])
    # carving compares float depths against the image: a voxel within rounding of the threshold may flip
    same = dmp["count"] == g[f"{tag}_count"]
    assert int((~same).sum()) <= 4, int((~same).sum())
    lut = np.vectorize(lambda o: phi.get(int(o), -12345))
    occ = same & (g[f"{tag}_count"] > 0)
    assert np.array_equal(dmp["object_id"][occ], lut(g[f"{tag}_object_id"][occ]))
    assert np.array_equal(dmp["class_id"][occ], g[f"{tag}_class_id"][occ])
    assert np.allclose(dmp["confidence"][occ], g[f"{tag}_confidence"][occ], rtol=2e-6, atol=1e-9)
    assert (g[f"{tag}_object_id"][occ] > 0).sum() > 200


def _one_voxel(kind, voxel, cls, inst, depths=None, points=None):
    G = oracle.numpy_semantic_grid(voxel, kind)
    n = len(cls)
    G.integrate(np.zeros((n, 3)) if points is None else points, np.zeros((n, 3), np.uint8), np.array(cls, np.int32),
                np.array(inst, np.int32), None if depths is None else np.array(depths, np.float32))
    return G.get_voxels(1, 0.0)


def test_reference_kats_hold_for_the_oracle():
    base = 0.10536051565782628
    v = _one_voxel("voting", 0.1, [1, 2], [1, 2])                         # :20-36 label switch, confidence 0.5
    assert list(v["object_ids"]) == [2] and list(v["class_ids"]) == [2]
    assert v["confidences"][0] == pytest.approx(0.5, abs=1e-3)
    v = _one_voxel("probabilistic", 0.1, [5, 5, 5, 6], [1, 1, 1, 2])      # :39-55 majority
    assert (v["object_ids"][0], v["class_ids"][0]) == (1, 5) and v["confidences"][0] > 0.5
    v = _one_voxel("probabilistic", 0.1, [7, 8], [3, 4], [1.0, 20.0])     # :58-76 depth decay
    assert (v["object_ids"][0], v["class_ids"][0]) == (3, 7) and v["confidences"][0] > 0.5
    v = _one_voxel("voting", 0.1, [10, 20], [101, 202], points=np.array([[0.0, 0, 0], [0.2, 0, 0]]))  # :79-97
    pairs = sorted(zip(map(tuple, v["points"]), v["object_ids"], v["class_ids"]))
    assert [p[1:] for p in pairs] == [(101, 10), (202, 20)]
    v = _one_voxel("probabilistic", 0.1, [5] * 12 + [6], [1] * 12 + [2])  # :100-120 strong majority
    assert (v["object_ids"][0], v["class_ids"][0]) == (1, 5) and v["confidences"][0] > 0.7
    for kind, seed, maj, noise, labels, bound in (("probabilistic", 0, 50, 5, ((111, 11), (222, 12)), 0.75),
                                                  ("voting", 1, 30, 3, ((210, 21), (220, 22)), None)):   # :123-185
        rng = np.random.default_rng(seed)
        tot = maj + noise
        pts = rng.uniform(0.0, 0.05, size=(tot, 3))
        cls = np.array([labels[0][1]] * maj + [labels[1][1]] * noise, np.int32)
        ins = np.array([labels[0][0]] * maj + [labels[1][0]] * noise, np.int32)
        perm = rng.permutation(tot)
        v = _one_voxel(kind, 0.2, cls[perm], ins[perm], points=pts[perm])
        assert (v["object_ids"][0], v["class_ids"][0]) == labels[0]
        if bound:
            assert v["confidences"][0] > bound
        else:
            assert v["confidences"][0] == pytest.approx((maj - noise) / tot, abs=1e-2)
    pc = {(1, 10): 3, (1, 11): 3, (2, 10): 4}                              # :188-229 exact softmax of k * BASE_LOG
    ins = np.concatenate([[o] * k for (o, c), k in pc.items()]).astype(np.int32)
    cls = np.concatenate([[c] * k for (o, c), k in pc.items()]).astype(np.int32)
    perm = np.random.default_rng(42).permutation(10)
    v = _one_voxel("probabilistic", 0.1, cls[perm], ins[perm])
    lp = np.array([4, 3, 3]) * base
    assert (v["object_ids"][0], v["class_ids"][0]) == (2, 10)
    assert v["confidences"][0] == pytest.approx(np.exp(lp[0]) / np.exp(lp).sum(), rel=1e-4, abs=1e-4)


def test_the_oracle_stands_apart_from_the_cuda_library():
    src = inspect.getsource(oracle.numpy_semantic_grid)
    assert "pyslam_b200" not in src and "ctypes" not in src and "C." not in src and "_L." not in src


# ---- (3) census of the edge scenes ----------------------------------------------------------------------------------

def _play(scene, kind, upto=None):
    G = oracle.numpy_semantic_grid(SC.VS, kind)
    if "depth_threshold" in scene:
        G.set_depth_threshold(scene["depth_threshold"])
    if "depth_decay_rate" in scene:
        G.set_depth_decay_rate(scene["depth_decay_rate"])
    maps = []
    for op, kw in scene["steps"][:upto]:
        maps.append(SC.apply(G, "oracle", op, kw))
    return G, maps


def _voxel(G, key):
    k = np.array(key)
    b = G.block_of[tuple((k // 8).tolist())]
    l = k - (k // 8) * 8
    return b, int(l[0] + 8 * l[1] + 64 * l[2])


def test_eviction_scene_evicts_the_slots_it_names():
    G, _ = _play(SC.scene_eviction(), "probabilistic")
    p = SC._pairs(17)
    held = {v: {(s[0], s[1]) for s in G.slots[_voxel(G, v)]} for v in SC.VOX[:5]}
    assert held[SC.VOX[0]] == set(p[:8])                                     # p8 came and went, p2 is back
    assert held[SC.VOX[1]] == set(p[:1] + p[2:8] + p[9:10])                  # slot 1 went twice
    assert held[SC.VOX[2]] == set(p[1:8] + p[16:17])                         # slot 0 went nine times, the argmax stayed
    assert held[SC.VOX[3]] == set(p[:5] + p[6:7] + p[8:10])                  # the two deepest went
    assert held[SC.VOX[4]] == set(p[:8])
    assert G.label_overflows == 2 + 2 + 9 + 2
    assert tuple(G.slots[_voxel(G, SC.VOX[2])][7][:2]) == p[7] and G.obj[_voxel(G, SC.VOX[2])] == p[7][0]
    # the same stream cut at the first eviction ends in the same state
    H, _ = _play(SC.scene_eviction(True), "probabilistic")
    a, b = G.dump(), H.dump()
    assert len(SC.scene_eviction(True)["steps"]) == 2 and all(np.array_equal(a[k], b[k]) for k in a)


def test_softmax_scene_depends_on_the_fold_order():
    """Folding the label evidence in slot (insertion) order gives another float32 confidence than the (object,
    class) order for at least one voxel, and the slots are not inserted in key order."""
    G, _ = _play(SC.scene_softmax_fold(), "probabilistic")
    differs = 0
    for (b, l), slots in G.slots.items():
        assert len(slots) >= 5 and slots != sorted(slots, key=lambda s: (s[0], s[1]))
        total = np.float32(-np.inf)
        for _, _, lp in slots:
            total = G._log_add_exp(total, lp)
        differs += int(G._exp(np.float32(G.ml_logp[b, l] - total)) != G.conf[b, l])
    assert differs >= 1
    assert min(s[0] for sl in G.slots.values() for s in sl) < -1 and max(s[1] for sl in G.slots.values() for s in sl) == SC.IMAX


def test_depth_and_tie_scenes_reach_their_cases():
    sc = SC.scene_depth_threshold()
    V, _ = _play(sc, "voting", 1)
    B, _ = _play(sc, "probabilistic", 1)
    v0, v1 = _voxel(V, SC.VOX[0]), _voxel(V, SC.VOX[1])
    assert (V.obj[v0], V.counter[v0], V.count[v0]) == (1, 1, 3)          # both at-threshold observations ignored
    assert (V.obj[v1], V.counter[v1]) == (2, 1)                          # the at-threshold first observation too
    assert B.slots[_voxel(B, SC.VOX[3])][0][2] == B.BASE_LOG             # full evidence at the threshold
    assert B.slots[_voxel(B, SC.VOX[1])][1][2] < 2 * B.BASE_LOG          # one ulp above it decays
    B, _ = _play(SC.scene_argmax_ties(), "probabilistic")
    assert [int(B.obj[_voxel(B, v)]) for v in SC.VOX[:4]] == [1, 1, 3, 1]
    lp = {v: [s[2] for s in B.slots[_voxel(B, v)]] for v in SC.VOX[:4]}
    assert lp[SC.VOX[1]][0] == lp[SC.VOX[1]][1] and lp[SC.VOX[3]][1] == lp[SC.VOX[3]][2]    # ties at the end


def test_association_scene_reaches_the_resolve_edges():
    from tests import _grid_prep_scenes as E
    for T in E.cam_poses():
        sc = SC.scene_association(T)
        G, maps = _play(sc, "voting")
        first, second = [m for m in maps if m is not None][:2]
        assert first == {0: 0, 5: 1, 6: -1, 7: 4, 8: 51, 9: -1, 11: -1, 12: -1, 13: -1}
        assert second == {0: 0, 5: 1, 6: 1, 7: 4, 8: 51, 9: -1, 11: -1, 12: -1, 13: 1}
        # the first association spent ids on instances 7, 8 and 11; the second on 11 again
        H, _ = _play(sc, "voting", 3)
        assert H.next_object_id == 53 and _play(sc, "voting", 4)[0].next_object_id == 54
        # carving removed exactly the voxel one ulp in front of the threshold
        before, _ = _play(sc, "voting", 2)
        assert int((before.count > 0).sum()) - int((H.count > 0).sum()) == 1
        nc, _ = _play(SC.scene_association(T, carving=False), "voting", 3)
        assert int((nc.count > 0).sum()) == int((before.count > 0).sum())


def test_positions_only_and_confidence_scenes_reach_their_cases():
    sc = SC.scene_positions_only_first()
    G, _ = _play(sc, "probabilistic", 1)
    v = _voxel(G, SC.VOX[0])
    assert G.count[v] == 2 and G.ml_logp[v] == -np.inf and v not in G.slots and G.obj[v] == -1
    G, _ = _play(sc, "probabilistic", 2)
    assert G.count[v] == 5 and (G.obj[v], G.cls[v]) == (5, 3) and len(G.slots[v]) == 2
    assert len(_play(SC.scene_positions_only_first(many_blocks=True), "voting", 1)[0].keys) > 16
    G, _ = _play(SC.scene_confidence_threshold(), "voting")
    assert sorted(G.confidence()[G.count > 0].tolist()) == [0.25, 0.5, 0.5, 0.75, 1.0]
    G, _ = _play(SC.scene_counter_walk(), "voting", 4)
    v = _voxel(G, SC.VOX[0])
    assert (G.obj[v], G.counter[v], G.count[v]) == (2, 1, 6)             # 3 -> 2 -> 1 -> 0: flipped on the third call
    G, _ = _play(SC.scene_counter_walk(), "voting", 3)
    assert (G.obj[v], G.counter[v]) == (1, 1)


# ---- (4) live against the compiled reference ------------------------------------------------------------------------

@pytest.mark.skipif(not oracle.have_ref_semantic(), reason="compiled reference (oracle/_ref) not built")
@pytest.mark.parametrize("kind", ["voting", "probabilistic"])
def test_oracle_matches_the_compiled_reference_on_the_edge_scenes(kind):
    tag = "vote" if kind == "voting" else "prob"
    for name, sc in SC.scenes().items():
        if not sc.get("ref_ok", True):
            continue
        G = oracle.numpy_semantic_grid(SC.VS, kind)
        R = oracle.RefSemanticGrid(SC.VS, kind)
        oracle.RefSemanticGrid.set_next_object_id(1)
        for t in (G, R):
            t.set_depth_threshold(sc.get("depth_threshold", 5.0 if tag == "prob" else 10.0))
            t.set_depth_decay_rate(sc.get("depth_decay_rate", 0.07))
        phi = {-1: -1, 0: 0}
        for op, kw in sc["steps"]:
            m, r = SC.apply(G, "oracle", op, kw), SC.apply(R, "ref", op, kw)
            if G.label_overflows:       # past the first eviction the reference holds more labels than 8 slots
                break
            if m is not None:           # new ids come in another order: compare through the bijection
                assert sorted(m) == sorted(r), (name, m, r)
                for k, ro in r.items():
                    assert phi.setdefault(ro, m[k]) == m[k], (name, k, m, r)
            if op == "assign" and len(phi) > 2:
                continue                # dumps hold ids of both orders: the maps above are the comparison
            a, b = G.dump(), sort_dump(R.dump_blocks(8))
            for k in DUMP_FIELDS[:7 if tag == "vote" else 9]:
                assert np.array_equal(a[k], b[k]), (name, op, k)
            if tag == "prob":
                fin = np.isfinite(b["lab_logp"])
                assert np.allclose(a["lab_logp"][fin], b["lab_logp"][fin], rtol=1e-6, atol=0), (name, op)
            assert np.allclose(a["confidence"], b["confidence"], rtol=2e-6, atol=1e-9), (name, op)
            for bb in sc.get("boxes", []):
                x, y = _rows(G.get_voxels_in_bb(bb, 1, 0.0)), _rows(R.get_voxels_in_bb(bb, 1, 0.0))
                assert x.shape == y.shape and np.array_equal(x[:, :8], y[:, :8]), (name, op)
            for c in sc.get("cams", []):
                args = (c["W"], c["H"], c["Tcw"], c["depth_max"], c["depth_min"], 1, 0.0)
                x = _rows(G.get_voxels_in_camera_frustrum(c["K"], *args))
                y = _rows(R.get_voxels_in_camera_frustrum(np.array(c["K"], np.float32), *args))
                assert x.shape == y.shape and np.array_equal(x[:, :8], y[:, :8]), (name, op)
