"""The Bayesian grid with an overflow label store (b2v_sgrid_set_label_overflow), shared by
tests/test_semantic_labels_cpu.py and tests/test_gpu_semantic_labels.py: the reference's unbounded label map restated
on top of `oracle.numpy_semantic_grid`, and scenes whose voxels collect more than 8 (object, class) pairs.

`UnboundedSemanticGrid` is `numpy_semantic_grid` without its 8-slot eviction: a voxel keeps every pair in insertion
order (`_observe_bayes` appends below MAX_LABELS), and the confidence already folds every pair in ascending
(object, class) order, the std::map order of voxel_data_semantic.h:561-570, 607-624.  Its `dump(K)` shows K pairs
per voxel (None: the most any voxel holds, at least 8)."""

import numpy as np

import oracle
from tests import _semantic_scenes as SC

f32 = np.float32


class UnboundedSemanticGrid(oracle.numpy_semantic_grid):
    MAX_LABELS = 1 << 62

    def __init__(self, voxel_size, kind="probabilistic"):
        super().__init__(voxel_size, kind)

    def max_pairs(self):
        return max((len(s) for s in self.slots.values()), default=0)

    def dump(self, K=None):
        K = max(8, self.max_pairs()) if K is None else K
        order = np.lexsort((self.keys[:, 2], self.keys[:, 1], self.keys[:, 0]))
        nb = len(order)
        lab_obj = np.full((nb, 512, K), -1, np.int32)
        lab_cls = np.full((nb, 512, K), -1, np.int32)
        lab_logp = np.full((nb, 512, K), -np.inf, np.float32)
        aux = np.zeros_like(self.counter)
        for (b, l), slots in self.slots.items():
            aux[b, l] = len(slots)
            for k, (o, c, lp) in enumerate(sorted(slots, key=lambda s: (s[0], s[1]))[:K]):
                lab_obj[b, l, k], lab_cls[b, l, k], lab_logp[b, l, k] = o, c, lp
        d = dict(keys=self.keys.astype(np.int32), count=self.count.astype(np.int32), pos_sum=self.pos,
                 col_sum=self.col, object_id=self.obj, class_id=self.cls, confidence=self.conf, aux=aux,
                 lab_obj=lab_obj, lab_cls=lab_cls, lab_logp=lab_logp)
        return {k: a[order].copy() for k, a in d.items()}


def pairs(n, first=0):
    """n distinct (object, class) pairs whose object order is not their insertion order."""
    return [(10 + ((first + i) * 7) % 61, 100 + (first + i) % 3) for i in range(n)]


def many_pair_streams(n):
    """Per voxel, n distinct pairs (n > 8):
      VOX[0]  each once: every pair ties
      VOX[1]  uneven repetitions: the argmax changes while the chain fills
      VOX[2]  each once, then the last pair three more times: the argmax moves to a pair held in a chunk
      VOX[3]  depth-decayed evidence on both sides of the threshold 1.5
      VOX[4]  the pairs in reverse order
      VOX[5]  8 pairs: no chain"""
    p = pairs(n)
    s = {SC.VOX[0]: [(o, c, 1.0) for o, c in p],
         SC.VOX[1]: [(o, c, 1.0) for i, (o, c) in enumerate(p) for _ in range(1 + (5 * i) % 3)],
         SC.VOX[2]: [(o, c, 1.0) for o, c in p] + [(*p[-1], 1.0)] * 3,
         SC.VOX[3]: [(o, c, 1.0 + 0.125 * (i % 9)) for i, (o, c) in enumerate(p)],
         SC.VOX[4]: [(o, c, 1.0) for o, c in p[::-1]],
         SC.VOX[5]: [(o, c, 1.0) for o, c in p[:8]] * 2}
    return s


def scene_many_pairs(n):
    """The streams of `many_pair_streams(n)` cut in two calls, the edits that release chains (remove_segment of a
    voxel's argmax object, merge_segments, remove_low_count_voxels, remove_low_confidence_segments), each followed by a
    labelled call that builds chains again on other voxels, then clear and the first call once more."""
    kw = SC.stream(many_pair_streams(n))
    again = SC.stream({k: [(o, c, 1.0) for o, c in pairs(n, 3)] for k in SC.VOX[4:8]})
    late = pairs(n)[-1][0]
    steps = SC.split(kw, len(kw["points"]) // 3)
    for op, a in (("remove_segment", dict(object_id=late)), ("merge_segments", dict(a=5, b=pairs(n)[0][0])),
                  ("remove_low_count_voxels", dict(min_count=n + 2)),
                  ("remove_low_confidence_segments", dict(min_confidence=1))):
        steps += [(op, a), ("integrate", again)]
    steps += [("clear", {}), ("integrate", kw)]
    return dict(steps=steps, depth_threshold=1.5, depth_decay_rate=1.0)


def churn_stream(seed=31, n=50000, calls=4, first=0):
    """`SC.random_stream` with object ids that churn: every point's instance id is drawn from 48, so a voxel of the
    shell (about 6 points per call) collects a new pair with almost every observation."""
    out = []
    for op, kw in SC.random_stream(seed=seed, n=n, calls=calls, first=first):
        rng = np.random.default_rng(seed + 1000 + first + len(out))
        kw = dict(kw, instance_ids=rng.integers(-1, 48, len(kw["points"])).astype(np.int32))
        out.append((op, kw))
    return out


def scene_churn(T):
    sc = SC.scene_random(T)
    n_edits = len(sc["steps"]) - 6
    edits = sc["steps"][4:4 + n_edits]
    return dict(sc, steps=churn_stream() + edits + churn_stream(calls=2, first=100))


def chunks_of(n_pairs):
    """Chunks of 8 a voxel with n_pairs pairs holds past its 8 in-voxel slots."""
    return max(0, -(-(n_pairs - 8) // 8))


def census(scene):
    """Play `scene` on the unbounded oracle: (most pairs of a voxel, most chunks of a voxel, chunks in use after every
    step, whether an edit released chunks that a later call needed again)."""
    G = UnboundedSemanticGrid(SC.VS)
    for t in (G,):
        t.set_depth_threshold(scene.get("depth_threshold", 5.0))
        t.set_depth_decay_rate(scene.get("depth_decay_rate", 0.07))
    most, used, reuse, freed = 0, [], False, False
    for op, kw in scene["steps"]:
        before = sum(chunks_of(len(s)) for s in G.slots.values())
        SC.apply(G, "oracle", op, kw)
        now = sum(chunks_of(len(s)) for s in G.slots.values())
        most = max(most, G.max_pairs())
        freed = freed or now < before
        reuse = reuse or (freed and now > before)
        used.append(now)
    return most, chunks_of(most), used, reuse
