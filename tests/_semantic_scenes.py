"""Scenes shared by tests/test_gpu_semantic_edges.py and tests/test_semantic_oracle_cpu.py: small scripted call
sequences that drive the semantic grids (b2v_semantic.cu) through the edges of the label state machines, and
`apply`, which plays one step on a GPU grid, on `oracle.numpy_semantic_grid` or on `oracle.RefSemanticGrid`.

A scene is a dict: `steps` [(op, kwargs)], optional `depth_threshold` / `depth_decay_rate`, optional `boxes` and
`cams` to query after every step, `ref_ok` False when the compiled reference's harness cannot express it (it has no
colourless integrate).  Voxel size 2^-6 m; coordinates are multiples of 2^-12 and colours of 2^-8, so every sum is
exact; observations of different voxels are interleaved in the input, so a voxel's order is the stable sort's."""

import numpy as np

from tests import _grid_prep_scenes as E

f32 = np.float32
VS = E.VS_EXACT
IMAX = 2 ** 31 - 1
# voxel keys in six blocks, negative and far keys included
VOX = [(0, 0, 0), (-1, -1, -1), (9, -17, 3), (-8, 0, 7), (100, -100, 50), (7, 7, 7), (-64, 33, -9), (3, 4, 5)]


def cam(T, depth_max=E.DEPTH_MAX, depth_min=E.DEPTH_MIN):
    return dict(K=E.CAM_K, W=E.CAM_W, H=E.CAM_H, Tcw=T, depth_max=depth_max, depth_min=depth_min)


def stream(per_voxel):
    """{voxel key: [(object, class, depth), ...]} -> integrate kwargs with the voxels' observations interleaved round
    robin.  The j-th observation of a voxel lies at key + (4 + j % 8, 4 + (3 j) % 8, 8) / 16 voxels."""
    pts, cols, cls, ins, dep = [], [], [], [], []
    j = 0
    while any(j < len(o) for o in per_voxel.values()):
        for k, obs in per_voxel.items():
            if j < len(obs):
                o, c, d = obs[j]
                pts.append((np.array(k) + np.array([4 + j % 8, 4 + (3 * j) % 8, 8]) / 16.0) / 64.0)
                cols.append(np.array([j % 7, (2 * j) % 5, 1 + j % 3]) / 8.0)
                cls.append(c)
                ins.append(o)
                dep.append(d)
        j += 1
    return dict(points=np.array(pts, f32).reshape(-1, 3), colors=np.array(cols, f32).reshape(-1, 3),
                class_ids=np.array(cls, np.int32), instance_ids=np.array(ins, np.int32), depths=np.array(dep, f32))


def split(kw, at):
    """The integrate step `kw` as two steps cut at observation `at`."""
    return [("integrate", {k: v[:at] for k, v in kw.items()}), ("integrate", {k: v[at:] for k, v in kw.items()})]


def _pairs(n, first=0):
    return [(10 + first + i, 100 + first + i) for i in range(n)]


def _reps(pairs, reps, d=1.0):
    return [(o, c, d) for (o, c), r in zip(pairs, reps) for _ in range(r)]


def eviction_streams():
    """Per voxel: observations that fill the 8 slots with chosen evidence, then further distinct pairs.
      VOX[0]  argmax in slot 0 (3 observations), the weakest pair in slot 2; the 9th pair evicts slot 2, then the evicted
              pair returns and evicts its successor
      VOX[1]  10 pairs seen once each: all candidates tie, the first non-argmax slot (1) goes both times
      VOX[2]  argmax in slot 7; 17 distinct pairs in all: every candidate ties, so slot 0 goes each time
      VOX[3]  8 pairs with distinct depth-decayed evidence: the 9th evicts the deepest one (slot 5), the 10th the next
      VOX[4]  exactly 8 pairs: no eviction"""
    p = _pairs(17)
    s = {}
    s[VOX[0]] = _reps(p[:8], [3, 2, 1, 2, 2, 2, 2, 2]) + [(*p[8], 1.0), (*p[2], 1.0), (*p[2], 1.0)]
    s[VOX[1]] = _reps(p[:10], [1] * 10)
    s[VOX[2]] = _reps(p[:8], [1] * 7 + [3]) + _reps(p[8:17], [1] * 9)
    depths = [1.5, 2.0, 1.75, 2.25, 1.0, 3.5, 2.5, 3.0]
    s[VOX[3]] = [(*p[i], depths[i]) for i in range(8)] + [(*p[8], 1.5), (*p[9], 1.5)]
    s[VOX[4]] = _reps(p[:8], [2, 1, 1, 1, 1, 1, 1, 1])
    return s


def scene_eviction(split_at_first_eviction=False):
    kw = stream(eviction_streams())
    steps = [("integrate", kw)]
    if split_at_first_eviction:
        seen, at = {}, None
        vk = np.floor(kw["points"] * 64).astype(int)
        for i in range(len(vk)):
            pairs = seen.setdefault(tuple(vk[i]), set())
            pairs.add((int(kw["instance_ids"][i]), int(kw["class_ids"][i])))
            if len(pairs) == 9:
                at = i
                break
        steps = split(kw, at)
    return dict(steps=steps, depth_threshold=1.5, depth_decay_rate=1.0)


def scene_softmax_fold():
    """Up to 8 labels per voxel with unequal evidence, inserted in an order that is not the (object, class) order and
    with negative ids and INT32_MAX in both positions."""
    labels = [(5, 2), (-3, 7), (IMAX, 1), (0, 0), (5, -2), (-3, -9), (2, IMAX), (-IMAX, 4)]
    reps = [6, 5, 5, 8, 3, 7, 6, 1]      # evidence whose float32 log-sum depends on the order of the fold
    s = {VOX[0]: _reps(labels, reps), VOX[1]: _reps(labels[:5][::-1], reps[:5]),
         VOX[2]: [(o, c, 1.0 + 0.25 * i) for i, (o, c) in enumerate(labels)] + _reps(labels[2:6], [2, 2, 2, 2], 2.0),
         VOX[5]: _reps(labels[::-1], [1, 7, 1, 5, 1, 3, 4, 4][::-1])}
    return dict(steps=[("integrate", stream(s))], depth_threshold=1.0, depth_decay_rate=0.5)


def scene_depth_threshold():
    """Depths exactly at the threshold 1.5, one float32 ulp below and above it, and +inf under an infinite threshold
    (the second call).  Voting ignores depth >= threshold; Bayesian gives full evidence at depth <= threshold."""
    t = f32(1.5)
    lo, hi = float(np.nextafter(t, f32(0))), float(np.nextafter(t, f32(2)))
    s = {VOX[0]: [(1, 1, lo), (2, 2, 1.5), (2, 2, 1.5)],
         VOX[1]: [(1, 1, 1.5), (2, 2, lo), (2, 2, hi)],
         VOX[2]: [(1, 1, hi), (1, 1, 1.5), (2, 2, lo), (2, 2, 2.0)],
         VOX[3]: [(1, 1, 1.5), (2, 2, 2.5), (2, 2, 1.5)]}
    inf = {VOX[4]: [(1, 1, np.inf), (2, 2, 3.0e38), (2, 2, np.inf)], VOX[0]: [(2, 2, np.inf)]}
    return dict(steps=[("integrate", stream(s)), ("set_depth_threshold", dict(v=np.inf)), ("integrate", stream(inf))],
                depth_threshold=1.5, depth_decay_rate=2.0)


def scene_argmax_ties():
    """Equal evidence keeps the earlier label; the overtaken argmax's own evidence is read again when it returns."""
    a, b, c = (1, 1, 1.0), (2, 2, 1.0), (3, 3, 1.0)
    s = {VOX[0]: [a, b, b, a, a], VOX[1]: [a, b], VOX[2]: [b, a, a, b, c, c, c, b], VOX[3]: [a, b, c, c, b, a, a]}
    return dict(steps=[("integrate", stream(s))])


def _positions(keys, reps=2):
    s = stream({k: [(0, 0, 1.0)] * reps for k in keys})
    return dict(points=s["points"])


def scene_positions_only_first(clear_first=False, many_blocks=False):
    """A colourless call (count > 0, no label state), then a labelled call on the same voxels and on fresh ones.
    `many_blocks`: the first call touches 27 blocks, so a grid created with 8 grows inside it."""
    keys = list(VOX[:4])
    if many_blocks:
        keys += [(16 * x, 16 * y, 16 * z) for x in (-1, 0, 1) for y in (-1, 0, 1) for z in (-1, 0, 1)][:23]
    lab = stream({k: [(4, 2, 1.0), (5, 3, 1.0), (5, 3, 1.0)] for k in keys[:3] + [VOX[5]]})
    steps = [("integrate", _positions(keys)), ("integrate", lab), ("integrate", _positions(keys[1:5], 1)),
             ("integrate", stream({k: [(-1, -1, 1.0), (5, 3, 1.0)] for k in keys}))]
    if clear_first:
        warm = stream({k: _reps(_pairs(9), [1] * 9) for k in keys})
        steps = [("integrate", warm), ("clear", {})] + steps
    return dict(steps=steps, ref_ok=False)


def scene_labelled_after_edits():
    """A labelled call after each edit: reset voxels start again; a voxel merged onto a valid id holds one slot with
    evidence 0; one merged onto an invalid id holds none (count still positive)."""
    a, b, c = (1, 1, 1.0), (2, 2, 1.0), (3, 1, 1.0)
    first = {VOX[0]: [a, a, b], VOX[1]: [b, b, a], VOX[2]: [c, c, c, a], VOX[3]: [a], VOX[4]: [b, c, c], VOX[5]: [c, b]}
    again = stream({k: [b, a, a, c] for k in VOX[:6]})
    steps = [("integrate", stream(first))]
    for op, kw in (("remove_segment", dict(object_id=1)), ("merge_segments", dict(a=7, b=2)),
                   ("merge_segments", dict(a=-7, b=3)), ("remove_low_count_voxels", dict(min_count=6)),
                   ("remove_low_confidence_segments", dict(min_confidence=1)), ("merge_segments", dict(a=2, b=1))):
        steps += [(op, kw), ("integrate", again)]
    return dict(steps=steps)


def scene_edit_ids():
    """merge_segments(a, a), merge_segments(a, -1) and remove_segment(-1): -1 is the id of every empty voxel and of
    voxels labelled with an invalid instance."""
    s = {VOX[0]: [(1, 1, 1.0), (1, 1, 1.0), (2, 1, 1.0)], VOX[1]: [(-1, 4, 1.0), (-1, 4, 1.0)],
         VOX[2]: [(2, 2, 1.0), (3, 2, 1.0), (2, 2, 1.0)], VOX[3]: [(-1, -1, 1.0)], VOX[4]: [(0, 0, 1.0)]}
    more = stream({k: [(1, 1, 1.0), (9, 4, 1.0)] for k in VOX[:6]})
    return dict(steps=[("integrate", stream(s)), ("merge_segments", dict(a=1, b=1)), ("integrate", more),
                       ("merge_segments", dict(a=6, b=-1)), ("integrate", more), ("remove_segment", dict(object_id=-1)),
                       ("merge_segments", dict(a=-1, b=9)), ("remove_segment", dict(object_id=-1)),
                       ("integrate", more), ("merge_segments", dict(a=0, b=0))])


def scene_low_confidence():
    """remove_low_confidence_segments takes an int: 0 removes nothing, 1 everything below confidence 1."""
    s = {VOX[0]: [(1, 1, 1.0)] * 3, VOX[1]: [(1, 1, 1.0), (1, 1, 1.0), (2, 2, 1.0)], VOX[2]: [(2, 2, 1.0)],
         VOX[3]: [(-1, 3, 1.0)] * 2, VOX[4]: [(1, 1, 1.0), (2, 2, 1.0)]}
    return dict(steps=[("integrate", stream(s)), ("remove_low_confidence_segments", dict(min_confidence=0)),
                       ("integrate", _positions(VOX[:2], 1)), ("remove_low_confidence_segments", dict(min_confidence=1)),
                       ("integrate", stream(s)), ("remove_low_confidence_segments", dict(min_confidence=2))],
                ref_ok=False)


def scene_counter_walk():
    """The voting counter walks 3 -> 0 over four calls and the label flips on the call that reaches zero; the
    confidence min(1, counter / count) after remove_low_count_voxels (reset, then counted again)."""
    a, b = (1, 1, 1.0), (2, 2, 1.0)
    steps = [("integrate", stream({VOX[0]: [a, a, a], VOX[1]: [a, a], VOX[2]: [a]}))]
    for _ in range(4):
        steps.append(("integrate", stream({VOX[0]: [b], VOX[1]: [b], VOX[2]: [b, b]})))
    steps += [("remove_low_count_voxels", dict(min_count=7)), ("integrate", stream({k: [b, a, a] for k in VOX[:3]})),
              ("integrate", stream({k: [a] * 5 for k in VOX[:3]}))]
    return dict(steps=steps)


def scene_extreme_ids():
    ids = [IMAX, 0, -1, -2, -IMAX, 1]
    s = {}
    for n, k in enumerate(VOX[:6]):
        s[k] = [(ids[(n + i) % 6], ids[(n + 2 * i + 1) % 6], 1.0) for i in range(7)]
    return dict(steps=[("integrate", stream(s)), ("integrate", stream(s)), ("remove_segment", dict(object_id=IMAX)),
                       ("merge_segments", dict(a=IMAX, b=-IMAX)), ("integrate", stream(s))])


# ---- instance -> object association --------------------------------------------------------------------------------

def _labelled_voxels(T, rows):
    """rows (u, v, z, object, class, observations) -> integrate kwargs, one voxel per row at the camera's pixel."""
    pts, cls, ins = [], [], []
    for u, v, z, o, c, n in rows:
        pts += [E.cam_point(T, u, v, z)] * n
        cls += [c] * n
        ins += [o] * n
    n = len(pts)
    return dict(points=np.array(pts).astype(f32), colors=np.full((n, 3), 0.5, f32), class_ids=np.array(cls, np.int32),
                instance_ids=np.array(ins, np.int32))


def scene_association(T, depth=True, carving=True):
    """One frame.  Image instances by pixel column block: see `rows`.  min_votes 4, min_vote_ratio 0.5.
      instance 5   objects 1 and 2 with 2 votes each: tie, the lower id wins; total == min_votes, ratio == 0.5 exactly
      instance 6   3 votes: below min_votes
      instance 7   object 3 x2, object 4 x3, one pending voxel: total 6, winner 4 at ratio 0.5
      instance 8   4 pending voxels only: a new object id, assigned to them
      instance 0   unlabelled voxels take object 0; the map says 0 whatever the votes
      instance 9   in the image, no voxel votes
      instance 11  pending voxels, but the votes fail the ratio: the new id is spent, the voxels stay unlabelled
      instance 13  objects 1, 2, 3 with one vote each: in the second association (min_votes 3, min_vote_ratio
                   float32(1) / float32(3)) total == min_votes and the ratio equals the bound, the lowest id wins
      instance 12  the depth cases below
      class -1 pixels, class mismatches, instance -1 pixels, image depth 0 / NaN, voxels in front of (carved) and
      behind the surface."""
    cls_img = np.full((E.CAM_H, E.CAM_W), 1, np.int32)
    inst_img = np.full((E.CAM_H, E.CAM_W), -1, np.int32)
    dep_img = np.full((E.CAM_H, E.CAM_W), 1.0, f32)
    rows = []

    def put(col, row, inst, obj, cls=1, z=1.0, n=1, img_cls=1, d=1.0):
        inst_img[row, col], cls_img[row, col], dep_img[row, col] = inst, img_cls, d
        rows.append((col + 0.5, row + 0.5, z, obj, cls, n))

    for i, o in enumerate((1, 1, 2, 2)):
        put(1 + i, 1, 5, o)
    for i in range(3):
        put(1 + i, 3, 6, 1)
    for i, o in enumerate((3, 3, 4, 4, 4, -1)):
        put(1 + i, 5, 7, o)
    for i in range(4):
        put(1 + i, 7, 8, -1, n=1 + i % 2)
    for i, o in enumerate((-1, -1, 2, 2, 2)):
        put(1 + i, 9, 0, o)
    inst_img[11, 1:4] = 9
    for i, o in enumerate((-1, 1, 2, 3, 4)):
        put(1 + i, 13, 11, o)
    put(10, 1, 5, 1, img_cls=-1)                 # pixel without class
    put(11, 1, 5, 1, cls=2)                      # class mismatch
    put(12, 1, -1, 1)                            # pixel without instance
    put(13, 1, 5, -1, cls=-1, img_cls=-1)        # voxel without class
    for i, o in enumerate((1, 2, 3)):
        put(1 + i, 15, 13, o)
    put(14, 1, 12, 1, d=0.0)
    put(15, 1, 12, 1, d=np.nan)
    put(16, 1, 12, 1, z=0.75, d=1.0)             # in front of the surface by 0.25 = threshold: kept, votes
    put(17, 1, 12, 1, z=float(np.nextafter(f32(0.75), f32(0))), d=1.0)   # one ulp nearer: carved (votes without carving)
    put(18, 1, 12, 1, z=1.25, d=1.0)             # behind by exactly the threshold: votes
    put(19, 1, 12, 1, z=float(np.nextafter(f32(1.25), f32(2))), d=1.0)   # one ulp farther: skipped
    assoc = dict(cam=cam(T), class_image=cls_img, instance_image=inst_img, depth_image=dep_img if depth else None,
                 depth_threshold=0.25, do_carving=carving, min_vote_ratio=0.5, min_votes=4)
    third = dict(assoc, min_vote_ratio=float(f32(1.0) / f32(3.0)), min_votes=3)
    return dict(steps=[("set_next_object_id", dict(v=50)), ("integrate", _labelled_voxels(T, rows)), ("assign", assoc), ("assign", third),
                       ("integrate", _labelled_voxels(T, rows[:12])), ("assign", assoc)], cams=[cam(T)])


# ---- read-outs and carve on bounds -----------------------------------------------------------------------------------

def _probe_labels(p):
    """Every probe point labelled, and every second one observed a second time under another object."""
    n = len(p)
    i = np.arange(n)
    cols = E.dyadic_colors(np.random.default_rng(1), n)
    return dict(points=np.concatenate([p, p[::2]]), colors=np.concatenate([cols, cols[::2]]),
                class_ids=np.concatenate([1 + i % 3, (1 + i % 3)[::2]]).astype(np.int32),
                instance_ids=np.concatenate([10 + i % 4, (11 + i % 4)[::2]]).astype(np.int32))


def scene_box(bb):
    """Box faces exactly on voxel means (each probe voxel holds one point, or the same point twice)."""
    return dict(steps=[("integrate", _probe_labels(E.box_probe_points(bb)))], boxes=[bb])


def scene_frustum(T):
    """Image borders and depth_min / depth_max at equality, then carve with depths at image - threshold."""
    pts, img = E.carve_scene(T)
    return dict(steps=[("integrate", _probe_labels(E.frustum_probe_points(T))), ("integrate", _probe_labels(pts)),
                       ("carve", dict(cam=cam(T), depth_image=img, depth_threshold=E.CARVE_THR)),
                       ("integrate", _probe_labels(pts[::3]))], cams=[cam(T)])


def scene_confidence_threshold():
    """Voting confidences k / n with float32-exact quotients (n a power of two) to query with min_confidence equal to
    them: 1/2, 1/4, 3/4, 1."""
    a, b = (1, 1, 1.0), (2, 2, 1.0)
    s = {VOX[0]: [a, a, a, b], VOX[1]: [a] * 5 + [b] * 3, VOX[2]: [a] * 7 + [b], VOX[3]: [a] * 4,
         VOX[4]: [a, a, a, b, b, a, a, a]}
    return dict(steps=[("integrate", stream(s))], confidences=(0.25, 0.5, 0.75, 1.0))


# ---- input variants and the randomised stream --------------------------------------------------------------------------

def random_stream(seed=17, n=50000, calls=4, first=0):
    """`calls` integrate steps of n / 4 points each: dyadic points on a shell around the origin (about 6 per voxel),
    6 classes, 12 instances, 20 % label noise with -1 among it, depths on both sides of the threshold 2.0."""
    rng = np.random.default_rng(seed + first)
    out = []
    for _ in range(calls):
        m = n // 4
        d = rng.normal(size=(m, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        p = np.round((d * (0.35 + 0.02 * rng.random((m, 1))) + [0.03, -0.06, 0.01]) / E.Q) * E.Q
        side = (p[:, 0] > 0).astype(np.int64) + 2 * (p[:, 1] > 0) + 4 * (p[:, 2] > 0)
        noise = rng.random(m) < 0.2
        cls = np.where(noise, rng.integers(-1, 6, m), side % 6).astype(np.int32)
        ins = np.where(noise, rng.integers(-1, 12, m), side + 4 * (p[:, 0] > 0.2)).astype(np.int32)
        dep = (rng.integers(64, 192, m) / 64.0).astype(f32)
        out.append(("integrate", dict(points=p.astype(f32), colors=E.dyadic_colors(rng, m), class_ids=cls,
                                      instance_ids=ins, depths=dep)))
    return out


def scene_random(T):
    pts = random_stream()[0][1]["points"]
    img = np.full((E.CAM_H, E.CAM_W), 0.55, f32)
    edits = [("merge_segments", dict(a=3, b=7)), ("remove_segment", dict(object_id=0)),
             ("remove_low_count_voxels", dict(min_count=3)),
             ("carve", dict(cam=cam(T, 2.0, 0.05), depth_image=img, depth_threshold=0.05)),
             ("remove_low_confidence_segments", dict(min_confidence=1))]
    box = np.concatenate([np.quantile(pts, 0.2, axis=0), np.quantile(pts, 0.8, axis=0)]).astype(np.float64)
    return dict(steps=random_stream() + edits + random_stream(calls=2, first=100), depth_threshold=2.0,
                depth_decay_rate=0.8, boxes=[box], cams=[cam(T, 2.0, 0.05)], rtol=True)


def input_variants():
    """(name, integrate kwargs): point and colour dtypes, absent instance ids and depths, n = 1, one 100 000-point run
    in one voxel next to 4 096 points with a voxel each."""
    rng = np.random.default_rng(5)
    base = random_stream(seed=23, n=8000, calls=1)[0][1]
    u8 = rng.integers(0, 2, base["colors"].shape).astype(np.uint8) * 255
    out = [("f32", base), ("f64", dict(base, points=base["points"].astype(np.float64))), ("u8", dict(base, colors=u8)),
           ("no_instances", dict(base, instance_ids=None)), ("no_depths", dict(base, depths=None)),
           ("no_instances_no_depths_f64_u8", dict(points=base["points"].astype(np.float64), colors=u8,
                                                  class_ids=base["class_ids"])),
           ("one_point", {k: v[:1] for k, v in base.items()})]
    n = 100000
    run = dict(points=(np.array([0.5, -0.25, 0.125]) + rng.integers(0, 64, (n, 3)) * E.Q).astype(f32),
               colors=E.dyadic_colors(rng, n), class_ids=rng.integers(0, 3, n).astype(np.int32),
               instance_ids=rng.integers(0, 3, n).astype(np.int32), depths=(rng.integers(64, 192, n) / 64.0).astype(f32))
    g = np.stack(np.meshgrid(np.arange(16), np.arange(16), np.arange(16), indexing="ij"), -1).reshape(-1, 3) - 8
    own = dict(points=((g + 0.5) / 64).astype(f32), colors=E.dyadic_colors(rng, len(g)),
               class_ids=rng.integers(0, 3, len(g)).astype(np.int32),
               instance_ids=rng.integers(0, 3, len(g)).astype(np.int32))
    return out + [("one_long_run", run), ("one_voxel_each", own)]


def rgbd_labels(seed=9):
    """Class and object images for E.rgbd_frames()."""
    rng = np.random.default_rng(seed)
    cls = rng.integers(-1, 4, (E.RGBD_H, E.RGBD_W)).astype(np.int32)
    obj = (cls * 10 + rng.integers(0, 2, cls.shape)).astype(np.int32)
    return cls, obj


# ---- playing a step ------------------------------------------------------------------------------------------------------

def apply(t, backend, op, kw):
    """Play step (op, kw) on `t`: backend "gpu" (a pyslam_b200 grid), "oracle" (numpy_semantic_grid) or "ref"
    (RefSemanticGrid).  Returns the instance map of an association, else None."""
    if op == "integrate":
        a = [kw["points"], kw.get("colors"), kw.get("class_ids"), kw.get("instance_ids"), kw.get("depths")]
        if backend == "ref" and a[1] is not None and a[1].dtype == np.uint8:
            a[1] = a[1].astype(f32) * (f32(1.0) / f32(255.0))      # voxel_data.h:82-85
        if backend == "ref" and len(a[0]) == 0:
            return None
        t.integrate(*a)
    elif op == "assign":
        c = kw["cam"]
        rest = (kw["class_image"], kw["instance_image"], kw["depth_image"], kw["depth_threshold"], kw["do_carving"],
                kw["min_vote_ratio"], kw["min_votes"])
        if backend == "gpu":
            return t.assign_object_ids_to_instance_ids(_frustrum(c), *rest)
        K = np.array(c["K"], f32) if backend == "ref" else c["K"]
        return t.assign_object_ids_to_instance_ids(K, c["W"], c["H"], c["Tcw"], c["depth_max"], c["depth_min"], *rest)
    elif op == "carve":
        c = kw["cam"]
        if backend == "gpu":
            t.carve(_frustrum(c), kw["depth_image"], kw["depth_threshold"])
        else:
            K = np.array(c["K"], f32) if backend == "ref" else c["K"]
            t.carve(K, c["W"], c["H"], c["Tcw"], c["depth_max"], c["depth_min"], kw["depth_image"],
                    kw["depth_threshold"])
    elif op == "merge_segments":
        t.merge_segments(kw["a"], kw["b"])
    elif op in ("set_depth_threshold", "set_next_object_id"):
        getattr(t, op)(kw["v"])
    else:
        getattr(t, op)(**kw)
    return None


def _frustrum(c):
    from pyslam_b200 import CameraFrustrum
    return CameraFrustrum(*c["K"], c["W"], c["H"], c["Tcw"], depth_max=c["depth_max"], depth_min=c["depth_min"])


def scenes():
    """name -> scene, for the scenes that need no special grid."""
    T0, T1 = E.cam_poses()
    return {
        "eviction": scene_eviction(),
        "eviction_split": scene_eviction(True),
        "softmax_fold": scene_softmax_fold(),
        "depth_threshold": scene_depth_threshold(),
        "argmax_ties": scene_argmax_ties(),
        "positions_only_first": scene_positions_only_first(),
        "positions_only_after_clear": scene_positions_only_first(clear_first=True),
        "labelled_after_edits": scene_labelled_after_edits(),
        "edit_ids": scene_edit_ids(),
        "low_confidence": scene_low_confidence(),
        "counter_walk": scene_counter_walk(),
        "extreme_ids": scene_extreme_ids(),
        "association": scene_association(T0),
        "association_rotated": scene_association(T1),
        "association_no_depth": scene_association(T0, depth=False),
        "association_no_carving": scene_association(T1, carving=False),
        "box0": scene_box(E.BOXES[0]),
        "box1": scene_box(E.BOXES[1]),
        "frustum0": scene_frustum(T0),
        "frustum1": scene_frustum(T1),
        "confidence_threshold": scene_confidence_threshold(),
    }
