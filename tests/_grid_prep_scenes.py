"""Scene builders shared by tests/test_gpu_grid_prep_edges.py and tests/test_grid_prep_oracles_cpu.py: small
deterministic inputs that drive the point-average grid (b2v_grid.cu) and the frame preparation (b2v_prep.cu) to their
edges, each with the census that proves the scene reaches the case it is built for.

Grid scenes whose voxels take more than two points use coordinates with few significant bits (multiples of 2^-12
below 2^3 in magnitude, at most 2^9 points per voxel) and dyadic colours, so every float32 sum is exact in any order
and the kernels' atomics must give the oracle's values exactly.  Voxels with non-dyadic inputs hold at most two points:
two-term float sums commute."""

import numpy as np

f32 = np.float32
Q = 2.0 ** -12          # coordinate quantum of the exact scenes
VS_EXACT = 2.0 ** -6    # exact inverse voxel size (64)
VS_REF = 0.015          # the reference's default voxel size: float32(1 / 0.015) rounds


def dyadic_points(rng, n, lo, hi):
    """n points, each coordinate a multiple of 2^-12 in [lo, hi)."""
    return (rng.integers(int(lo / Q), int(hi / Q), size=(n, 3)) * Q).astype(f32)


def dyadic_colors(rng, n):
    return (rng.integers(0, 256, size=(n, 3)) / 256.0).astype(f32)


def cap_per_voxel(points, keys, cap, *extra):
    """Keep at most `cap` points of each voxel (the first ones in input order)."""
    _, inv = np.unique(keys, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    order = np.argsort(inv, kind="stable")
    rank = np.empty(len(inv), np.int64)
    starts = np.r_[0, np.flatnonzero(np.diff(inv[order])) + 1]
    rank[order] = np.arange(len(inv)) - np.repeat(starts, np.diff(np.r_[starts, len(inv)]))
    keep = rank < cap
    return (points[keep],) + tuple(e[keep] for e in extra)


def voxel_counts(keys):
    return np.unique(keys, axis=0, return_counts=True)[1]


# ---------------------------------------------------------------------------------------------------------------------
# point-average grid: integrate / get_voxels / remove_low_count_voxels
# ---------------------------------------------------------------------------------------------------------------------

def exact_batches(seed=0):
    """Voxel size 2^-6: batches of dyadic points with dyadic float colours, in the order the test integrates them.
      warp_one_block   32 consecutive points (one warp) in one block, several voxels
      alternating      lanes alternate between two blocks of opposite sign
      full_block       one point in every voxel of block (-1, -1, -1)
      dense            clusters around the origin: mixed-sign keys, counts from 1 up to about 40
      hot              one voxel with 300 points (the maximum count)"""
    rng = np.random.default_rng(seed)
    out = []
    base = np.array([0.5, -0.5, 0.25], np.float64)
    out.append(("warp_one_block", (base + rng.integers(0, 2 ** 9, (32, 3)) * Q).astype(f32)))
    a = np.array([3 * 8 / 64 + 0.01, 0.02, 0.03]), np.array([-3 * 8 / 64 + 0.01, -0.02, 0.03])
    alt = np.stack([a[i % 2] for i in range(64)])
    alt = np.floor(alt / Q) * Q + rng.integers(0, 32, (64, 3)) * Q
    out.append(("alternating", alt.astype(f32)))
    l = np.arange(512)
    full = np.stack([l % 8, (l // 8) % 8, l // 64], 1) - 8
    out.append(("full_block", ((full + 0.5) / 64).astype(f32)))
    centers = dyadic_points(rng, 40, -0.6, 0.6)
    dense = centers[rng.integers(0, 40, 4000)] + rng.integers(-48, 48, (4000, 3)) * Q
    out.append(("dense", dense.astype(f32)))
    out.append(("hot", (np.array([-0.75, 1.5, -2.0]) + rng.integers(0, 64, (300, 3)) * Q).astype(f32)))
    return [(name, p, dyadic_colors(rng, len(p))) for name, p in out]


def far_points(seed=1, vs=VS_EXACT):
    """Points whose voxel keys lie around +-2^20 on every axis, at most two per voxel."""
    rng = np.random.default_rng(seed)
    k = (2 ** 20 + rng.integers(-20, 20, (600, 3))) * rng.choice([-1, 1], (600, 3))
    p = ((k + rng.random((600, 3))) * vs).astype(f32)
    keys = np.floor(p * (f32(1) / f32(vs))).astype(np.int64)
    return cap_per_voxel(p, keys, 2)[0]


def edge_points_ref_voxel(seed=2, vs=VS_REF):
    """Voxel size 0.015: points within one float32 ulp of voxel edges, where float32(x * inv_vs) rounds across the
    edge; at most two points per voxel (the coordinates are not dyadic)."""
    rng = np.random.default_rng(seed)
    inv = f32(1) / f32(vs)
    k = rng.integers(-300, 300, (6000, 3))
    edge = (k / np.float64(inv)).astype(f32)
    step = rng.integers(-2, 3, (6000, 3))
    p = edge.copy()
    for s in (-2, -1, 1, 2):
        m = step == s
        x = edge[m]
        for _ in range(abs(s)):
            x = np.nextafter(x, f32(np.inf if s > 0 else -np.inf))
        p[m] = x
    keys = np.floor(p * inv).astype(np.int64)
    return cap_per_voxel(p, keys, 2)[0]


def product_rounding_crossings(points, vs):
    """Coordinates whose float32 product x * inv_vs lands in another voxel than the exact product does."""
    inv = f32(1) / f32(vs)
    p = np.asarray(points, f32)
    return int((np.floor(p * inv) != np.floor(p.astype(np.float64) * np.float64(inv))).sum())


def float64_points(seed=7, vs=0.005):
    """float64 points within float32 rounding of voxel edges (the reference's float64 overload keys them in double);
    at most two points per voxel."""
    rng = np.random.default_rng(seed)
    inv = np.float64(f32(1) / f32(vs))
    k = rng.integers(-400, 400, size=(20000, 3)).astype(np.float64)
    p = k * (1.0 / inv) + rng.choice([-1e-9, 1e-9, 3e-10], size=(20000, 3))
    keys = np.floor(p * inv).astype(np.int64)
    return cap_per_voxel(p, keys, 2)[0]


# ---------------------------------------------------------------------------------------------------------------------
# box and frustum queries, carve
# ---------------------------------------------------------------------------------------------------------------------

# (min_x, min_y, min_z, max_x, max_y, max_z): the first box has negative min keys that are not block edges
# (-13, -29, -5) and positive max keys; the second has its min keys on negative block edges (-16, -8, -32) and
# negative max keys (-2, -1, -17)
BOXES = (
    np.array([-13 / 64 + 5 * Q, -29 / 64 + 3 * Q, -5 / 64 + 7 * Q, 27 / 64 + 9 * Q, 11 / 64 + Q, 37 / 64 + 2 * Q]),
    np.array([-16 / 64, -8 / 64, -32 / 64, -2 / 64 + 3 * Q, -Q, -17 / 64 + 5 * Q]),
)


def box_probe_points(bb):
    """One point per voxel (so each voxel mean is the point itself): on each face, 2^-12 inside and outside it, in the
    voxel just outside the key bounds, and inside.  The other two coordinates step through the box interior."""
    lo, hi = bb[:3], bb[3:]
    mid = np.floor(((lo + hi) / 2) / Q) * Q
    span = np.floor((hi - lo) * 64).astype(int)
    pts = []
    for a in range(3):
        cands = [lo[a], lo[a] + Q, lo[a] - Q, lo[a] - 1 / 64, hi[a], hi[a] - Q, hi[a] + Q, hi[a] + 1 / 64, mid[a]]
        for j, c in enumerate(cands):
            p = mid.copy()
            for b in range(3):
                if b != a:
                    p[b] = lo[b] + ((j * 3 + b) % max(span[b] - 1, 1) + 1) / 64 + 0.5 / 64
                    p[b] = np.floor(p[b] / Q) * Q
            p[a] = c
            pts.append(p)
    return np.array(pts).astype(f32)


def box_census(points, bb, vs=VS_EXACT):
    """Per box: points on each of the 6 faces, points in the voxel just outside the key bounds, and whether the min
    keys are negative non-multiples of 8 (where trunc division and floor division pick different blocks)."""
    p = np.asarray(points, np.float64)
    lo, hi = bb[:3], bb[3:]
    inv = np.float64(f32(1) / f32(vs))
    kmin, kmax = np.floor(lo * inv), np.floor(hi * inv)
    k = np.floor(np.asarray(points, f32) * f32(inv))
    return dict(on_min_face=[int((p[:, a] == lo[a]).sum()) for a in range(3)],
                on_max_face=[int((p[:, a] == hi[a]).sum()) for a in range(3)],
                outside_keys=int(np.any((k < kmin) | (k > kmax), axis=1).sum()),
                min_key_not_block_edge=[bool(m < 0 and m % 8 != 0) for m in kmin],
                min_key_negative_block_edge=[bool(m < 0 and m % 8 == 0) for m in kmin])


# cameras with exact projections: power-of-two focal lengths, integer principal points, axis-aligned rotations
CAM_W, CAM_H = 32, 24
CAM_K = (64.0, 32.0, 16.0, 12.0)
DEPTH_MIN, DEPTH_MAX = 0.5, 2.0


def cam_poses():
    T0 = np.eye(4)
    T0[:3, 3] = [0.125, -0.0625, 0.25]
    T1 = np.zeros((4, 4))
    T1[:3, :3] = [[0, 1, 0], [0, 0, -1], [-1, 0, 0]]   # world -> camera axis permutation with sign flips
    T1[:3, 3] = [-0.25, 0.5, 0.125]
    T1[3, 3] = 1
    return T0, T1


def cam_point(T, u, v, z):
    """World point that the camera T (world -> camera) projects to pixel (u, v) at depth z."""
    fx, fy, cx, cy = CAM_K
    pc = np.array([(u - cx) * z / fx, (v - cy) * z / fy, z])
    return np.linalg.solve(T[:3, :3], pc - T[:3, 3])


def frustum_probe_points(T):
    """One point per voxel at u = 0 (in), u = W (out), v = H (out), u = -2^-6 (out), v = H - 2^-5 (in),
    depth = depth_min / depth_max (in), depth just outside them and behind the camera (out), plus interior points."""
    cases = [(0.0, 5.0, 1.0), (CAM_W, 5.0, 1.0), (7.0, CAM_H, 1.0), (-1 / 64, 6.0, 1.0), (9.0, CAM_H - 1 / 32, 1.0),
             (CAM_W - 1 / 64, 7.0, 1.0), (11.0, 0.0, 1.0), (3.0, 3.0, DEPTH_MIN), (4.0, 20.0, DEPTH_MAX),
             (5.0, 9.0, DEPTH_MIN - 1 / 64), (6.0, 9.0, DEPTH_MAX + 1 / 64), (8.0, 8.0, -1.0), (12.0, 12.0, -0.5)]
    for i in range(40):
        cases.append((1.0 + (i * 7) % 30, 1.0 + (i * 5) % 22, 0.75 + (i % 5) * 0.25))
    return np.array([cam_point(T, *c) for c in cases]).astype(f32)


def frustum_census(points, T):
    """Projections of the probe points (exact by construction): how many land exactly on each bound."""
    import oracle
    ok, u, v, depth = oracle.numpy_grid.project(points, CAM_K, CAM_W, CAM_H, T, DEPTH_MAX, DEPTH_MIN)
    return dict(u0_in=int((ok & (u == 0)).sum()), uW=int((u == CAM_W).sum()), vH=int((v == CAM_H).sum()),
                dmin_in=int((ok & (depth == f32(DEPTH_MIN))).sum()), dmax_in=int((ok & (depth == f32(DEPTH_MAX))).sum()),
                behind=int((depth < 0).sum()), inside=int(ok.sum()))


CARVE_THR = 0.25


def carve_scene(T):
    """(points, depth image): one point per voxel and per pixel.  Image depths 0, -1, NaN, +inf, -inf (never carve),
    a voxel exactly at image - thr (kept) and one float32 ulp nearer (carved), projections at u = 5.75 and
    u = W - 2^-6 (the truncated column decides), voxels well in front (carved) and behind the surface (kept)."""
    img = np.zeros((CAM_H, CAM_W), f32)
    pts = []

    def add(u, v, z, d):
        img[int(v), int(u)] = d
        pts.append(cam_point(T, u, v, z))

    for i, d in enumerate([0.0, -1.0, np.nan, np.inf, -np.inf]):
        add(2.5 + i, 2.5, 1.0, d)
    add(2.5, 5.5, 1.25, 1.5)                                   # depth == 1.5 - 0.25: kept
    add(3.5, 5.5, float(np.nextafter(f32(1.25), f32(0))), 1.5)   # one ulp nearer: carved
    add(4.5, 5.5, 1.0, 1.5)                                    # well in front: carved
    add(5.5, 5.5, 1.5, 1.5)                                    # on the surface: kept
    add(6.5, 5.5, 1.75, 1.5)                                   # behind the surface: kept
    add(5.75, 8.5, 1.0, 1.5)                                   # column 5 carves; column 6 (rounding) holds 0
    img[8, 6] = 0.0
    add(CAM_W - 1 / 64, 10.5, 1.0, 1.5)                        # last column
    add(7.5, CAM_H - 1 / 32, 1.0, 1.5)                         # last row
    for i in range(30):
        u, v = 8.5 + (i % 20), 12.5 + (i // 20) * 3
        add(u, v, 1.0 + (i % 3) * 0.25, 1.0 + (i % 4) * 0.25)
    return np.array(pts).astype(f32), img


def carve_census(points, img, T):
    """Which probe reaches which branch of the carve: per-pixel depth class of the voxels in the frustum."""
    import oracle
    ok, u, v, depth = oracle.numpy_grid.project(points, CAM_K, CAM_W, CAM_H, T, DEPTH_MAX, DEPTH_MIN)
    u, v, depth = u[ok], v[ok], depth[ok]
    d = img[v.astype(int), u.astype(int)]
    with np.errstate(invalid="ignore"):
        thr = d - f32(CARVE_THR)
        return dict(at_threshold=int((depth == thr).sum()),
                    ulp_nearer=int((depth == np.nextafter(thr, f32(0))).sum()),
                    carved=int(((d > 0) & np.isfinite(d) & (depth < thr)).sum()),
                    special=int((~np.isfinite(d) | (d <= 0)).sum()),
                    nan=int(np.isnan(d).sum()), posinf=int((d == np.inf).sum()), neginf=int((d == -np.inf).sum()),
                    truncation_matters=int(((u % 1 >= 0.5) & (np.floor(u) != np.rint(u))).sum()),
                    last_column=int((u.astype(int) == CAM_W - 1).sum()))


# ---------------------------------------------------------------------------------------------------------------------
# fused RGBD front end
# ---------------------------------------------------------------------------------------------------------------------

RGBD_K = (64.0, 64.0, 20.0, 15.0)
RGBD_H, RGBD_W = 30, 40


def rgbd_frames(seed=3, n=3):
    """Depths that are multiples of 2^-6 in [0.5, 2.5) (a plane with a raised box: depth discontinuities for the
    shadow filter), colours 0 or 255 (dyadic after / 255), poses with identity rotation and dyadic translation."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        d = (64 + rng.integers(0, 3, (RGBD_H, RGBD_W))).astype(np.float64) / 64
        d[8:20, 10 + i:25 + i] = (120 + rng.integers(0, 3, (12, 15))) / 64
        d[0, :5] = 0.0
        c = (rng.integers(0, 2, (RGBD_H, RGBD_W, 3)) * 255).astype(np.uint8)
        Twc = np.eye(4)
        Twc[:3, 3] = [0.125 * i, -0.25, 0.0625 * i]
        out.append((d.astype(f32), c, Twc))
    return out


def rgbd_points(depth, color, K, Twc, max_depth=np.inf, min_depth=0.0):
    """depth2pointcloud + Twc in the order of b2v_grid.cu's rgbd_point (float64, then float32)."""
    fx, fy, cx, cy = K
    valid = (depth > min_depth) & (depth < max_depth)
    rows, cols = np.nonzero(valid)
    z = depth[valid].astype(np.float64)
    x = ((cols - cx) * z) * (1.0 / fx)
    y = ((rows - cy) * z) * (1.0 / fy)
    R, t = Twc[:3, :3], Twc[:3, 3]
    p = np.stack([((x * R[a, 0] + y * R[a, 1]) + z * R[a, 2]) + t[a] for a in range(3)], 1).astype(f32)
    return p, (color[valid] / 255.0).astype(f32)


# ---------------------------------------------------------------------------------------------------------------------
# shadow filter
# ---------------------------------------------------------------------------------------------------------------------

def positive_deltas(d, dx, dy):
    d = np.asarray(d, f32)
    with np.errstate(invalid="ignore"):
        v = np.concatenate([np.abs(d[dy:] - d[:-dy]).ravel(), np.abs(d[:, dx:] - d[:, :-dx]).ravel()])
        return np.sort(v[v > 0])


def _plane(rng, H, W):
    return (1.0 + rng.integers(0, 64, (H, W)) / 1024).astype(f32)


def shadow_scenes():
    """name -> (depth, dx, dy).  Each name states the case it reaches; test_grid_prep_oracles_cpu checks it."""
    rng = np.random.default_rng(11)
    S = {}
    S["count0_constant"] = (np.full((5, 6), 1.5, f32), 2, 2)
    one = np.ones((2, 3), f32)
    one[0, 1] = 1.5
    S["count1"] = (one, 2, 1)
    two = np.ones((2, 4), f32)
    two[0, 1], two[0, 2] = 1.5, 3.0
    S["count2"] = (two, 3, 1)
    S["tiny_3x3_d1"] = (_plane(rng, 3, 3), 1, 1)
    S["tiny_3x3_dmax"] = (_plane(rng, 3, 3), 2, 2)
    for name, parity in (("odd", 1), ("even", 0)):
        for s in range(100):
            d = _plane(np.random.default_rng(100 + s), 17, 23)
            d[4:9, 6:14] += f32(0.75)
            if len(positive_deltas(d, 2, 2)) % 2 == parity:
                S[f"{name}_count"] = (d, 2, 2)
                break
    # even count whose two middle deltas differ (1 and 2): the delta 7.5 lies above 3 * 1.4826 * 1.5 and below
    # 3 * 1.4826 * 2, so it is filtered only when the median averages both middle elements
    mid = np.stack([np.full(12, 10, f32), 10 + np.array([0, 1, 1, 1, 1, 2, 2, 2, 2, 7.5, 1, 0], f32)]).astype(f32)
    S["even_middles_differ"] = (mid, 11, 1)
    eq = np.ones((9, 12), f32)
    eq[:, 1::2] = 1.5
    S["all_equal"] = (eq, 1, 2)
    ties = (1.0 + 0.25 * rng.integers(0, 3, (40, 50))).astype(f32)
    ties[rng.random((40, 50)) < 0.02] = 6.0
    S["ties"] = (ties, 1, 1)
    rows = np.where(np.arange(32)[:, None] % 2 == 0, 2.0, 3.0 + rng.integers(0, 200, (32, 1)) / 1024).astype(f32)
    p2 = np.repeat(rows, 20, axis=1)
    p2[5, 3] = 40.0
    S["pass2"] = (p2, 3, 1)      # all positive deltas in [1, 1.25): top 11 bits shared
    rows = np.where(np.arange(32)[:, None] % 2 == 0, 2.0, 3.0 + rng.integers(0, 400, (32, 1)) * 2.0 ** -22).astype(f32)
    p3 = np.repeat(rows, 20, axis=1)
    p3[7, 9] = 40.0
    S["pass3"] = (p3, 3, 1)      # deltas 1 + k 2^-22, k < 512: top 22 bits shared
    sub = (rng.integers(0, 8, (20, 24)) * 2.0 ** -140).astype(f32)
    sub[3:6, 4:9] = f32(1e-38)
    S["subnormal"] = (sub, 2, 2)
    inf = _plane(rng, 24, 30)
    inf[rng.random((24, 30)) < 0.05] = np.inf
    inf[10:14, 10:20] = 3.0
    S["posinf"] = (inf, 2, 2)
    many_inf = np.full((8, 9), np.inf, f32)
    many_inf[::2, ::3] = 1.0
    S["median_inf"] = (many_inf, 1, 1)
    nan = _plane(rng, 24, 30)
    nan[rng.random((24, 30)) < 0.05] = np.nan
    nan[3:9, 5:12] = 2.5
    S["nan"] = (nan, 2, 2)
    nz = _plane(rng, 16, 16)
    nz[::3, ::2] = 0.0
    nz[1::3, ::2] = -0.0
    S["negzero"] = (nz, 2, 2)
    wide = _plane(rng, 13, 61)
    wide[:, 30:] += f32(0.5)
    S["dx_W-1_dy_H-1"] = (wide, 60, 12)
    S["d3"] = (wide, 3, 3)
    big = _plane(rng, 480, 640)
    big[100:300, 200:400] += f32(0.625)
    big[rng.random((480, 640)) < 0.01] = 0.0
    S["vga"] = (big, 2, 2)
    return S


# ---------------------------------------------------------------------------------------------------------------------
# remap
# ---------------------------------------------------------------------------------------------------------------------

REMAP_SIZES = ((1, 1), (1, 7), (61, 83), (480, 640))


def remap_maps(kind, H, W, seed=0):
    """(map_x, map_y) float32 [H,W] of one adversarial family."""
    rng = np.random.default_rng(seed)
    u = lambda lo, hi: rng.uniform(lo, hi, (H, W)).astype(f32)   # noqa: E731
    if kind == "uniform":
        return u(-5, W + 5), u(-5, H + 5)
    if kind == "ties64":            # odd multiples of 1/64: map * 32 is a half-integer
        return ((2 * rng.integers(-64, 64 * W + 64, (H, W)) + 1) / 64).astype(f32), \
            ((2 * rng.integers(-64, 64 * H + 64, (H, W)) + 1) / 64).astype(f32)
    if kind == "half":              # nearest ties
        return (rng.integers(-4, W + 4, (H, W)) + 0.5).astype(f32), (rng.integers(-4, H + 4, (H, W)) + 0.5).astype(f32)
    if kind == "border":            # a band around each border
        bx = np.where(rng.random((H, W)) < 0.5, rng.uniform(-1.5, 0.5, (H, W)), rng.uniform(W - 1.5, W + 0.5, (H, W)))
        by = np.where(rng.random((H, W)) < 0.5, rng.uniform(-1.5, 0.5, (H, W)), rng.uniform(H - 1.5, H + 0.5, (H, W)))
        return bx.astype(f32), by.astype(f32)
    mx, my = u(-5, W + 5), u(-5, H + 5)
    pick = rng.random((H, W)) < 0.4
    if kind == "huge":
        vals = np.array([4e4, -4e4, 1e5, -1e5, 1e9, -1e9, 3.4e38, -3.4e38], f32)
        mx[pick] = rng.choice(vals, int(pick.sum()))
        pick_y = rng.random((H, W)) < 0.4
        my[pick_y] = rng.choice(vals, int(pick_y.sum()))
    elif kind == "inf":
        mx[pick] = rng.choice([np.inf, -np.inf], int(pick.sum()))
        my[rng.random((H, W)) < 0.3] = -np.inf
    elif kind == "nan_x":
        mx[pick] = np.nan
    elif kind == "nan_y":
        my[pick] = np.nan
    elif kind == "nan_both":
        mx[pick] = np.nan
        my[pick | (rng.random((H, W)) < 0.3)] = np.nan
    else:
        raise ValueError(kind)
    return mx, my


REMAP_KINDS = ("uniform", "ties64", "half", "border", "huge", "inf", "nan_x", "nan_y", "nan_both")
