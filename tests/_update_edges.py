"""Scene builders for the TSDF update at its per-voxel decision boundaries, shared by
tests/test_gpu_tsdf_update_edges.py and tests/test_update_edges_cpu.py.

Each builder restates in numpy float32 the projection chain the twin (oracle/tsdf_oracle.c) and the update kernels
share (DESIGN §3): the voxel centre h = (float)((double)(vl/2 + vl*x) + unit*L), p = ((E0*h0 + E1*h1) + E2*h2) + E3,
one p += vl*E[:,2] per z step from the unit's z = 0, u_f = (p.x*fx / p.z + cx) + 0.5, lambda and sdf.  It then steps
a pose translation or a depth with float32 ulps until a chosen voxel lands exactly on a boundary:

- margins: u_f / v_f just inside and just outside the 0.0001 margin and the safe_w / safe_h bound (at W = 2208,
  safe_w == W: the right margin collapses);
- truncation: sdf == -tau (not live) against nextafter(-tau, +inf), and sdf * inv_tau == 1 against the float below;
- single live voxel: one valid pixel whose footprint is narrower than a voxel, so exactly one voxel of the frame
  takes it, at every run position k and in every warp of its block; and the same frame one ulp past truncation;
- exact division: non-rigid poses whose depth row puts p.z below 2^-100 for every voxel, or across one 4-voxel run.

A frame is (depth f32 [H, W], colour u8 [H, W, 3], Tcw float64 [4, 4]); the frames of a scene share its K."""

from dataclasses import dataclass, field

import numpy as np

f32 = np.float32
MARGIN = f32(0.0001)
DIV_LO = f32(2.0 ** -100)           # b2v_tsdf.cu kDivLo: below it the update's quotients take __fdiv_rn


@dataclass
class Scene:
    name: str
    H: int
    W: int
    K: tuple                 # fx, fy, cx, cy
    voxel_size: float
    sdf_trunc: float
    depth_trunc: float
    stride: int
    unit: int                # volume_unit_resolution the frames are built for (it moves the voxel centres' chain)
    frames: list
    # per frame: (block key, (lx, ly, lz), expected to take the frame) of the voxel the frame is built around
    targets: list = field(default_factory=list)
    # per frame: the emulated value that sits on the boundary, and the constant it is compared with
    values: list = field(default_factory=list)

    def batch(self, frames=None):
        fr = self.frames if frames is None else frames
        return tuple(np.stack([f[k] for f in fr]) for k in range(3))


# ---------------------------------------------------------------------------------------------------------------------
# the projection chain
# ---------------------------------------------------------------------------------------------------------------------

def pose_E(T):
    """The float32 world->camera rows the update reads: (float)Tcw[0:3, :]."""
    return np.asarray(T, np.float64)[..., :3, :].astype(f32)


def project(E, K, W, H, vs, unit, key, lx, ly, lz):
    """(p.x, p.y, p.z, u_f, v_f, in image) of voxel (lx, ly, lz) of block `key` under the float32 rows E [..., 3, 4],
    in the update's operation order; every array argument broadcasts."""
    S = unit // 8
    key = np.asarray(key, np.int64)
    u = key // S
    sb = key - u * S
    vsf = f32(vs)
    half = f32(vsf * f32(0.5))
    L = float(vs) * unit
    lx, ly, lz = (np.asarray(a, np.int64) for a in (lx, ly, lz))
    h0 = (np.float64(half + vsf * (sb[0] * 8 + lx).astype(f32)) + u[0] * L).astype(f32)
    h1 = (np.float64(half + vsf * (sb[1] * 8 + ly).astype(f32)) + u[1] * L).astype(f32)
    h2 = f32(np.float64(half) + u[2] * L)
    E = np.asarray(E, f32)
    p = [((E[..., r, 0] * h0 + E[..., r, 1] * h1) + E[..., r, 2] * h2) + E[..., r, 3] for r in range(3)]
    es = [E[..., r, 2] * vsf for r in range(3)]
    steps = sb[2] * 8 + lz
    shape = np.broadcast(p[0], p[1], p[2], steps).shape
    p = [np.broadcast_to(x, shape).astype(f32) for x in p]
    steps = np.broadcast_to(steps, shape)
    for s in range(int(steps.max(initial=0))):
        m = s < steps
        for r in range(3):
            p[r] = np.where(m, p[r] + es[r], p[r]).astype(f32)
    fx, fy, cx, cy = (f32(k) for k in K)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        uf = ((p[0] * fx) / p[2] + cx) + f32(0.5)
        vf = ((p[1] * fy) / p[2] + cy) + f32(0.5)
    safe_w, safe_h = f32(W) - MARGIN, f32(H) - MARGIN
    inb = (p[2] > 0) & (uf >= MARGIN) & (uf < safe_w) & (vf >= MARGIN) & (vf < safe_h)
    return p[0], p[1], p[2], uf.astype(f32), vf.astype(f32), inb


def lam(K, uu, vv):
    """Open3D's depth-to-distance multiplier of pixel (uu, vv): sqrtf(xx*xx + yy*yy + 1) with xx = (u - cx) / fx as
    (u - cx) * (1 / fx)."""
    fx, fy, cx, cy = (f32(k) for k in K)
    xx = (np.asarray(uu).astype(f32) - cx) * (f32(1) / fx)
    yy = (np.asarray(vv).astype(f32) - cy) * (f32(1) / fy)
    return np.sqrt((xx * xx + yy * yy) + f32(1)).astype(f32)


def block_update(frame, K, vs, tau, trunc, unit, key):
    """Per voxel of block `key` ([lz, ly, lx]): (live, sdf, t) of one frame as the update decides them."""
    d_img, _, T = frame
    H, W = d_img.shape
    l = np.arange(8)
    _, _, pz, uf, vf, inb = project(pose_E(T), K, W, H, vs, unit, key, l[None, None, :], l[None, :, None],
                                    l[:, None, None])
    uu = np.where(inb, uf, 0).astype(np.int64)
    vv = np.where(inb, vf, 0).astype(np.int64)
    d = np.where(inb, d_img[vv, uu], f32(0))
    with np.errstate(invalid="ignore", over="ignore"):
        sdf = ((d - pz) * lam(K, uu, vv)).astype(f32)
        t = np.minimum(f32(1), sdf * (f32(1) / f32(tau)))
    live = inb & (d > 0) & (d < f32(trunc)) & (sdf > -f32(tau))
    return live, sdf, t


def live_voxels(frame, K, vs, tau, trunc, unit, keys):
    """{block key: sorted flat voxel indices lx + 8 ly + 64 lz} of the voxels of `keys` that take the frame."""
    out = {}
    for k in keys:
        live = block_update(frame, K, vs, tau, trunc, unit, k)[0]
        idx = np.flatnonzero(live.reshape(-1))
        if len(idx):
            out[tuple(int(x) for x in k)] = idx
    return out


def ulp_steps(x, n):
    """The 2n + 1 float32 values from n ulps below x to n ulps above (x finite, not crossing zero)."""
    x = f32(x)
    i = np.arange(-n, n + 1, dtype=np.int64)
    bits = np.int64(np.array(x, f32).view(np.int32))
    return (bits + np.where(x >= 0, i, -i)).astype(np.int32).view(f32)


def _search_translation(T, axis, E_value, want, n=1 << 14):
    """T with its translation component `axis` moved by float32 ulps so that E_value(E [m, 3, 4]) hits `want`.  Where
    the rounding of the sums skips `want` along that axis, the depth component is stepped too."""
    T = T.copy()
    for dz in ulp_steps(np.float64(T[2, 3]), 64)[64:] if axis != 2 else [T[2, 3]]:
        T[2, 3] = float(dz)
        cand = ulp_steps(np.float64(T[axis, 3]), n)
        E = np.repeat(pose_E(T)[None], len(cand), 0)
        E[:, axis, 3] = cand
        hit = np.flatnonzero(E_value(E) == want)
        if len(hit):
            T[axis, 3] = float(cand[hit[np.argmin(np.abs(hit - n))]])
            return T
    raise AssertionError((axis, want))


def _rigid(t):
    T = np.eye(4)
    T[:3, 3] = t
    return T


def _colour(H, W, seed):
    return np.random.default_rng(seed).integers(0, 256, (H, W, 3), dtype=np.uint8)


# ---------------------------------------------------------------------------------------------------------------------
# margins
# ---------------------------------------------------------------------------------------------------------------------

MARGIN_KEY = (1, -1, 3)     # block of the target voxels (z: ~0.5 m in front of the camera)


def margin_values(W, H, K):
    """Per axis, the upper boundary's values: hi_in = the float below safe = n - 0.0001f, hi_out = safe.  (The lower
    margin's are found by margin_scene: near 0.0001, u_f = A + 0.5 with A in (-0.5, -0.25) sums exactly, so u_f is
    a multiple of 2^-25 or coarser and never equals 0.0001f itself; tests/test_update_edges_cpu.py checks every A.)"""
    out = {}
    for axis, n in (("u", W), ("v", H)):
        safe = f32(n) - MARGIN
        out[axis] = dict(hi_in=np.nextafter(safe, f32(0)), hi_out=safe)
    return out


def margin_scene(W, H, unit=16, fx=None, seed=0):
    """8 frames sharing K, one per boundary case: u_f and v_f at the low margin (in, out) and at safe_w / safe_h
    (in, out).  Flat depth tau / 2 behind the target voxel: the target takes the frame exactly when it is in the
    image.  The translation is stepped by ulps until the target's coordinate hits the case's value."""
    vs, tau, trunc = 0.02, 0.08, 4.0
    fx = float(fx or max(80.0, W / 2.2))
    K = (fx, fx, (W - 1) / 2.0, (H - 1) / 2.0)
    key, l = MARGIN_KEY, (3, 5, 2)
    h = project(pose_E(np.eye(4)), K, W, H, vs, unit, key, *l)        # identity pose: p = h
    hx, hy, hz = (float(x) for x in h[:3])
    Z = 0.5
    bounds = margin_values(W, H, K)
    frames, targets, values = [], [], []
    for case in ("u_lo_in", "u_lo_out", "u_hi_in", "u_hi_out", "v_lo_in", "v_lo_out", "v_hi_in", "v_hi_out"):
        axis, side, inside = case[0], case[2:4], case.endswith("_in")
        ai = 0 if axis == "u" else 1
        n = W if axis == "u" else H
        c, f = K[2 + ai], K[ai]
        edge = 0.0 if side == "lo" else float(n)
        off = (edge - 0.5 - c) / f * Z                  # camera-space offset that puts the voxel on the edge
        t = [-hx, -hy, Z - hz]
        t[ai] += off

        def coord(E, ai=ai):
            return project(E, K, W, H, vs, unit, key, *l)[3 + ai]

        T = _rigid(t)
        if side == "lo":
            # the reachable values next to the margin: step the translation and take the neighbours of 0.0001
            cand = ulp_steps(np.float64(T[ai, 3]), 1 << 14)
            E = np.repeat(pose_E(T)[None], len(cand), 0)
            E[:, ai, 3] = cand
            v = coord(E)
            want = v[v >= MARGIN].min() if inside else v[v < MARGIN].max()
        else:
            want = bounds[axis]["hi_in" if inside else "hi_out"]
        T = _search_translation(T, ai, coord, want)
        pz = project(pose_E(T), K, W, H, vs, unit, key, *l)[2]
        d = np.full((H, W), f32(pz + f32(tau / 2)), f32)
        frames.append((d, _colour(H, W, 100 * seed + len(frames)), T))
        targets.append((key, l, inside))
        values.append((case, want, MARGIN if side == "lo" else f32(n) - MARGIN))
    return Scene(f"margins-{W}x{H}-U{unit}", H, W, K, vs, tau, trunc, 4, unit, frames, targets, values)


# ---------------------------------------------------------------------------------------------------------------------
# truncation
# ---------------------------------------------------------------------------------------------------------------------

TRUNC_KEY = (0, 0, 1)


def truncation_scene(unit=16):
    """4 frames sharing K: the target voxel on the optical axis (p.x = p.y = 0 exactly, so its pixel is the integer
    principal point and lambda == 1) with sdf == -tau, sdf == nextafter(-tau, +inf), sdf * inv_tau == 1 and
    sdf * inv_tau == the float below 1.  Flat depth: the translation's z and the depth are stepped by ulps until
    the float32 difference d - p.z is the wanted sdf."""
    vs, tau, trunc = 0.02, 0.08, 4.0
    W, H = 96, 72
    K = (80.0, 80.0, 48.0, 36.0)
    key, l = TRUNC_KEY, (4, 2, 1)
    hx, hy, hz = (float(x) for x in project(pose_E(np.eye(4)), K, W, H, vs, unit, key, *l)[:3])
    tauf, inv = f32(tau), f32(1) / f32(tau)
    below1 = np.nextafter(f32(1), f32(0))
    # (name, value the target's sdf or t must take, whether the target takes the frame, sdf -> compared value).  t
    # just below 1: sdf is a multiple of 2^-26 there and sdf * inv_tau steps by 3 ulps of 1, so a t within 16 ulps
    # under 1 is taken
    cases = (("sdf=-tau", -tauf, False, lambda s: s), ("sdf=next(-tau)", np.nextafter(-tauf, f32(1)), True,
                                                       lambda s: s),
             ("t=1", f32(1), True, lambda s: (s * inv).astype(f32)),
             ("t<1", None, True, lambda s: (s * inv).astype(f32)))
    frames, targets, values = [], [], []
    for name, want, inside, val in cases:
        found = None
        for tz in ulp_steps(f32(0.18 - hz), 4096):
            T = _rigid([float(-hx), float(-hy), float(tz)])
            p = project(pose_E(T), K, W, H, vs, unit, key, *l)
            assert p[0] == 0 and p[1] == 0 and int(p[3]) == 48 and int(p[4]) == 36
            pz = p[2]
            guess = f32(np.float64(pz) + (np.float64(want) if name.startswith("sdf") else 1.0 / np.float64(inv)))
            d = ulp_steps(guess, 4)
            v = val((d - pz).astype(f32))
            hit = np.flatnonzero(v == want) if want is not None else np.flatnonzero((v < 1) & (v >= below1 - f32(2 ** -20)))
            if len(hit):
                found = (T, d[hit[-1]], v[hit[-1]])
                break
        assert found, name
        T, dv, got = found
        frames.append((np.full((H, W), dv, f32), _colour(H, W, 200 + len(frames)), T))
        targets.append((key, l, inside))
        values.append((name, got, -tauf if name.startswith("sdf") else f32(1)))
    return Scene(f"truncation-U{unit}", H, W, K, vs, tau, trunc, 4, unit, frames, targets, values)


# ---------------------------------------------------------------------------------------------------------------------
# single live voxel
# ---------------------------------------------------------------------------------------------------------------------

SINGLE_KEY = (5, -3, 7)
SINGLE_DIR = (0.0137, -0.0091)      # a generic viewing direction: no other voxel centre near the ray


def single_voxel_scene(unit):
    """32 frames sharing K (fx = 2e4: a pixel is 25 um wide at 0.5 m, a voxel 10 mm; tau = 4 mm < half a voxel).
    Frames 2i and 2i + 1 are built around voxel (3, ly, lz) of block SINGLE_KEY with lz = i % 8 (run position
    lz % 4, warp half lz // 4) and ly = 1 or 5 (the other warp half): one valid pixel, the target's, with the surface
    tau / 2 behind the target (exactly that voxel takes the frame), then with the largest depth for which the target
    is one ulp past the truncation bound (no voxel takes it; its block is still touched)."""
    vs, tau, trunc = 0.01, 0.004, 4.0
    W = H = 32
    Z = 0.5
    a, b = SINGLE_DIR
    fx = 2.0e4
    K = (fx, fx, 16.3 - a * fx, 15.7 - b * fx)
    frames, targets, values = [], [], []
    for i in range(16):
        l = (3, 1 if i < 8 else 5, i % 8)
        hx, hy, hz = (float(x) for x in project(pose_E(np.eye(4)), K, W, H, vs, unit, SINGLE_KEY, *l)[:3])
        T = _rigid([a * Z - hx, b * Z - hy, Z - hz])
        _, _, pz, uf, vf, inb = project(pose_E(T), K, W, H, vs, unit, SINGLE_KEY, *l)
        assert inb
        uu, vv = int(uf), int(vf)
        lm = lam(K, uu, vv)
        d_live = f32(pz + f32(tau / 2))
        # the depths around pz - tau / lambda: the last one whose sdf is not above -tau
        cand = ulp_steps(f32(np.float64(pz) - tau / np.float64(lm)), 64)
        live = ((cand - pz) * lm).astype(f32) > -f32(tau)
        k = np.flatnonzero(live)[0]
        assert k > 0 and not live[k - 1]
        for d, inside in ((d_live, True), (cand[k - 1], False)):
            img = np.zeros((H, W), f32)
            img[vv, uu] = d
            frames.append((img, _colour(H, W, 300 + len(frames)), T))
            targets.append((SINGLE_KEY, l, inside))
            values.append(("sdf", ((d - pz) * lm).astype(f32), -f32(tau)))
    return Scene(f"single-voxel-U{unit}", H, W, K, vs, tau, trunc, 1, unit, frames, targets, values)


def warp_and_run(l):
    """(warp of the block's 128 threads, run position k) of voxel l = (lx, ly, lz) in the update kernels."""
    lx, ly, lz = l
    t = lx + 8 * ly + 64 * (lz // 4)
    return t // 32, lz % 4


# ---------------------------------------------------------------------------------------------------------------------
# exact division inside fused groups
# ---------------------------------------------------------------------------------------------------------------------

DIV_T = (0.013, -0.021, 0.96)       # rigid translation: the plane z_cam = 1 runs between voxel z = 1 and z = 2


def division_frames(kind, n=32, seed=0):
    """n rigid frames (kind 'rigid'), or the same poses with every row scaled by 2^-110 ('tiny': p.z < 2^-100 for
    every voxel) or by 2^-100 ('straddle': p.z < 2^-100 exactly where the rigid z_cam < 1, which cuts the runs
    lz = 0..3 of block z = 0 between lz = 1 and lz = 2).  A power-of-two scale keeps p.x / p.z the rigid quotient,
    so the degenerate frames update the voxels the rigid ones see, through __fdiv_rn.  Flat depth 1.03 m and a
    colour image per frame."""
    W, H = 96, 72
    scale = {"rigid": 1.0, "tiny": 2.0 ** -110, "straddle": 2.0 ** -100}[kind]
    out = []
    for i in range(n):
        T = _rigid([DIV_T[0] + 0.0013 * (i % 7), DIV_T[1] - 0.0007 * (i % 5), DIV_T[2]])
        T[:3] *= scale
        out.append((np.full((H, W), f32(1.03), f32), _colour(H, W, 1000 * seed + 17 * i + len(kind)), T))
    return out


DIV_K = (80.0, 80.0, 47.5, 35.5)
DIV_PARAMS = dict(voxel_size=0.02, sdf_trunc=0.08, depth_trunc=4.0)


def division_sequence(kind, positions, seed=0):
    """32 rigid frames with the `kind` frame in place of those at `positions` (every one when positions is 'all')."""
    rigid = division_frames("rigid", seed=seed)
    odd = division_frames(kind, seed=seed + 1)
    pos = range(32) if positions == "all" else positions
    return [odd[i] if i in pos else rigid[i] for i in range(32)]


def division_split(frame, unit, keys):
    """Per block of `keys`: (in-image voxels on the exact path, in-image voxels on the fast path) masks [lz, ly, lx]."""
    d, _, T = frame
    H, W = d.shape
    l = np.arange(8)
    out = {}
    for k in keys:
        _, _, pz, _, _, inb = project(pose_E(T), DIV_K, W, H, DIV_PARAMS["voxel_size"], unit, k, l[None, None, :],
                                      l[None, :, None], l[:, None, None])
        rare = (pz > 0) & (pz < DIV_LO)
        out[tuple(int(x) for x in k)] = (rare & inb, ~rare & inb)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# uploaded weights
# ---------------------------------------------------------------------------------------------------------------------

ACCEPTED_WEIGHTS = (2.0 ** 24 - 1, 2.0 ** 24, 0.5, 0.0, 1.0)
REJECTED_WEIGHTS = (2.0 ** 24 + 2, 1e20, 2.0 ** 100, 2.0 ** 127, -1.0, np.inf, np.nan)


def weight_blocks(keys, w, seed=0):
    """Blocks at `keys` with every weight `w`, tsdf uniform in [-1, 1] and colours in [0, 255]."""
    rng = np.random.default_rng(seed)
    vox = np.empty((len(keys), 5, 512), f32)
    vox[:, 0] = rng.uniform(-1.0, 1.0, (len(keys), 512))
    vox[:, 1] = f32(w)
    vox[:, 2:] = rng.uniform(0.0, 255.0, (len(keys), 3, 512))
    return np.asarray(keys, np.int32), vox
