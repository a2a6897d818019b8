"""Scene builders shared by tests/test_gpu_tsdf_edges.py and tests/test_tsdf_edges_cpu.py: small deterministic inputs
that drive the TSDF kernels through their rarely taken branches (allocation capacity fallbacks, boundary depths and
poses, adversarial blocks for the mesher), plus the numpy census that proves each scene reaches the branch it is
meant to reach."""

import os
import re
from dataclasses import dataclass

import numpy as np

from pyslam_b200 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def kernel_constants():
    """The allocation capacities as b2v_tsdf.cu declares them (`constexpr int kName = value;`)."""
    src = open(os.path.join(ROOT, "pyslam_b200", "csrc", "b2v_tsdf.cu")).read()
    out = {}
    for name in ("kAllocTile", "kBoxSet", "kBoxList", "kKeySet", "kListCap"):
        m = re.search(r"constexpr\s+int\s+" + name + r"\s*=\s*(\d+)\s*;", src)
        assert m, name
        out[name] = int(m.group(1))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# §1 scenes: images that overflow the allocate kernel's per-tile shared-memory sets
# ---------------------------------------------------------------------------------------------------------------------

@dataclass(frozen=True)
class Scene:
    name: str
    H: int
    W: int
    K: tuple               # fx, fy, cx, cy
    voxel_size: float
    sdf_trunc: float
    depth_trunc: float
    unit: int              # volume_unit_resolution (8 = decision D1, 16 = Open3D units)
    stride: int = 4

    def frame(self, seed):
        """(depth f32 [H,W], colour u8 [H,W,3], Tcw identity) of one independently seeded frame."""
        rng = np.random.default_rng(1000 * (1 + seed) + len(self.name))
        H, W = self.H, self.W
        if self.name.startswith("noisy"):
            d = rng.uniform(0.3, 3.9, (H, W))
        elif self.name == "far-U16":
            d = 0.3 + rng.uniform(0.0, 0.01, (H, W))
            d[:, ::8] = 9.0 + rng.uniform(0.0, 0.05, (H, W // 8))
        elif self.name == "veryfar-D1":
            d = 0.3 + rng.uniform(0.0, 0.01, (H, W))
            d[:, ::8] = 280.0 + rng.uniform(0.0, 1.0, (H, W // 8))
        elif self.name == "widebox-D1":
            d = 1.5 + rng.uniform(0.0, 0.02, (H, W))
        else:
            raise KeyError(self.name)
        c = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        return d.astype(np.float32), c, np.eye(4)


SCENES = {
    "noisy-D1": Scene("noisy-D1", 64, 64, (60.0, 60.0, 31.5, 31.5), 0.01, 0.12, 4.0, 8),
    "noisy-U16": Scene("noisy-U16", 64, 64, (60.0, 60.0, 31.5, 31.5), 0.01, 0.04, 4.0, 16),
    "far-U16": Scene("far-U16", 64, 64, (60.0, 60.0, 31.5, 31.5), 0.0005, 0.002, 10.0, 16),
    "veryfar-D1": Scene("veryfar-D1", 32, 32, (60.0, 60.0, 15.5, 15.5), 0.0005, 0.002, 300.0, 8),
    "widebox-D1": Scene("widebox-D1", 32, 32, (60.0, 60.0, 15.5, 15.5), 0.01, 0.7, 4.0, 8),
}
SEEDS = (0, 1, 2, 3)      # the frames of a scene's sequence


def sample_boxes(scene, depth):
    """Per depth sample of an identity-pose frame: (tile index, lo [3], n [3]) of the +-tau box in allocation units,
    computed like allocate_body (float64 back-projection; D1: pyslam's float32 key rule, else floor(p / L))."""
    st = scene.stride
    d = depth[::st, ::st]
    gh, gw = d.shape
    ii, jj = np.meshgrid(np.arange(gh), np.arange(gw), indexing="ij")
    ok = (d > 0) & (d < f32(scene.depth_trunc))
    z = d[ok].astype(np.float64)
    fx, fy, cx, cy = scene.K
    x = ((jj[ok] * st).astype(np.float64) - cx) * z / fx
    y = ((ii[ok] * st).astype(np.float64) - cy) * z / fy
    pw = np.stack([x, y, z], 1)
    if scene.unit > 8:
        L = scene.voxel_size * scene.unit
        lo = np.floor((pw - scene.sdf_trunc) / L).astype(np.int64)
        hi = np.floor((pw + scene.sdf_trunc) / L).astype(np.int64)
    else:
        tau = float(f32(scene.sdf_trunc))
        inv = f32(1.0) / f32(scene.voxel_size)
        lo = np.floor((pw - tau).astype(np.float32) * inv).astype(np.int64) >> 3
        hi = np.floor((pw + tau).astype(np.float32) * inv).astype(np.int64) >> 3
    T = kernel_constants()["kAllocTile"]
    tiles_x = (gw + T - 1) // T
    tile = (ii[ok] // T) * tiles_x + jj[ok] // T
    return tile, lo, hi - lo + 1


def tile_census(scene, depth):
    """Per allocation tile: distinct unit keys, the keys no other tile touches, the spans of the box origins and of
    the unit keys, and the largest box side.  The tile's reference key is whichever sample wins a shared-memory CAS,
    so the spans (not the offsets from one sample) decide whether a far path is certain."""
    tile, lo, n = sample_boxes(scene, depth)
    keysets = {}
    for t in np.unique(tile):
        sel = tile == t
        ks = set()
        for l, m in zip(lo[sel], n[sel]):
            if m.max() > 15:
                continue            # over-sized boxes are counted by max_n; their keys are not needed here
            g = np.stack(np.meshgrid(*[np.arange(k) for k in m], indexing="ij"), -1).reshape(-1, 3) + l
            ks.update(map(tuple, g))
        keysets[int(t)] = ks
    count = {}
    for ks in keysets.values():
        for k in ks:
            count[k] = count.get(k, 0) + 1
    sub = (scene.unit // 8) ** 3
    out = {}
    for t, ks in keysets.items():
        sel = tile == t
        hi = lo[sel] + n[sel] - 1
        out[t] = dict(units=len(ks), blocks=len(ks) * sub,
                      own_blocks=sum(1 for k in ks if count[k] == 1) * sub,
                      box_span=int((lo[sel].max(0) - lo[sel].min(0)).max()),
                      key_span=int((hi.max(0) - lo[sel].min(0)).max()),
                      max_n=int(n[sel].max()), min_max_n=int(n[sel].max(1).min()))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# §2 boundary inputs
# ---------------------------------------------------------------------------------------------------------------------

def depth_specials(depth_trunc):
    dt = f32(depth_trunc)
    return np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, -1.0, dt, np.nextafter(dt, f32(0)), 1e-45, 1e-30, 0.03],
                    np.float32)


def specials_frame(i=0, seed=5):
    """T0 frame i with about 30 % of its pixels (on and off the stride-4 samples) replaced by special depths."""
    cfg = S.CONFIGS["T0"]
    d, c, T = S.render_frame(cfg, i)
    rng = np.random.default_rng(seed)
    sp = depth_specials(cfg.depth_trunc)
    hit = rng.random(d.shape) < 0.3
    d = d.copy()
    d[hit] = sp[rng.integers(0, len(sp), int(hit.sum()))]
    # every special value also sits on a depth sample of the default stride
    for k, v in enumerate(sp):
        d[4 * (k % 6), 4 * (k // 6 + 2)] = v
    return d, c, T


def band_frames(cfg):
    """Flat depth 0.03 m under a wide field of view with tau 0.08: voxels behind the camera, first from the identity
    pose, then from band_pose's.  (depth, colour, K, Tcw) per frame."""
    _, c, _ = S.render_frame(cfg, 0)
    d = np.full((cfg.height, cfg.width), 0.03, np.float32)
    K = np.array([10.0, 10.0, cfg.cx, cfg.cy])
    return [(d, c, K, np.eye(4)), (d, c, K, band_pose(cfg))]


def band_pose(cfg):
    """World->camera pose (identity rotation) that puts the centres of the voxel layer z = 0 of volume unit z = 0 at
    camera z = +0.0 exactly: the translation is minus that layer's float32 centre coordinate
    h2 = (float)((double)(vl / 2) + 0 * L) = vl / 2 (DESIGN §3), and p.z = ((0 h0 + 0 h1) + 1 h2) - h2 = +0.0."""
    h2 = f32(cfg.voxel_size) * f32(0.5)
    T = np.eye(4)
    T[2, 3] = -float(h2)
    return T


def crop(cfg, i, H, W, y0=16, x0=24):
    """An H x W window of T0 frame i with the intrinsics moved with it."""
    d, c, T = S.render_frame(cfg, i)
    K = np.array([cfg.fx, cfg.fy, cfg.cx - x0, cfg.cy - y0])
    return np.ascontiguousarray(d[y0:y0 + H, x0:x0 + W]), np.ascontiguousarray(c[y0:y0 + H, x0:x0 + W]), K, T


def invalid_depth(shape, seed):
    """A depth image no pixel of which is valid: zeros, negatives, NaN, +inf."""
    rng = np.random.default_rng(seed)
    vals = np.array([0.0, -0.0, -1.0, np.nan, np.inf, -np.inf], np.float32)
    return vals[rng.integers(0, len(vals), shape)]


# ---------------------------------------------------------------------------------------------------------------------
# §3 adversarial blocks for the mesher
# ---------------------------------------------------------------------------------------------------------------------

def random_blocks(seed=3, n_keys=300):
    """About 300 keys of a 9 x 9 x 5 region with holes (negative keys included); tsdf uniform in [-1, 1] with exact
    0.0, -0.0, +-0.98 and +-nextafter(0.98) sprinkled in; 25 % zero weights; colours random floats in 0..255."""
    rng = np.random.default_rng(seed)
    grid = np.stack(np.meshgrid(np.arange(-4, 5), np.arange(-5, 4), np.arange(-2, 3), indexing="ij"), -1).reshape(-1, 3)
    keys = grid[np.sort(rng.choice(len(grid), n_keys, replace=False))].astype(np.int32)
    vox = np.zeros((n_keys, 5, 512), np.float32)
    vox[:, 0] = rng.uniform(-1.0, 1.0, (n_keys, 512))
    a = f32(0.98)
    special = np.array([0.0, -0.0, a, -a, np.nextafter(a, f32(0)), -np.nextafter(a, f32(0)), np.nextafter(a, f32(1)),
                        -np.nextafter(a, f32(1))], np.float32)
    hit = rng.random((n_keys, 512)) < 0.1
    vox[:, 0][hit] = special[rng.integers(0, len(special), int(hit.sum()))]
    vox[:, 1] = np.where(rng.random((n_keys, 512)) < 0.25, 0.0, rng.integers(1, 50, (n_keys, 512))).astype(np.float32)
    vox[:, 2:] = rng.uniform(0.0, 255.0, (n_keys, 3, 512))
    return keys, vox


def max_output_blocks(seed=4):
    """Block (0, 0, 0) with a checkerboard tsdf sign and its 7 forward neighbours, all fully observed: every edge of
    every cube of the block crosses the surface, so the block holds 3 * 512 = 1536 vertices."""
    rng = np.random.default_rng(seed)
    l = np.arange(512)
    lx, ly, lz = l % 8, (l // 8) % 8, l // 64
    keys, vox = [], []
    for o in range(8):
        k = np.array([o & 1, (o >> 1) & 1, (o >> 2) & 1], np.int32)
        v = np.zeros((5, 512), np.float32)
        parity = (lx + ly + lz + k.sum() * 8) & 1
        v[0] = np.where(parity == 0, 1.0, -1.0) * rng.uniform(0.05, 0.95, 512)
        v[1] = rng.integers(1, 9, 512)
        v[2:] = rng.uniform(0.0, 255.0, (3, 512))
        keys.append(k)
        vox.append(v)
    return np.array(keys, np.int32), np.stack(vox).astype(np.float32)


def cube_cases(keys, vox):
    """Marching-cubes case (corner order 000,100,110,010,001,101,111,011; bit set = tsdf < 0) of every cube whose 8
    corners exist and are observed."""
    idx = {tuple(k): i for i, k in enumerate(keys)}
    nb = len(keys)
    f = vox[:, 0].reshape(nb, 8, 8, 8)          # [b, z, y, x]
    w = vox[:, 1].reshape(nb, 8, 8, 8)
    # 9^3 tiles with the +x / +y / +z halo from the neighbours (missing = unobserved)
    F = np.zeros((nb, 9, 9, 9), np.float32)
    Wt = np.zeros((nb, 9, 9, 9), np.float32)
    for b, k in enumerate(keys):
        for o in range(8):
            dx, dy, dz = o & 1, (o >> 1) & 1, (o >> 2) & 1
            j = idx.get((k[0] + dx, k[1] + dy, k[2] + dz))
            if j is None:
                continue
            sz, sy, sx = (slice(0, 8), slice(8, 9))[dz], (slice(0, 8), slice(8, 9))[dy], (slice(0, 8), slice(8, 9))[dx]
            src = (slice(0, 8) if dz == 0 else slice(0, 1), slice(0, 8) if dy == 0 else slice(0, 1),
                   slice(0, 8) if dx == 0 else slice(0, 1))
            F[b, sz, sy, sx] = f[j][src]
            Wt[b, sz, sy, sx] = w[j][src]
    corners = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
    case = np.zeros((nb, 8, 8, 8), np.int64)
    ok = np.ones((nb, 8, 8, 8), bool)
    for bit, (cx, cy, cz) in enumerate(corners):
        fc = F[:, cz:cz + 8, cy:cy + 8, cx:cx + 8]
        case |= (fc < 0).astype(np.int64) << bit
        ok &= Wt[:, cz:cz + 8, cy:cy + 8, cx:cx + 8] != 0
    return case[ok]
