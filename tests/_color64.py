"""Float64 colour restated on top of the unchanged oracles, for the float64-colour volume's parity tests.

Open3D's TSDFVoxel keeps an Eigen::Vector3d colour, updated as (c * w + rgb) / (w + 1) in float64
(oracle/open3d_order.c:253-254).  Which voxels take a frame and which pixel each reads does not depend on the voxels'
values, so the block twin (oracle/tsdf_oracle.c) gives both: integrated alone into an empty twin, a frame leaves
weight 1 exactly on the voxels that take it and, since fmaf(0, 0, x) * RN(1 / 1) = x, the pixel's 8-bit colour x in
their colour planes.  `Color64Twin` applies those updates to float64 colours with numpy's IEEE operations (no FMA)
in frame order, next to a twin that integrates every frame for keys, tsdf and weights.  The mesh and point-cloud
colour formulas are restated from a dump with float64 colours (`mesh_colors`, `point_colors`).
tests/test_color64_cpu.py pins all of it to the Open3D-order restatement and to `tsdf_T0.npz`."""

import numpy as np

import oracle

VOX = 512


class Color64Twin:
    def __init__(self, cfg, unit_resolution=16, stride=4):
        self.cfg = cfg
        self._args = dict(block_size=8, stride=stride, unit_resolution=unit_resolution)
        self.tw = oracle.TsdfOracle(cfg.voxel_size, cfg.sdf_trunc, cfg.depth_trunc, **self._args)
        self.row = {}                                  # key -> row of the colour state
        self.keys = np.zeros((0, 3), np.int32)
        self.w = np.zeros((0, VOX), np.float32)        # weights before each frame (float32, as the voxel keeps them)
        self.rgb = np.zeros((0, 3, VOX), np.float64)

    def _rows(self, keys):
        new = [tuple(k) for k in keys.tolist() if tuple(k) not in self.row]
        if new:
            base = len(self.keys)
            for i, k in enumerate(new):
                self.row[k] = base + i
            self.keys = np.concatenate([self.keys, np.array(new, np.int32).reshape(-1, 3)])
            self.w = np.concatenate([self.w, np.zeros((len(new), VOX), np.float32)])
            self.rgb = np.concatenate([self.rgb, np.zeros((len(new), 3, VOX), np.float64)])
        return np.array([self.row[tuple(k)] for k in keys.tolist()], np.int64)

    def integrate(self, depth, color, K, Tcw, nthreads=8):
        self.tw.integrate(depth, color, K, Tcw, nthreads=nthreads)
        one = oracle.TsdfOracle(self.cfg.voxel_size, self.cfg.sdf_trunc, self.cfg.depth_trunc, **self._args)
        one.integrate(depth, color, K, Tcw, nthreads=nthreads)
        f = one.dump_blocks()
        rows = self._rows(f["keys"])
        live = f["vox"][:, 1] == np.float32(1.0)
        x = f["vox"][:, 2:].astype(np.float64)
        w0 = self.w[rows]
        wn = w0 + np.float32(1.0)                      # float32: saturates at 2^24
        c0 = self.rgb[rows]
        c = (c0 * w0.astype(np.float64)[:, None, :] + x) / wn.astype(np.float64)[:, None, :]
        self.rgb[rows] = np.where(live[:, None, :], c, c0)
        self.w[rows] = np.where(live, wn, w0)

    def upload(self, keys, vox, rgb64):
        """seed blocks: vox float32 [n,5,512] (its colour planes are replaced by rgb64 rounded), rgb64 [n,3,512]"""
        vox = np.array(vox, np.float32)
        vox[:, 2:] = np.asarray(rgb64, np.float64).astype(np.float32)
        for k, v in zip(np.asarray(keys), vox):
            self.tw.set_block(k, v)
        rows = self._rows(np.asarray(keys, np.int32).reshape(-1, 3))
        self.w[rows] = vox[:, 1]
        self.rgb[rows] = rgb64

    def dump_blocks(self):
        """keys, hashes, vox float32 [n,5,512] (colours rounded to float32) and rgb64 [n,3,512], in the twin's order"""
        d = self.tw.dump_blocks()
        rows = self._rows(d["keys"])
        assert np.array_equal(self.w[rows], d["vox"][:, 1]), "colour state out of step with the twin's weights"
        vox = d["vox"].copy()
        vox[:, 2:] = self.rgb[rows].astype(np.float32)
        return dict(keys=d["keys"], hashes=d["hashes"], vox=vox, rgb64=self.rgb[rows].copy())


def _lookup(dump, g):
    """(tsdf float32, colour float64 [3]) of global voxels g int [n,3] in a dump with rgb64"""
    g = np.asarray(g, np.int64)
    b = np.floor_divide(g, 8)
    l = g - 8 * b
    index = {tuple(k): i for i, k in enumerate(np.asarray(dump["keys"]).tolist())}
    ub, inv = np.unique(b, axis=0, return_inverse=True)
    row = np.array([index[tuple(k)] for k in ub.tolist()], np.int64)[inv.reshape(-1)]
    v = l[:, 0] + 8 * l[:, 1] + 64 * l[:, 2]
    return dump["vox"][row, 0, v], dump["rgb64"][row, :, v]


def _ends(edges):
    e = np.asarray(edges, np.int64)
    g1 = e[:, :3].copy()
    g1[np.arange(len(e)), e[:, 3]] += 1
    return e[:, :3], g1


def mesh_colors(dump, edges):
    """ExtractTriangleMesh's vertex colour on edge (voxel e, axis a), float64:
    (|f1| (c0 / 255) + |f0| (c1 / 255)) / (|f0| + |f1|), f0, c0 at e and f1, c1 at e + a (open3d_order.c:439,472)"""
    g0, g1 = _ends(edges)
    f0, c0 = _lookup(dump, g0)
    f1, c1 = _lookup(dump, g1)
    a0, a1 = np.abs(f0.astype(np.float64))[:, None], np.abs(f1.astype(np.float64))[:, None]
    return (a1 * (c0 / 255.0) + a0 * (c1 / 255.0)) / (a0 + a1)


def point_colors(dump, edges):
    """ExtractPointCloud's colour with float64 voxel colours: ((c0 r1 + c1 r0) / rs) / 255 with r0 = |f0|, r1 = |f1|
    and rs = r0 + r1 in float32, widened (Vector3d times float promotes to double).  A restatement no running Open3D
    pins, like the float32 one of oracle.numpy_point_cloud."""
    g0, g1 = _ends(edges)
    f0, c0 = _lookup(dump, g0)
    f1, c1 = _lookup(dump, g1)
    r0, r1 = np.abs(f0), np.abs(f1)
    rs = (r0 + r1).astype(np.float64)[:, None]
    return ((c0 * r1.astype(np.float64)[:, None] + c1 * r0.astype(np.float64)[:, None]) / rs) / 255.0


def point_cloud(dump, voxel_length):
    """oracle.numpy_point_cloud's points and edges, with the float64 colours of `point_colors`"""
    p = oracle.numpy_point_cloud(dict(keys=dump["keys"], vox=dump["vox"]), voxel_length)
    return dict(points=p["points"], edges=p["edges"], colors=point_colors(dump, p["edges"]))


def mesh(tw_mesh, dump):
    """the twin's mesh (topology and float64 vertices) with the float64 vertex colours of `mesh_colors`"""
    return dict(vertices=tw_mesh["vertices"], edges=tw_mesh["edges"], triangles=tw_mesh["triangles"],
                colors=mesh_colors(dump, tw_mesh["edges"]))
