"""TEST INFRASTRUCTURE ONLY: ctypes front-ends for the oracle libraries + numpy cross-checks."""

from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_DIR = os.path.dirname(os.path.abspath(__file__))
_TSDF_SO = os.path.join(_DIR, "liboracle_tsdf.so")
_REF_SO = os.path.join(_DIR, "_ref", "libref_grid.so")

_f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
_u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
_u64p = np.ctypeslib.ndpointer(np.uint64, flags="C_CONTIGUOUS")


def build(quiet: bool = True) -> None:
    """Compile the oracle libraries (the C restatement always; `_ref` when /root/reference exists)."""
    subprocess.run(["make", "-C", _DIR, "all"], check=True,
                   stdout=subprocess.DEVNULL if quiet else None)


def have_ref() -> bool:
    return os.path.exists(_REF_SO)


_tsdf_lib = None
_ref_lib = None


def _tsdf():
    global _tsdf_lib
    if _tsdf_lib is None:
        if not os.path.exists(_TSDF_SO):
            build()
        L = C.CDLL(_TSDF_SO)
        L.tsdf_oracle_create.restype = C.c_void_p
        L.tsdf_oracle_create.argtypes = [C.c_float, C.c_int, C.c_float, C.c_float, C.c_int]
        L.tsdf_oracle_destroy.argtypes = [C.c_void_p]
        L.tsdf_oracle_reset.argtypes = [C.c_void_p]
        L.tsdf_oracle_num_blocks.restype = C.c_int64
        L.tsdf_oracle_num_blocks.argtypes = [C.c_void_p]
        L.tsdf_oracle_num_touched.restype = C.c_int64
        L.tsdf_oracle_num_touched.argtypes = [C.c_void_p]
        L.tsdf_oracle_integrate.restype = C.c_int64
        L.tsdf_oracle_integrate.argtypes = [C.c_void_p, _f32p, _u8p, C.c_int, C.c_int, _f64p, _f64p,
                                            C.c_int]
        L.tsdf_oracle_last_touched.restype = C.c_int64
        L.tsdf_oracle_last_touched.argtypes = [C.c_void_p, _i32p]
        L.tsdf_oracle_dump.restype = C.c_int64
        L.tsdf_oracle_dump.argtypes = [C.c_void_p, _i32p, _u64p, _f32p]
        L.tsdf_oracle_extract_mesh.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.tsdf_oracle_mesh_copy.argtypes = [_f64p, _f64p, _i32p, _i32p]
        L.tsdf_oracle_block_key_hash.restype = C.c_uint64
        L.tsdf_oracle_block_key_hash.argtypes = [C.c_int32] * 3
        L.tsdf_oracle_floor_div.restype = C.c_int64
        L.tsdf_oracle_floor_div.argtypes = [C.c_int64, C.c_int64]
        L.tsdf_oracle_voxel_coord.restype = C.c_int32
        L.tsdf_oracle_voxel_coord.argtypes = [C.c_float, C.c_float]
        L.tsdf_oracle_max_threads.restype = C.c_int
        L.tsdf_oracle_set_block.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, _f32p]
        L.tsdf_oracle_set_units.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double]
        _tsdf_lib = L
    return _tsdf_lib


def _ref():
    global _ref_lib
    if _ref_lib is None:
        if not have_ref():
            raise RuntimeError("oracle/_ref/libref_grid.so missing (needs /root/reference to build)")
        L = C.CDLL(_REF_SO)
        L.refgrid_create.restype = C.c_void_p
        L.refgrid_create.argtypes = [C.c_float, C.c_int]
        L.refgrid_destroy.argtypes = [C.c_void_p]
        L.refgrid_clear.argtypes = [C.c_void_p]
        L.refgrid_integrate.restype = C.c_double
        L.refgrid_integrate.argtypes = [C.c_void_p, _f32p, C.c_void_p, C.c_int64]
        L.refgrid_integrate_f64.restype = C.c_double
        L.refgrid_integrate_f64.argtypes = [C.c_void_p, _f64p, C.c_void_p, C.c_int64]
        L.refgrid_num_blocks.restype = C.c_int64
        L.refgrid_num_blocks.argtypes = [C.c_void_p]
        L.refgrid_block_size.argtypes = [C.c_void_p]
        L.refgrid_inv_voxel_size.restype = C.c_float
        L.refgrid_inv_voxel_size.argtypes = [C.c_void_p]
        L.refgrid_dump_blocks.restype = C.c_int64
        L.refgrid_dump_blocks.argtypes = [C.c_void_p] * 6
        L.refgrid_get_voxels.restype = C.c_int64
        L.refgrid_get_voxels.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                         C.POINTER(C.c_double)]
        L.refgrid_remove_low_count_voxels.argtypes = [C.c_void_p, C.c_int]
        L.refgrid_carve.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int,
                                    C.c_int, _f64p, C.c_float, C.c_float, _f32p, C.c_float]
        L.refgrid_get_voxels_in_frustum.restype = C.c_int64
        L.refgrid_get_voxels_in_frustum.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float,
                                                    C.c_int, C.c_int, _f64p, C.c_float, C.c_float, C.c_int,
                                                    C.c_void_p, C.c_void_p]
        L.refgrid_get_voxels_in_bb.restype = C.c_int64
        L.refgrid_get_voxels_in_bb.argtypes = [C.c_void_p, _f64p, C.c_int, C.c_void_p, C.c_void_p]
        L.ref_voxel_key_inv.argtypes = [C.c_float] * 4 + [_i32p]
        L.ref_floor_div.restype = C.c_int64
        L.ref_floor_div.argtypes = [C.c_int64, C.c_int64]
        L.ref_block_and_local_key.argtypes = [_i32p, C.c_int, _i32p, _i32p]
        L.ref_block_key_hash.restype = C.c_uint64
        L.ref_block_key_hash.argtypes = [C.c_int32] * 3
        L.ref_sizeof_voxel_data.restype = C.c_int
        _ref_lib = L
    return _ref_lib


# ---------------------------------------------------------------------------------------------
# compiled reference
# ---------------------------------------------------------------------------------------------

def ref_block_key_hash(x, y, z) -> int:
    return int(_ref().ref_block_key_hash(int(x), int(y), int(z)))


def ref_floor_div(a, b) -> int:
    return int(_ref().ref_floor_div(int(a), int(b)))


def ref_keys(point, voxel_size, block_size=8):
    """(voxel key, block key, local key) of one point exactly as the reference computes them."""
    L = _ref()
    inv = np.float32(1.0) / np.float32(voxel_size)
    vk = np.zeros(3, np.int32)
    L.ref_voxel_key_inv(float(np.float32(point[0])), float(np.float32(point[1])),
                        float(np.float32(point[2])), float(inv), vk)
    bk, lk = np.zeros(3, np.int32), np.zeros(3, np.int32)
    L.ref_block_and_local_key(vk, int(block_size), bk, lk)
    return vk, bk, lk


class RefGrid:
    """The unmodified reference `volumetric::VoxelBlockGrid` (sequential branch)."""

    def __init__(self, voxel_size: float, block_size: int = 8):
        self._L = _ref()
        self._h = self._L.refgrid_create(float(voxel_size), int(block_size))
        self.block_size = block_size
        self.last_elapsed_s = 0.0

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.refgrid_destroy(self._h)
            self._h = None

    def integrate(self, points, colors=None) -> float:
        f64 = np.asarray(points).dtype == np.float64        # the reference's float64-points overload
        pts = np.ascontiguousarray(points, dtype=np.float64 if f64 else np.float32)
        assert pts.ndim == 2 and pts.shape[1] == 3
        cp = None
        if colors is not None:
            cols = np.ascontiguousarray(colors, dtype=np.float32)
            assert cols.shape == pts.shape
            cp = cols.ctypes.data
        fn = self._L.refgrid_integrate_f64 if f64 else self._L.refgrid_integrate
        self.last_elapsed_s = fn(self._h, pts.reshape(-1) if f64 else pts, cp, pts.shape[0])
        return self.last_elapsed_s

    def num_blocks(self) -> int:
        return int(self._L.refgrid_num_blocks(self._h))

    def clear(self):
        self._L.refgrid_clear(self._h)

    def dump_blocks(self):
        nb = self.num_blocks()
        nv = self.block_size ** 3
        keys = np.zeros((nb, 3), np.int32)
        hashes = np.zeros(nb, np.uint64)
        count = np.zeros((nb, nv), np.int32)
        pos = np.zeros((nb, nv, 3), np.float32)
        col = np.zeros((nb, nv, 3), np.float32)
        self._L.refgrid_dump_blocks(self._h, keys.ctypes.data, hashes.ctypes.data, count.ctypes.data,
                                    pos.ctypes.data, col.ctypes.data)
        return dict(keys=keys, hashes=hashes, count=count, pos_sum=pos, col_sum=col)

    def get_voxels(self, min_count=1):
        el = C.c_double(0.0)
        n = self._L.refgrid_get_voxels(self._h, int(min_count), None, None, C.byref(el))
        pts = np.zeros((n, 3), np.float32)
        cols = np.zeros((n, 3), np.float32)
        if n:
            self._L.refgrid_get_voxels(self._h, int(min_count), pts.ctypes.data, cols.ctypes.data,
                                       C.byref(el))
        self.last_elapsed_s = el.value
        return pts, cols

    def remove_low_count_voxels(self, min_count):
        self._L.refgrid_remove_low_count_voxels(self._h, int(min_count))

    def get_voxels_in_frustum(self, K, width, height, Tcw, min_count=1, depth_max=10.0, depth_min=1e-2):
        T = np.ascontiguousarray(Tcw, np.float64).reshape(16)
        a = (self._h, K[0], K[1], K[2], K[3], int(width), int(height), T, depth_max, depth_min, int(min_count))
        n = self._L.refgrid_get_voxels_in_frustum(*a, None, None)
        pts, cols = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.float32)
        if n:
            self._L.refgrid_get_voxels_in_frustum(*a, pts.ctypes.data, cols.ctypes.data)
        return pts, cols

    def get_voxels_in_bb(self, bbox, min_count=1):
        bb = np.ascontiguousarray(bbox, np.float64).reshape(6)
        n = self._L.refgrid_get_voxels_in_bb(self._h, bb, int(min_count), None, None)
        pts, cols = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.float32)
        if n:
            self._L.refgrid_get_voxels_in_bb(self._h, bb, int(min_count), pts.ctypes.data, cols.ctypes.data)
        return pts, cols

    def carve(self, K, width, height, Tcw, depth, depth_threshold=1e-2, depth_max=10.0,
              depth_min=1e-2):
        d = np.ascontiguousarray(depth, np.float32)
        T = np.ascontiguousarray(Tcw, np.float64).reshape(16)
        self._L.refgrid_carve(self._h, K[0], K[1], K[2], K[3], int(width), int(height), T,
                              depth_max, depth_min, d, depth_threshold)


# ---------------------------------------------------------------------------------------------
# C restatement of the TSDF path
# ---------------------------------------------------------------------------------------------

class TsdfOracle:
    def __init__(self, voxel_size, sdf_trunc, depth_trunc, block_size=8, stride=4, unit_resolution=16):
        self._L = _tsdf()
        self.block_size = block_size
        self.nvox = block_size ** 3
        self._h = self._L.tsdf_oracle_create(float(np.float32(voxel_size)), int(block_size),
                                             float(np.float32(sdf_trunc)),
                                             float(np.float32(depth_trunc)), int(stride))
        self.set_units(unit_resolution, voxel_size, sdf_trunc)

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.tsdf_oracle_destroy(self._h)
            self._h = None

    @staticmethod
    def max_threads() -> int:
        return int(_tsdf().tsdf_oracle_max_threads())

    def reset(self):
        self._L.tsdf_oracle_reset(self._h)

    def set_units(self, unit_resolution, voxel_length, sdf_trunc):
        """Open3D volume-unit resolution: 16 = the reference's setting (allocation by LocateVolumeUnit), 8 = decision
        D1 (allocation by the float32 pyslam key range); voxel_length / sdf_trunc as the float64 values Open3D holds."""
        self._L.tsdf_oracle_set_units(self._h, int(unit_resolution), float(voxel_length), float(sdf_trunc))

    def integrate(self, depth, color, K, Tcw, nthreads=1) -> int:
        d = np.ascontiguousarray(depth, np.float32)
        c = np.ascontiguousarray(color, np.uint8)
        H, W = d.shape
        assert c.shape == (H, W, 3)
        return int(self._L.tsdf_oracle_integrate(self._h, d, c, H, W,
                                                 np.ascontiguousarray(K, np.float64).reshape(4),
                                                 np.ascontiguousarray(Tcw, np.float64).reshape(16),
                                                 int(nthreads)))

    def num_blocks(self) -> int:
        return int(self._L.tsdf_oracle_num_blocks(self._h))

    def set_block(self, key, vox):
        """test hook: overwrite / create one block with vox f32 [5, B^3]"""
        v = np.ascontiguousarray(vox, np.float32).reshape(5 * self.nvox)
        self._L.tsdf_oracle_set_block(self._h, int(key[0]), int(key[1]), int(key[2]), v)

    def last_touched(self):
        n = int(self._L.tsdf_oracle_num_touched(self._h))
        keys = np.zeros((n, 3), np.int32)
        self._L.tsdf_oracle_last_touched(self._h, keys)
        return keys

    def dump_blocks(self):
        nb = self.num_blocks()
        keys = np.zeros((nb, 3), np.int32)
        hashes = np.zeros(nb, np.uint64)
        vox = np.zeros((nb, 5, self.nvox), np.float32)
        self._L.tsdf_oracle_dump(self._h, keys, hashes, vox)
        return dict(keys=keys, hashes=hashes, vox=vox)

    def extract_mesh(self):
        nv, nt = C.c_int64(0), C.c_int64(0)
        self._L.tsdf_oracle_extract_mesh(self._h, C.byref(nv), C.byref(nt))
        V64 = np.zeros((nv.value, 3), np.float64)
        Cc = np.zeros((nv.value, 3), np.float64)
        E = np.zeros((nv.value, 4), np.int32)
        T = np.zeros((nt.value, 3), np.int32)
        self._L.tsdf_oracle_mesh_copy(V64.reshape(-1), Cc.reshape(-1), E.reshape(-1), T.reshape(-1))
        return dict(vertices=V64, colors=Cc, edges=E, triangles=T)


# ---------------------------------------------------------------------------------------------
# Open3D ScalableTSDFVolume in Open3D's own operation order (oracle/open3d_order.c)
# ---------------------------------------------------------------------------------------------
_O3D_SO = os.path.join(_DIR, "libopen3d_order.so")
_o3d_lib = None


def _o3d():
    global _o3d_lib
    if _o3d_lib is None:
        if not os.path.exists(_O3D_SO):
            build()
        L = C.CDLL(_O3D_SO)
        vp = C.c_void_p
        L.o3d_create.restype = vp
        L.o3d_create.argtypes = [C.c_double, C.c_double, C.c_int, C.c_int]
        L.o3d_destroy.argtypes = [vp]
        L.o3d_reset.argtypes = [vp]
        L.o3d_num_units.restype = C.c_int64
        L.o3d_num_units.argtypes = [vp]
        L.o3d_num_touched.restype = C.c_int64
        L.o3d_num_touched.argtypes = [vp]
        L.o3d_prepare_depth.argtypes = [_f32p, _f32p, C.c_int64, C.c_double, C.c_double]
        L.o3d_multiplier.argtypes = [_f32p, C.c_int, C.c_int, _f64p]
        L.o3d_integrate.restype = C.c_int64
        L.o3d_integrate.argtypes = [vp, _f32p, _u8p, _f32p, C.c_int, C.c_int, _f64p, _f64p, C.c_int]
        L.o3d_last_touched.restype = C.c_int64
        L.o3d_last_touched.argtypes = [vp, _i32p]
        L.o3d_dump_blocks.restype = C.c_int64
        L.o3d_dump_blocks.argtypes = [vp, vp, vp]
        L.o3d_extract_mesh.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.o3d_mesh_copy.argtypes = [_f64p, _f64p, _i32p, _i32p]
        _o3d_lib = L
    return _o3d_lib


class Open3DOrderVolume:
    """`o3d.pipelines.integration.ScalableTSDFVolume(voxel_length, sdf_trunc, RGB8, volume_unit_resolution,
    depth_sampling_stride)` as the reference constructs it (volumetric_integrator_tsdf.py:104-108), restated in
    Open3D's own operation order and types.  `integrate` takes what the reference passes at tsdf.py:215-223:
    a float32 depth in metres (depth_scale 1.0), the depth truncation of create_from_color_and_depth, RGB u8,
    the intrinsics and the world->camera pose."""

    def __init__(self, voxel_length, sdf_trunc, volume_unit_resolution=16, depth_sampling_stride=4):
        self._L = _o3d()
        self.R = int(volume_unit_resolution)
        assert self.R % 8 == 0
        self._h = self._L.o3d_create(float(voxel_length), float(sdf_trunc), self.R, int(depth_sampling_stride))
        self._mult_key, self._mult = None, None

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.o3d_destroy(self._h)
            self._h = None

    def reset(self):
        self._L.o3d_reset(self._h)

    def integrate(self, depth, color, K, Tcw, depth_trunc, depth_scale=1.0, nthreads=1) -> int:
        d_in = np.ascontiguousarray(depth, np.float32)
        c = np.ascontiguousarray(color, np.uint8)
        H, W = d_in.shape
        assert c.shape == (H, W, 3)
        d = np.empty_like(d_in)
        self._L.o3d_prepare_depth(d_in.reshape(-1), d.reshape(-1), d.size, float(depth_scale), float(depth_trunc))
        K4 = np.ascontiguousarray(K, np.float64).reshape(4)
        key = (H, W, tuple(K4))
        if self._mult_key != key:
            self._mult = np.zeros((H, W), np.float32)
            self._L.o3d_multiplier(self._mult.reshape(-1), H, W, K4)
            self._mult_key = key
        return int(self._L.o3d_integrate(self._h, d.reshape(-1), c.reshape(-1), self._mult.reshape(-1), H, W, K4,
                                         np.ascontiguousarray(Tcw, np.float64).reshape(16), int(nthreads)))

    def num_units(self) -> int:
        return int(self._L.o3d_num_units(self._h))

    def last_touched_units(self):
        n = int(self._L.o3d_num_touched(self._h))
        idx = np.zeros((n, 3), np.int32)
        self._L.o3d_last_touched(self._h, idx.reshape(-1))
        return idx

    def dump_blocks(self):
        """Every unit as (R/8)^3 blocks in the product's layout: keys int32 [nb,3], vox float64 [nb,5,512]."""
        nb = self.num_units() * (self.R // 8) ** 3
        keys = np.zeros((nb, 3), np.int32)
        vox = np.zeros((nb, 5, 512), np.float64)
        self._L.o3d_dump_blocks(self._h, keys.ctypes.data, vox.ctypes.data)
        return dict(keys=keys, vox=vox)

    def extract_triangle_mesh(self):
        nv, nt = C.c_int64(0), C.c_int64(0)
        self._L.o3d_extract_mesh(self._h, C.byref(nv), C.byref(nt))
        V = np.zeros((nv.value, 3), np.float64)
        Cc = np.zeros((nv.value, 3), np.float64)
        E = np.zeros((nv.value, 4), np.int32)
        T = np.zeros((nt.value, 3), np.int32)
        self._L.o3d_mesh_copy(V.reshape(-1), Cc.reshape(-1), E.reshape(-1), T.reshape(-1))
        return dict(vertices=V, colors=Cc, edges=E, triangles=T)


def canonical_mesh(vertices, colors, edges, triangles):
    """Order-independent form of a welded mesh: vertices sorted by canonical edge id
    (gx,gy,gz,axis); triangles re-indexed, each rotated so its smallest index leads (winding kept),
    then sorted.  Two extractions of the same volume are equal iff these arrays are equal."""
    edges = np.asarray(edges)
    order = np.lexsort((edges[:, 3], edges[:, 2], edges[:, 1], edges[:, 0]))
    inv = np.empty_like(order)
    inv[order] = np.arange(order.size)
    tri = inv[np.asarray(triangles)] if len(triangles) else np.zeros((0, 3), np.int64)
    if len(tri):
        k = np.argmin(tri, axis=1)
        idx = (k[:, None] + np.arange(3)[None, :]) % 3
        tri = np.take_along_axis(tri, idx, axis=1)
        tri = tri[np.lexsort((tri[:, 2], tri[:, 1], tri[:, 0]))]
    return dict(vertices=np.asarray(vertices)[order], colors=np.asarray(colors)[order],
                edges=edges[order], triangles=tri.astype(np.int64))


# ---------------------------------------------------------------------------------------------
# independent numpy restatement (pins the C oracle; float32 numpy, no FMA -> tolerance compare)
# ---------------------------------------------------------------------------------------------

def numpy_touched_blocks(depth, K, Tcw, voxel_size, sdf_trunc, depth_trunc, block_size=8, stride=4):
    """A.2 touched-block set of one frame as a sorted int32 [n,3] array (numpy, vectorised)."""
    fx, fy, cx, cy = [float(v) for v in K]
    d = np.asarray(depth, np.float32)[::stride, ::stride]
    H, W = d.shape
    jj, ii = np.meshgrid(np.arange(W) * stride, np.arange(H) * stride)
    valid = (d > 0) & (d < np.float32(depth_trunc))
    z = d[valid].astype(np.float64)
    x = (jj[valid].astype(np.float64) - cx) * z / fx
    y = (ii[valid].astype(np.float64) - cy) * z / fy
    Tcw = np.asarray(Tcw, np.float64).reshape(4, 4)
    R = Tcw[:3, :3].T
    t = -np.stack([(R[a, 0] * Tcw[0, 3] + R[a, 1] * Tcw[1, 3]) + R[a, 2] * Tcw[2, 3]
                   for a in range(3)])
    pw = np.stack([((R[a, 0] * x + R[a, 1] * y) + R[a, 2] * z) + t[a] for a in range(3)], axis=1)
    tau = float(np.float32(sdf_trunc))
    inv_vs = np.float32(1.0) / np.float32(voxel_size)
    lo = np.floor((pw - tau).astype(np.float32) * inv_vs).astype(np.int64) // block_size
    hi = np.floor((pw + tau).astype(np.float32) * inv_vs).astype(np.int64) // block_size
    keys = set()
    span = (hi - lo).max(axis=0) + 1 if len(lo) else np.zeros(3, np.int64)
    for dx in range(int(span[0])):
        for dy in range(int(span[1])):
            for dz in range(int(span[2])):
                k = lo + np.array([dx, dy, dz])
                ok = np.all(k <= hi, axis=1)
                keys.update(map(tuple, k[ok]))
    out = np.array(sorted(keys), dtype=np.int32).reshape(-1, 3)
    return out


def numpy_point_cloud(dump, voxel_length, unit_resolution=16):
    """A.4 ExtractPointCloud restated in numpy from a block dump (keys int32 [nb,3], vox float32 [nb,5,512]): the
    formulas DESIGN §3 and b2v_mesh.cu state, evaluated with numpy's IEEE operations (float64 positions, float32
    weights of the blend and float32 colours).  It pins that documented formula, not a running Open3D; whether
    Open3D also re-evaluates the two off-axis coordinates through the blend is not pinned.
      selection  w != 0 and -0.98 <= f < 0.98 at both ends of an edge along +x / +y / +z (across block borders;
                 a missing neighbour is unobserved) and f0 * f1 < 0 in float32
      position   p0 = (vl/2 + vl * x_in_unit) + unit * L (float64, L = vl * unit_resolution); on the edge's axis
                 p = (p0 r1 + (p0 + vl) r0) / rs with r0 = |f0|, r1 = |f1|, rs = r0 + r1 in float32
      colour     ((c0 r1 + c1 r0) / rs) / 255 in float32, widened
    Returns dict(points f64 [n,3], colors f64 [n,3], edges int32 [n,4] = global voxel (x, y, z) + axis)."""
    keys = np.asarray(dump["keys"], np.int64)
    vox = np.asarray(dump["vox"], np.float32)
    nb = len(keys)
    S = {8: 0, 16: 1, 32: 2}[int(unit_resolution)]
    vl = float(voxel_length)
    half = vl * 0.5
    L = vl * float(8 << S)
    idx = {tuple(k): i for i, k in enumerate(keys.tolist())}
    f = vox[:, 0].reshape(nb, 8, 8, 8)      # [b, z, y, x]
    w = vox[:, 1].reshape(nb, 8, 8, 8)
    c = vox[:, 2:].reshape(nb, 3, 8, 8, 8)
    lz, ly, lx = np.meshgrid(np.arange(8), np.arange(8), np.arange(8), indexing="ij")
    loc = (lx, ly, lz)
    pts, cols, edges = [], [], []
    a98 = np.float32(0.98)
    for a in range(3):
        # the voxel at +1 along axis a: shift inside the block, the first slab of the neighbour at the border
        ax = 3 - a                          # array axis of spatial axis a in [b, z, y, x] (c: one more)
        nbr = np.array([idx.get((k[0] + (a == 0), k[1] + (a == 1), k[2] + (a == 2)), -1) for k in keys.tolist()],
                       np.int64)
        has = nbr >= 0
        nsafe = np.where(has, nbr, 0)

        def shifted(arr, axis):
            inner = np.take(arr, range(1, 8), axis=axis)
            border = np.take(arr[nsafe], [0], axis=axis)
            return np.concatenate([inner, border], axis=axis)

        f1, w1, c1 = shifted(f, ax), shifted(w, ax), shifted(c, ax + 1)
        border_missing = np.zeros((nb, 8, 8, 8), bool)
        sl = [slice(None)] * 4
        sl[ax] = slice(7, 8)
        border_missing[tuple(sl)] = ~has[:, None, None, None]
        ok0 = (w != 0) & (f < a98) & (f >= -a98)
        ok1 = (w1 != 0) & (f1 < a98) & (f1 >= -a98) & ~border_missing
        sel = ok0 & ok1 & (f * f1 < np.float32(0))
        b, z, y, x = np.nonzero(sel)
        l3 = np.stack([x, y, z], 1)
        k3 = keys[b]
        u = k3 >> S
        xin = (k3 - (u << S)) * 8 + l3
        p0 = (half + vl * xin.astype(np.float64)) + u.astype(np.float64) * L
        r0 = np.abs(f[b, z, y, x])
        r1 = np.abs(f1[b, z, y, x])
        rs = r0 + r1                                    # float32
        pa = p0[:, a]
        p = p0.copy()
        p[:, a] = (pa * r1.astype(np.float64) + (pa + vl) * r0.astype(np.float64)) / rs.astype(np.float64)
        col = np.empty((len(b), 3), np.float64)
        for k in range(3):
            num = c[b, k, z, y, x] * r1 + c1[b, k, z, y, x] * r0   # float32 products and sum
            col[:, k] = ((num / rs) / np.float32(255.0)).astype(np.float64)
        pts.append(p)
        cols.append(col)
        edges.append(np.concatenate([k3 * 8 + l3, np.full((len(b), 1), a)], 1).astype(np.int32))
    return dict(points=np.concatenate(pts), colors=np.concatenate(cols), edges=np.concatenate(edges))


class numpy_grid:
    """The point-average `VoxelBlockGrid` (b2v_grid.cu, voxel_block_grid.hpp) restated in numpy, voxel by voxel.
      keys       float32 points: floor(float32(x * inv_vs)), inv_vs = float32(1 / voxel_size);
                 float64 points: floor(x * float64(inv_vs)); block = floor_div(voxel, 8)
      sums       count += 1, pos += float32(x), col += c (float32 c, or float32(c) * float32(1/255) for uint8),
                 accumulated in input order in float32 (np.add.at)
      means      sum / float32(count)
      queries    count >= min_count, voxel key inside the float64 key bounds floor(bb * float64(inv_vs)), then the
                 float64 box test or the frustum test of CameraFrustrum::contains (R p + t in float64, in the kernel's
                 order; u = float32(fx * (x / z) + cx), 0 <= u < W, depth = float32(z) in [depth_min, depth_max])
      carve      the depth at truncated (v, u); skipped when <= 0 or not finite; reset when depth < image - thr
    A block exists once a point lands in it; resetting voxels (remove_low_count_voxels, carve) keeps the block."""

    def __init__(self, voxel_size):
        self.inv_vs = np.float32(1.0) / np.float32(voxel_size)
        self.clear()

    def clear(self):
        self.keys = np.zeros((0, 3), np.int64)      # voxel keys, one row per voxel ever touched
        self.count = np.zeros(0, np.int64)
        self.pos = np.zeros((0, 3), np.float32)
        self.col = np.zeros((0, 3), np.float32)

    def voxel_keys(self, points):
        p = np.asarray(points)
        if p.dtype == np.float64:
            return np.floor(p * np.float64(self.inv_vs)).astype(np.int64)
        assert p.dtype == np.float32
        return np.floor(p * self.inv_vs).astype(np.int64)

    def integrate(self, points, colors=None):
        p = np.asarray(points)
        if len(p) == 0:
            return
        vk = self.voxel_keys(p)
        allk, inv = np.unique(np.concatenate([self.keys, vk]), axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        old, new = inv[:len(self.keys)], inv[len(self.keys):]
        count = np.zeros(len(allk), np.int64)
        pos = np.zeros((len(allk), 3), np.float32)
        col = np.zeros((len(allk), 3), np.float32)
        count[old], pos[old], col[old] = self.count, self.pos, self.col
        np.add.at(count, new, 1)
        np.add.at(pos, new, p.astype(np.float32))
        if colors is not None:
            c = np.asarray(colors)
            c = c.astype(np.float32) * (np.float32(1.0) / np.float32(255.0)) if c.dtype == np.uint8 else \
                c.astype(np.float32)
            np.add.at(col, new, c)
        self.keys, self.count, self.pos, self.col = allk, count, pos, col

    def block_keys(self):
        return np.unique(self.keys // 8, axis=0).astype(np.int32).reshape(-1, 3)

    def dump(self):
        """Like `sort_dump(grid.dump_blocks())` without the hashes: keys [nb,3] sorted, count [nb,512],
        pos_sum / col_sum [nb,512,3]."""
        bk = self.block_keys()
        nb = len(bk)
        count = np.zeros((nb, 512), np.int32)
        pos = np.zeros((nb, 512, 3), np.float32)
        col = np.zeros((nb, 512, 3), np.float32)
        if nb:
            b = np.searchsorted(self._block_ids(bk), self._block_ids(self.keys // 8))
            lk = self.keys - (self.keys // 8) * 8
            l = lk[:, 0] + 8 * lk[:, 1] + 64 * lk[:, 2]
            count[b, l], pos[b, l], col[b, l] = self.count, self.pos, self.col
        return dict(keys=bk, count=count, pos_sum=pos, col_sum=col)

    @staticmethod
    def _block_ids(k):
        k = np.asarray(k, np.int64) + (1 << 20)
        return (k[:, 0] << 42) | (k[:, 1] << 21) | k[:, 2]

    def remove_low_count_voxels(self, min_count):
        low = self.count < min_count
        self.count[low] = 0
        self.pos[low] = 0
        self.col[low] = 0

    def _means(self, sel):
        c = self.count[sel].astype(np.float32)[:, None]
        return self.pos[sel] / c, self.col[sel] / c

    def get_voxels(self, min_count=1):
        """(points, colours) of the voxels with count >= min_count (min_count >= 1), in voxel-key order."""
        return self._means(self.count >= min_count)

    def _key_bounds(self, bb):
        bb = np.asarray(bb, np.float64)
        return (np.floor(bb[:3] * np.float64(self.inv_vs)).astype(np.int64),
                np.floor(bb[3:] * np.float64(self.inv_vs)).astype(np.int64))

    def _in_keys(self, bb, min_count):
        lo, hi = self._key_bounds(bb)
        return (self.count >= min_count) & np.all((self.keys >= lo) & (self.keys <= hi), axis=1)

    def get_voxels_in_bb(self, bbox, min_count=1):
        bb = np.asarray(bbox, np.float64).reshape(6)
        sel = np.flatnonzero(self._in_keys(bb, min_count))
        p, c = self._means(sel)
        q = p.astype(np.float64)
        ok = np.all((q >= bb[:3]) & (q <= bb[3:]), axis=1)
        return p[ok], c[ok]

    @staticmethod
    def frustum_bounds(K, W, H, Tcw, depth_max, depth_min):
        """BlockGridCore::frustum_query: the world AABB [6] of the 8 frustum corners, float64, in the kernel's order."""
        fx, fy, cx, cy = [np.float64(np.float32(v)) for v in K]
        T = np.asarray(Tcw, np.float64).reshape(4, 4)
        R, t = T[:3, :3], T[:3, 3]
        twc = [-((R[0, i] * t[0] + R[1, i] * t[1]) + R[2, i] * t[2]) for i in range(3)]
        lo, hi = np.full(3, 1e300), np.full(3, -1e300)
        for u, v in ((0.0, 0.0), (float(W), 0.0), (float(W), float(H)), (0.0, float(H))):
            xn, yn = (u - cx) / fx, (v - cy) / fy
            for d in (np.float64(np.float32(depth_min)), np.float64(np.float32(depth_max))):
                pc = (xn * d, yn * d, d)
                for a in range(3):
                    w = ((R[0, a] * pc[0] + R[1, a] * pc[1]) + R[2, a] * pc[2]) + twc[a]
                    lo[a], hi[a] = min(lo[a], w), max(hi[a], w)
        return np.concatenate([lo, hi])

    @staticmethod
    def project(points, K, W, H, Tcw, depth_max, depth_min):
        """CameraFrustrum::contains on float32 points -> (inside, u, v, depth) with u, v, depth float32."""
        return numpy_grid.project64(np.asarray(points, np.float32).astype(np.float64), K, W, H, Tcw, depth_max,
                                    depth_min)

    @staticmethod
    def project64(points, K, W, H, Tcw, depth_max, depth_min):
        """`project` on float64 points (the semantic grids' float64 means)."""
        fx, fy, cx, cy = [np.float64(np.float32(v)) for v in K]
        T = np.asarray(Tcw, np.float64).reshape(4, 4)
        p = np.asarray(points, np.float64).reshape(-1, 3)
        pc = [((T[a, 0] * p[:, 0] + T[a, 1] * p[:, 1]) + T[a, 2] * p[:, 2]) + T[a, 3] for a in range(3)]
        depth = pc[2].astype(np.float32)
        with np.errstate(divide="ignore", invalid="ignore"):
            u = (fx * (pc[0] / pc[2]) + cx).astype(np.float32)
            v = (fy * (pc[1] / pc[2]) + cy).astype(np.float32)
        ok = (depth >= np.float32(depth_min)) & (depth <= np.float32(depth_max))
        ok &= (u >= 0) & (u < np.float32(W)) & (v >= 0) & (v < np.float32(H))
        return ok, u, v, depth

    def _frustum_select(self, K, W, H, Tcw, depth_max, depth_min, min_count):
        bb = self.frustum_bounds(K, W, H, Tcw, depth_max, depth_min)
        sel = np.flatnonzero(self._in_keys(bb, min_count))
        p, c = self._means(sel)
        ok, u, v, depth = self.project(p, K, W, H, Tcw, depth_max, depth_min)
        return sel[ok], p[ok], c[ok], u[ok], v[ok], depth[ok]

    def get_voxels_in_frustum(self, K, W, H, Tcw, depth_max=10.0, depth_min=1e-2, min_count=1):
        _, p, c, _, _, _ = self._frustum_select(K, W, H, Tcw, depth_max, depth_min, min_count)
        return p, c

    def carve(self, K, W, H, Tcw, depth_image, depth_threshold, depth_max=10.0, depth_min=1e-2):
        """Resets the carved voxels; returns their indices into `keys`."""
        sel, _, _, u, v, depth = self._frustum_select(K, W, H, Tcw, depth_max, depth_min, 1)
        img = np.asarray(depth_image, np.float32)[v.astype(np.int64), u.astype(np.int64)]
        with np.errstate(invalid="ignore"):
            cut = (img > 0) & np.isfinite(img) & (depth < img - np.float32(depth_threshold))
        gone = sel[cut]
        self.count[gone] = 0
        self.pos[gone] = 0
        self.col[gone] = 0
        return gone


class numpy_semantic_grid:
    """The semantic block grids `VoxelBlockSemanticGrid` (kind="voting") and `VoxelBlockSemanticProbabilisticGrid`
    (kind="probabilistic") of b2v_semantic.cu restated voxel by voxel in plain Python / numpy.  Every float32
    operation is one np.float32 operation; exp and log are evaluated in float64 and rounded to float32.

    keys       as numpy_grid (voxel_hashing.h:69-75, voxel_block_grid.hpp:473); a block exists once a point lands in it
               and holds 512 voxels in the cleared state: count 0, sums 0, object = class = -1, counter 0, no label
               slots, ml_logp = -inf, confidence 0
    per point  in input order (voxel_block_grid.hpp:12-112, 220-288, 524-614):
                 labels (below) when the call has class ids AND colours (no colours: positions only, hpp:228-231);
                 the object id is the instance id, or 0 without instance ids (hpp:259-286)
                 pos_sum += float64(x) (voxel_data.h:53-57); col_sum += c in float32, c = float32 colour or
                 float32(u8) * float32(1/255) (voxel_data.h:79-90); count += 1
    voting     (voxel_data_semantic.h:153-198) an observation with depth >= depth_threshold is ignored; otherwise
               count == 0: take the label, counter = 1; same label: counter += 1; other label: counter -= 1 and at
               counter <= 0 take the label with counter = 1.  confidence = min(1, float32(counter) / float32(count))
               (:117-132), 0 for an empty voxel
    Bayesian   (voxel_data_semantic.h:312-451) evidence w = -log(0.9) as float32 (:287) for depth <= depth_threshold or
               no depth, else float32(exp(float32(-(depth - threshold)) * rate)) * -log(0.9).
               count == 0: slot[label] = w, argmax = label, ml_logp = w.  Known label: slot += w; if it is the argmax
               ml_logp follows it, else it takes the argmax only when strictly larger than ml_logp (ties keep the
               earlier label).  New label: slot = w, argmax when w > ml_logp.
               The reference keeps a std::map; the kernel keeps 8 slots in insertion order.  A ninth distinct label
               replaces the slot with the least evidence that is not the argmax (the first such slot on ties) and
               counts one label overflow: the kernel's own rule, not the reference's.
               confidence (:561-570, 607-624): 0 when the argmax has a -1 id or there is no slot, else
               exp(ml_logp - logsumexp) with the sum folded over the slots in ascending (object, class) order by
               log_add_exp(a, b) = m + log(exp(a - m) + exp(b - m)), m = max(a, b) (:626-635); evaluated for every
               voxel a labelled call touched, at the end of the call
    read-outs  count >= min_count and confidence >= min_confidence (voxel_block_grid.hpp:797-803); mean position
               pos_sum / float64(count), mean colour col_sum / float32(count) (voxel_data.h:58-69, 98-109).  Box
               (hpp:822-1016) and frustum (:1019-1195, 1336-1460): count >= 1, the key bounds and the fine test of
               numpy_grid on the float64 mean
    edits      applied to every voxel of every block, empty ones included (voxel_block_grid.hpp:625-647,
               voxel_block_semantic_grid.hpp:101-183): remove_low_count_voxels(n) resets count < n;
               remove_low_confidence_segments(int n) resets confidence < float32(n); remove_segment(id) resets
               object == id; merge_segments(a, b) gives every voxel with object == b the object a, and a Bayesian voxel
               then holds the single slot (a, class) with evidence 0, ml_logp 0 and confidence 1 when a >= 0 and
               class >= 0, else no slot, ml_logp -inf and confidence 0 (set_object_id, voxel_data_semantic.h:135,
               455-460, 589-605).  -1 is also the object id of every empty voxel.  Reset = the cleared state.
    carve      voxel_grid_carving.h:47-80, as numpy_grid.carve
    association  assign_object_ids_to_instance_ids (voxel_semantic_data_association.h:69-373): every voxel in the
               frustum looks up its truncated pixel; skipped when the pixel's class < 0, the voxel's class < 0 or
               differs, the pixel's instance < 0, or (with a depth image) the image depth is <= 0 or not finite;
               with carving, depth < image - thr resets the voxel; depth > image + thr is skipped.  A voxel without
               object id takes object 0 at once for instance 0, else is pending.  Each remaining voxel votes
               (instance -> its object).  Instances with pending voxels get new object ids in ascending instance
               order (the reference: block-iteration order), the pending votes count for them.  Winner per instance:
               the most votes, the lowest object id on ties (:287-320); -1 when total < min_votes or
               float32(max) / float32(total) < min_vote_ratio.  Every pixel with instance >= 0 and class >= 0 adds
               its instance with -1 if absent, and instance 0 maps to 0 (:322-352).  Pending voxels whose instance
               won an id >= 0 take it (:354-370).
    `dump()` has the layout of `sort_dump(grid.dump_blocks(8))` without the hashes: `aux` is the voting counter or the
    number of slots, `lab_*` the slots in ascending (object, class) order padded with (-1, -1, -inf); dump_blocks never
    shows the kernel's stale slots past `aux`.  The class neither loads nor calls the CUDA library."""

    MAX_LABELS = 8
    BASE_LOG = np.float32(0.10536051565782628)   # voxel_data_semantic.h:287

    def __init__(self, voxel_size, kind="voting"):
        assert kind in ("voting", "probabilistic")
        self.bayes = kind == "probabilistic"
        self.inv_vs = np.float32(1.0) / np.float32(voxel_size)
        self.depth_threshold = np.float32(5.0 if self.bayes else 10.0)   # voxel_data_semantic.h:107-108, 251-254
        self.depth_decay_rate = np.float32(0.07)
        self.next_object_id = 1
        self.clear()

    def set_depth_threshold(self, v):
        self.depth_threshold = np.float32(v)

    def set_depth_decay_rate(self, v):
        if self.bayes:
            self.depth_decay_rate = np.float32(v)

    def set_next_object_id(self, v):
        self.next_object_id = int(v)

    def clear(self):
        self.block_of = {}                      # block key -> row of the arrays below
        self.keys = np.zeros((0, 3), np.int64)
        self.count = np.zeros((0, 512), np.int64)
        self.pos = np.zeros((0, 512, 3), np.float64)
        self.col = np.zeros((0, 512, 3), np.float32)
        self.obj = np.zeros((0, 512), np.int32)
        self.cls = np.zeros((0, 512), np.int32)
        self.counter = np.zeros((0, 512), np.int32)
        self.ml_logp = np.zeros((0, 512), np.float32)
        self.conf = np.zeros((0, 512), np.float32)
        self.slots = {}                         # (row, voxel) -> [[object, class, float32 evidence], ...]
        self.label_overflows = 0

    def _add_blocks(self, block_keys):
        new = [k for k in dict.fromkeys(map(tuple, block_keys.tolist())) if k not in self.block_of]
        if not new:
            return
        for k in new:
            self.block_of[k] = len(self.block_of)
        m = len(new)
        self.keys = np.concatenate([self.keys, np.array(new, np.int64).reshape(m, 3)])
        self.count = np.concatenate([self.count, np.zeros((m, 512), np.int64)])
        self.pos = np.concatenate([self.pos, np.zeros((m, 512, 3), np.float64)])
        self.col = np.concatenate([self.col, np.zeros((m, 512, 3), np.float32)])
        self.obj = np.concatenate([self.obj, np.full((m, 512), -1, np.int32)])
        self.cls = np.concatenate([self.cls, np.full((m, 512), -1, np.int32)])
        self.counter = np.concatenate([self.counter, np.zeros((m, 512), np.int32)])
        self.ml_logp = np.concatenate([self.ml_logp, np.full((m, 512), -np.inf, np.float32)])
        self.conf = np.concatenate([self.conf, np.zeros((m, 512), np.float32)])

    # ---- float32 helpers ----
    @staticmethod
    def _exp(x):
        return np.float32(np.exp(np.float64(x)))

    @staticmethod
    def _log(x):
        return np.float32(np.log(np.float64(x)))

    @classmethod
    def _log_add_exp(cls, a, b):
        if a == -np.inf:
            return b
        if b == -np.inf:
            return a
        m = max(a, b)
        return np.float32(m + cls._log(np.float32(cls._exp(np.float32(a - m)) + cls._exp(np.float32(b - m)))))

    def _confidence_of(self, slots, obj, cls, ml):
        if obj == -1 or cls == -1 or not slots:
            return np.float32(0.0)
        total = np.float32(-np.inf)
        for _, _, lp in sorted(slots, key=lambda s: (s[0], s[1])):
            total = self._log_add_exp(total, lp)
        return self._exp(np.float32(ml - total))

    def _weight(self, depth):
        if depth is None or depth <= self.depth_threshold:
            return self.BASE_LOG
        e = self._exp(np.float32(np.float32(-np.float32(depth - self.depth_threshold)) * self.depth_decay_rate))
        return np.float32(e * self.BASE_LOG)

    # ---- integrate ----
    def integrate(self, points, colors=None, class_ids=None, instance_ids=None, depths=None):
        p = np.asarray(points)
        assert p.dtype in (np.float32, np.float64) and p.ndim == 2 and p.shape[1] == 3
        n = len(p)
        if n == 0:
            return
        inv = np.float64(self.inv_vs) if p.dtype == np.float64 else self.inv_vs
        vk = np.floor(p * inv).astype(np.int64)
        bk = vk // 8
        self._add_blocks(bk)
        lk = vk - bk * 8
        local = (lk[:, 0] + 8 * lk[:, 1] + 64 * lk[:, 2]).tolist()
        rows = [self.block_of[k] for k in map(tuple, bk.tolist())]
        c = None
        if colors is not None:
            c = np.asarray(colors)
            c = c.astype(np.float32) * (np.float32(1.0) / np.float32(255.0)) if c.dtype == np.uint8 else \
                c.astype(np.float32)
        semantics = class_ids is not None and c is not None
        assert instance_ids is None or class_ids is not None
        oc = None if class_ids is None else np.asarray(class_ids, np.int32).tolist()
        oo = None if instance_ids is None else np.asarray(instance_ids, np.int32).tolist()
        dep = None if depths is None else np.asarray(depths, np.float32)
        p64 = p.astype(np.float64)
        touched = set()
        for i in range(n):
            b, l = rows[i], local[i]
            if semantics:
                label = (oo[i] if oo is not None else 0, oc[i])
                d = None if dep is None else dep[i]
                if self.bayes:
                    self._observe_bayes(b, l, label, d)
                    touched.add((b, l))
                else:
                    self._observe_vote(b, l, label, d)
            self.pos[b, l] += p64[i]
            if c is not None:
                self.col[b, l] += c[i]
            self.count[b, l] += 1
        for b, l in touched:
            self.conf[b, l] = self._confidence_of(self.slots.get((b, l), []), self.obj[b, l], self.cls[b, l],
                                                  self.ml_logp[b, l])

    def integrate_segment(self, points, colors, class_id, object_id):
        """voxel_block_semantic_grid.hpp:52-99: one label for every point; a negative id skips the segment."""
        n = len(points)
        if class_id < 0 or object_id < 0 or n == 0:
            return
        self.integrate(points, colors, np.full(n, class_id, np.int32), np.full(n, object_id, np.int32))

    def _observe_vote(self, b, l, label, depth):
        if depth is not None and not depth < self.depth_threshold:
            return
        if self.count[b, l] == 0:
            self.obj[b, l], self.cls[b, l], self.counter[b, l] = label[0], label[1], 1
        elif (self.obj[b, l], self.cls[b, l]) == label:
            self.counter[b, l] += 1
        else:
            self.counter[b, l] -= 1
            if self.counter[b, l] <= 0:
                self.obj[b, l], self.cls[b, l], self.counter[b, l] = label[0], label[1], 1

    def _observe_bayes(self, b, l, label, depth):
        w = self._weight(depth)
        slots = self.slots.setdefault((b, l), [])
        arg = (int(self.obj[b, l]), int(self.cls[b, l]))
        k = next((q for q, s in enumerate(slots) if (s[0], s[1]) == label), None)
        if self.count[b, l] == 0:
            if k is None:
                slots.append([label[0], label[1], w])
            else:
                slots[k][2] = w
            self.obj[b, l], self.cls[b, l], self.ml_logp[b, l] = label[0], label[1], w
        elif k is not None:
            slots[k][2] = np.float32(slots[k][2] + w)
            if label == arg:
                self.ml_logp[b, l] = slots[k][2]
            elif slots[k][2] > self.ml_logp[b, l]:
                self.obj[b, l], self.cls[b, l], self.ml_logp[b, l] = label[0], label[1], slots[k][2]
        else:
            if len(slots) < self.MAX_LABELS:
                slots.append([label[0], label[1], w])
            else:
                weakest = None
                for q, s in enumerate(slots):
                    if (s[0], s[1]) != arg and (weakest is None or s[2] < slots[weakest][2]):
                        weakest = q
                slots[weakest] = [label[0], label[1], w]
                self.label_overflows += 1
            if w > self.ml_logp[b, l]:
                self.obj[b, l], self.cls[b, l], self.ml_logp[b, l] = label[0], label[1], w

    # ---- read-outs ----
    def confidence(self):
        """[nb, 512] float32: the read-out confidence of every voxel."""
        if self.bayes:
            return np.where(self.count > 0, self.conf, np.float32(0.0)).astype(np.float32)
        with np.errstate(divide="ignore", invalid="ignore"):
            q = self.counter.astype(np.float32) / self.count.astype(np.float32)
        return np.where(self.count > 0, np.minimum(np.float32(1.0), q), np.float32(0.0)).astype(np.float32)

    def _voxel_keys(self):
        l = np.arange(512)
        return self.keys[:, None, :] * 8 + np.stack([l % 8, (l // 8) % 8, l // 64], 1)[None]

    def _means(self):
        with np.errstate(divide="ignore", invalid="ignore"):
            return self.pos / self.count.astype(np.float64)[..., None]

    def _collect(self, sel):
        c = self.count[sel]
        with np.errstate(divide="ignore", invalid="ignore"):
            pts = np.where(c[:, None] > 0, self.pos[sel] / c.astype(np.float64)[:, None], 0.0)
            cols = np.where(c[:, None] > 0, self.col[sel] / c.astype(np.float32)[:, None], np.float32(0.0))
        return dict(points=pts, colors=cols.astype(np.float32), class_ids=self.cls[sel], object_ids=self.obj[sel],
                    confidences=self.confidence()[sel])

    def _keep(self, min_count, min_confidence):
        return (self.count >= min_count) & (self.confidence() >= np.float32(min_confidence))

    def get_voxels(self, min_count=1, min_confidence=0.0):
        return self._collect(self._keep(min_count, min_confidence))

    def _in_bounds(self, bb):
        bb = np.asarray(bb, np.float64)
        lo = np.floor(bb[:3] * np.float64(self.inv_vs)).astype(np.int64)
        hi = np.floor(bb[3:] * np.float64(self.inv_vs)).astype(np.int64)
        vk = self._voxel_keys()
        return (self.count >= 1) & np.all((vk >= lo) & (vk <= hi), axis=-1)

    def _in_box(self, bbox):
        bb = np.asarray(bbox, np.float64).reshape(6)
        m = self._means()
        with np.errstate(invalid="ignore"):
            return self._in_bounds(bb) & np.all((m >= bb[:3]) & (m <= bb[3:]), axis=-1)

    def _in_frustum(self, K, W, H, Tcw, depth_max, depth_min):
        """(inside [nb,512], u, v, depth [nb,512] float32)."""
        sel = self._in_bounds(numpy_grid.frustum_bounds(K, W, H, Tcw, depth_max, depth_min))
        ok, u, v, depth = numpy_grid.project64(self._means().reshape(-1, 3), K, W, H, Tcw, depth_max, depth_min)
        shape = self.count.shape
        return sel & ok.reshape(shape), u.reshape(shape), v.reshape(shape), depth.reshape(shape)

    def get_voxels_in_bb(self, bbox, min_count=1, min_confidence=0.0):
        return self._collect(self._keep(min_count, min_confidence) & self._in_box(bbox))

    def get_voxels_in_camera_frustrum(self, K, W, H, Tcw, depth_max, depth_min, min_count=1, min_confidence=0.0):
        return self._collect(self._keep(min_count, min_confidence) &
                             self._in_frustum(K, W, H, Tcw, depth_max, depth_min)[0])

    # ---- edits ----
    def _reset(self, sel):
        self.count[sel] = 0
        self.pos[sel] = 0
        self.col[sel] = 0
        self.obj[sel] = -1
        self.cls[sel] = -1
        self.counter[sel] = 0
        self.ml_logp[sel] = -np.inf
        self.conf[sel] = 0
        for b, l in zip(*np.nonzero(sel)):
            self.slots.pop((int(b), int(l)), None)

    def remove_low_count_voxels(self, min_count):
        self._reset(self.count < int(min_count))

    def remove_low_confidence_segments(self, min_confidence):
        self._reset(self.confidence() < np.float32(int(min_confidence)))

    def remove_segment(self, object_id):
        self._reset(self.obj == int(object_id))

    def _set_object_id(self, sel, object_id):
        self.obj[sel] = object_id
        if not self.bayes:
            return
        for b, l in zip(*np.nonzero(sel)):
            b, l = int(b), int(l)
            if object_id >= 0 and self.cls[b, l] >= 0:
                self.slots[(b, l)] = [[object_id, int(self.cls[b, l]), np.float32(0.0)]]
                self.ml_logp[b, l], self.conf[b, l] = 0.0, 1.0
            else:
                self.slots.pop((b, l), None)
                self.ml_logp[b, l], self.conf[b, l] = -np.inf, 0.0

    def merge_segments(self, a, b):
        self._set_object_id(self.obj == int(b), int(a))

    def carve(self, K, W, H, Tcw, depth_max, depth_min, depth_image, depth_threshold):
        ok, u, v, depth = self._in_frustum(K, W, H, Tcw, depth_max, depth_min)
        img = np.zeros(ok.shape, np.float32)
        img[ok] = np.asarray(depth_image, np.float32)[v[ok].astype(np.int64), u[ok].astype(np.int64)]
        with np.errstate(invalid="ignore"):
            self._reset(ok & (img > 0) & np.isfinite(img) & (depth < img - np.float32(depth_threshold)))

    def assign_object_ids_to_instance_ids(self, K, W, H, Tcw, depth_max, depth_min, class_image, instance_image,
                                          depth_image=None, depth_threshold=0.1, do_carving=False, min_vote_ratio=0.5,
                                          min_votes=3):
        ci, ii = np.asarray(class_image, np.int32), np.asarray(instance_image, np.int32)
        di = None if depth_image is None else np.asarray(depth_image, np.float32)
        thr = np.float32(depth_threshold)
        ok, u, v, depth = self._in_frustum(K, W, H, Tcw, depth_max, depth_min)
        votes, pending, carved = {}, [], np.zeros(ok.shape, bool)
        for b, l in zip(*np.nonzero(ok)):
            r, c = int(v[b, l]), int(u[b, l])
            if ci[r, c] < 0 or self.cls[b, l] < 0 or self.cls[b, l] != ci[r, c] or ii[r, c] < 0:
                continue
            inst, obj = int(ii[r, c]), int(self.obj[b, l])
            if di is not None:
                d = di[r, c]
                if not (d > 0 and np.isfinite(d)):
                    continue
                if do_carving and depth[b, l] < np.float32(d - thr):
                    carved[b, l] = True
                    continue
                if depth[b, l] > np.float32(d + thr):
                    continue
            if obj < 0:
                if inst == 0:
                    one = np.zeros(ok.shape, bool)
                    one[b, l] = True
                    self._set_object_id(one, 0)
                    obj = 0
                else:
                    pending.append((b, l, inst))
                    obj = None
            per = votes.setdefault(inst, {})
            per[obj] = per.get(obj, 0) + 1
        self._reset(carved)
        new_id = {}
        for inst in sorted({inst for _, _, inst in pending}):
            new_id[inst] = self.next_object_id
            self.next_object_id += 1
        result = {}
        for inst in sorted(votes):
            per = {}
            for obj, cnt in votes[inst].items():
                o = new_id[inst] if obj is None else obj
                per[o] = per.get(o, 0) + cnt
            best, winner, total = 0, -1, 0
            for o in sorted(per):
                total += per[o]
                if per[o] > best:
                    best, winner = per[o], o
            low = total < int(min_votes) or np.float32(best) / np.float32(total) < np.float32(min_vote_ratio)
            result[inst] = -1 if low else winner
        for inst in np.unique(ii[(ii >= 0) & (ci >= 0)]).tolist():
            if inst == 0:
                result[0] = 0
            else:
                result.setdefault(inst, -1)
        for b, l, inst in pending:
            if result[inst] >= 0:
                one = np.zeros(ok.shape, bool)
                one[b, l] = True
                self._set_object_id(one, result[inst])
        return dict(sorted(result.items()))

    def dump(self):
        order = np.lexsort((self.keys[:, 2], self.keys[:, 1], self.keys[:, 0]))
        nb, K = len(order), self.MAX_LABELS
        lab_obj = np.full((nb, 512, K), -1, np.int32)
        lab_cls = np.full((nb, 512, K), -1, np.int32)
        lab_logp = np.full((nb, 512, K), -np.inf, np.float32)
        aux = self.counter.copy()
        if self.bayes:
            aux[:] = 0
            for (b, l), slots in self.slots.items():
                aux[b, l] = len(slots)
                for k, (o, c, lp) in enumerate(sorted(slots, key=lambda s: (s[0], s[1]))):
                    lab_obj[b, l, k], lab_cls[b, l, k], lab_logp[b, l, k] = o, c, lp
        conf = self.conf if self.bayes else self.confidence()
        d = dict(keys=self.keys.astype(np.int32), count=self.count.astype(np.int32), pos_sum=self.pos,
                 col_sum=self.col, object_id=self.obj, class_id=self.cls, confidence=conf, aux=aux,
                 lab_obj=lab_obj, lab_cls=lab_cls, lab_logp=lab_logp)
        return {k: a[order].copy() for k, a in d.items()}


def numpy_shadow_filter(depth, delta_x=2, delta_y=2, fill_value=-1.0):
    """`filter_shadow_points(depth, delta_depth=None)` (pyslam/utilities/depth.py:103-146) restated in numpy 2:
    deltas |d[dy:] - d[:-dy]| and |d[:, dx:] - d[:, :-dx]| in float32, threshold 3 * (1.4826 * median of the
    positive deltas) in float32 (NaN without positive deltas: nothing is filtered), both pixels of an
    over-threshold pair set to fill_value.  Returns (filtered, threshold)."""
    d = np.asarray(depth, np.float32)
    assert d.ndim == 2 and 1 <= delta_y < d.shape[0] and 1 <= delta_x < d.shape[1]
    with np.errstate(invalid="ignore"):
        dv = np.abs(d[delta_y:] - d[:-delta_y])
        dh = np.abs(d[:, delta_x:] - d[:, :-delta_x])
        vals = np.concatenate([dv.ravel(), dh.ravel()])
        pos = vals[vals > 0]
        mad = np.median(pos) if len(pos) else np.float32(np.nan)
        thr = np.float32(3.0) * (np.float32(1.4826) * np.float32(mad))
        mv, mh = dv > thr, dh > thr
    mask = np.zeros(d.shape, bool)
    mask[delta_y:] |= mv
    mask[:-delta_y] |= mv
    mask[:, delta_x:] |= mh
    mask[:, :-delta_x] |= mh
    return np.where(mask, np.float32(fill_value), d), thr


def numpy_integrate_block(vox, key, depth, color, K, Tcw, voxel_size, sdf_trunc, depth_trunc,
                          block_size=8):
    """A.3 update of one block in float32 numpy (no FMA, true divisions): an independent second
    restatement.  vox: f32 [5, B^3] -> new f32 [5, B^3]."""
    B = block_size
    f32 = np.float32
    vs, tau = f32(voxel_size), f32(sdf_trunc)
    fx, fy, cx, cy = [f32(v) for v in K]
    E = np.asarray(Tcw, np.float64).reshape(4, 4).astype(np.float32)
    H, W = depth.shape
    l = np.arange(B ** 3)
    lx, ly, lz = l % B, (l // B) % B, l // (B * B)
    c = np.stack([(f32(key[0] * B) + lx.astype(np.float32) + f32(0.5)) * vs,
                  (f32(key[1] * B) + ly.astype(np.float32) + f32(0.5)) * vs,
                  (f32(key[2] * B) + lz.astype(np.float32) + f32(0.5)) * vs], axis=1)
    p = (c.astype(np.float64) @ E[:3, :3].astype(np.float64).T + E[:3, 3].astype(np.float64))
    p = p.astype(np.float32)
    out = np.array(vox, dtype=np.float32, copy=True)
    pz = p[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        u_f = p[:, 0] * fx / pz + cx + f32(0.5)
        v_f = p[:, 1] * fy / pz + cy + f32(0.5)
    ok = (pz > 0) & (u_f >= f32(0.0001)) & (u_f < f32(W) - f32(0.0001)) & \
         (v_f >= f32(0.0001)) & (v_f < f32(H) - f32(0.0001))
    u = np.where(ok, u_f, 0).astype(np.int64)
    v = np.where(ok, v_f, 0).astype(np.int64)
    d = depth[v, u].astype(np.float32)
    ok &= (d > 0) & (d < f32(depth_trunc))
    xx = (u.astype(np.float32) - cx) / fx
    yy = (v.astype(np.float32) - cy) / fy
    lam = np.sqrt(xx * xx + yy * yy + f32(1.0))
    sdf = (d - pz) * lam
    ok &= sdf > -tau
    t = np.minimum(f32(1.0), sdf / tau)
    w = out[1]
    wn = w + f32(1.0)
    rgb = color[v, u].astype(np.float32)
    new_t = (out[0] * w + t) / wn
    out[0] = np.where(ok, new_t, out[0])
    for k in range(3):
        out[2 + k] = np.where(ok, (out[2 + k] * w + rgb[:, k]) / wn, out[2 + k])
    out[1] = np.where(ok, wn, w)
    return out, ok


# ---------------------------------------------------------------------------------------------
# compiled reference: semantic voxel-block grids (SURVEY.md §8(f) rank 2)
# ---------------------------------------------------------------------------------------------
_EIGEN_SO = os.path.join(_DIR, "_ref", "libeigen_ops.so")


def have_eigen_ops() -> bool:
    return os.path.exists(_EIGEN_SO)


class EigenOps:
    """The three Eigen expressions of Open3D's TSDF path, evaluated by the Eigen vendored in the reference tree
    (oracle/eigen_ops.cpp; x86-64 baseline like Open3D's wheels).  Row-major numpy in and out."""

    def __init__(self):
        if not have_eigen_ops():
            raise RuntimeError("oracle/_ref/libeigen_ops.so missing (needs /root/reference to build)")
        self._L = C.CDLL(_EIGEN_SO)
        self.version = int(self._L.eig_version())

    def mat4f_times_vec4f(self, M, v):
        M = np.ascontiguousarray(M, np.float32).reshape(4, 4)
        v = np.ascontiguousarray(v, np.float32).reshape(4)
        out = np.zeros(4, np.float32)
        self._L.eig_mat4f_times_vec4f(C.c_void_p(M.ctypes.data), C.c_void_p(v.ctypes.data), C.c_void_p(out.ctypes.data))
        return out

    def mat4d_times_vec4d(self, M, v):
        M = np.ascontiguousarray(M, np.float64).reshape(4, 4)
        v = np.ascontiguousarray(v, np.float64).reshape(4)
        out = np.zeros(4, np.float64)
        self._L.eig_mat4d_times_vec4d(C.c_void_p(M.ctypes.data), C.c_void_p(v.ctypes.data), C.c_void_p(out.ctypes.data))
        return out

    def mat4d_inverse(self, M):
        M = np.ascontiguousarray(M, np.float64).reshape(4, 4)
        out = np.zeros((4, 4), np.float64)
        self._L.eig_mat4d_inverse(C.c_void_p(M.ctypes.data), C.c_void_p(out.ctypes.data))
        return out


def open3d_order_inverse4(M):
    """The float64 cofactor inverse oracle/open3d_order.c uses for camera_pose = extrinsic.inverse()."""
    L = _o3d()
    M = np.ascontiguousarray(M, np.float64).reshape(4, 4)
    out = np.zeros((4, 4), np.float64)
    L.o3d_inverse4(C.c_void_p(M.ctypes.data), C.c_void_p(out.ctypes.data))
    return out


_SEM_SO = os.path.join(_DIR, "_ref", "libref_semantic.so")
_sem_lib = None


def have_ref_semantic() -> bool:
    return os.path.exists(_SEM_SO)


def _sem():
    global _sem_lib
    if _sem_lib is None:
        if not have_ref_semantic():
            raise RuntimeError("oracle/_ref/libref_semantic.so missing (needs /root/reference to build)")
        L = C.CDLL(_SEM_SO)
        vp = C.c_void_p
        L.refsem_create.restype = vp
        L.refsem_create.argtypes = [C.c_int, C.c_double, C.c_int]
        L.refsem_destroy.argtypes = [vp]
        L.refsem_clear.argtypes = [vp]
        L.refsem_set_depth_threshold.argtypes = [C.c_int, C.c_float]
        L.refsem_set_depth_decay_rate.argtypes = [C.c_float]
        L.refsem_get_depth_threshold.restype = C.c_float
        L.refsem_get_depth_threshold.argtypes = [C.c_int]
        L.refsem_get_depth_decay_rate.restype = C.c_float
        L.refsem_integrate.argtypes = [vp, _f64p, C.c_int64, vp, vp, vp, vp]
        L.refsem_integrate_f32.argtypes = [vp, _f32p, C.c_int64, vp, vp, vp, vp]
        L.refsem_num_blocks.restype = C.c_int64
        L.refsem_num_blocks.argtypes = [vp]
        L.refsem_dump_blocks.restype = C.c_int64
        L.refsem_dump_blocks.argtypes = [vp] * 10 + [C.c_int] + [vp] * 3
        L.refsem_get_voxels.restype = C.c_int64
        L.refsem_get_voxels.argtypes = [vp, C.c_int, C.c_float, vp, vp, vp, vp, vp]
        L.refsem_assign_object_ids.restype = C.c_int64
        L.refsem_assign_object_ids.argtypes = [vp, _f32p, C.c_int, C.c_int, _f64p, C.c_float, C.c_float, _i32p, _i32p,
                                               vp, C.c_float, C.c_int, C.c_float, C.c_int, _i32p, _i32p, C.c_int64]
        L.refsem_query.restype = C.c_int64
        L.refsem_query.argtypes = [vp, vp, C.c_int, C.c_int, vp, C.c_float, C.c_float, vp, C.c_int, C.c_float, vp, vp,
                                   vp, vp, vp]
        L.refsem_carve.argtypes = [vp, _f32p, C.c_int, C.c_int, _f64p, C.c_float, C.c_float, _f32p, C.c_float]
        L.refsem_set_next_object_id.argtypes = [C.c_int32]
        L.refsem_get_next_object_id.restype = C.c_int32
        L.refsem_integrate_segment.argtypes = [vp, _f64p, C.c_int64, _f32p, C.c_int, C.c_int]
        L.refsem_segments.restype = C.c_int64
        L.refsem_segments.argtypes = [vp, C.c_int, C.c_int, C.c_float] + [vp] * 8 + [C.POINTER(C.c_int64)]
        L.refsem_remove_low_count_voxels.argtypes = [vp, C.c_int]
        L.refsem_remove_low_confidence_segments.argtypes = [vp, C.c_int]
        L.refsem_merge_segments.argtypes = [vp, C.c_int, C.c_int]
        L.refsem_remove_segment.argtypes = [vp, C.c_int]
        _sem_lib = L
    return _sem_lib


class RefSemanticGrid:
    """The unmodified reference `VoxelBlockSemanticGrid` (kind="voting") or
    `VoxelBlockSemanticProbabilisticGrid` (kind="probabilistic"), sequential branch.  The depth threshold
    and decay rate are class-static in the reference (process-wide): set them right before use."""

    KINDS = {"voting": 0, "probabilistic": 1}

    def __init__(self, voxel_size: float, kind: str = "voting", block_size: int = 8):
        self._L = _sem()
        self.kind = self.KINDS[kind]
        self._h = self._L.refsem_create(self.kind, float(voxel_size), int(block_size))

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.refsem_destroy(self._h)
            self._h = None

    def set_depth_threshold(self, v):
        self._L.refsem_set_depth_threshold(self.kind, float(v))

    def set_depth_decay_rate(self, v):
        self._L.refsem_set_depth_decay_rate(float(v))

    def integrate(self, points, colors=None, class_ids=None, instance_ids=None, depths=None):
        """float32 points take the reference's float overload (keys computed in float32), anything else float64."""
        f32 = np.asarray(points).dtype == np.float32
        pts = np.ascontiguousarray(points, np.float32 if f32 else np.float64)
        n = pts.shape[0]
        cols = np.ascontiguousarray(colors if colors is not None else np.zeros((n, 3)), np.float32)
        hold = [pts, cols]

        def ptr(a, dt):
            if a is None:
                return None
            b = np.ascontiguousarray(a, dt)
            assert b.shape == (n,)
            hold.append(b)
            return b.ctypes.data

        fn = self._L.refsem_integrate_f32 if f32 else self._L.refsem_integrate
        fn(self._h, pts, n, cols.ctypes.data, ptr(class_ids, np.int32), ptr(instance_ids, np.int32),
           ptr(depths, np.float32))

    def integrate_segment(self, points, colors, class_id, object_id):
        pts = np.ascontiguousarray(points, np.float64)
        cols = np.ascontiguousarray(colors, np.float32)
        self._L.refsem_integrate_segment(self._h, pts.reshape(-1), pts.shape[0], cols.reshape(-1), int(class_id),
                                         int(object_id))

    def _segments(self, by_class, min_count, min_confidence):
        tot = C.c_int64(0)
        a = (self._h, int(by_class), int(min_count), float(min_confidence))
        n = self._L.refsem_segments(*a, None, None, None, None, None, None, None, None, C.byref(tot))
        ids, cls, npts = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int64)
        cmin, cmax, obb = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros((n, 10), np.float64)
        pts, cols = np.zeros((tot.value, 3), np.float64), np.zeros((tot.value, 3), np.float32)
        if n:
            self._L.refsem_segments(*a, ids.ctypes.data, cls.ctypes.data, npts.ctypes.data, cmin.ctypes.data,
                                    cmax.ctypes.data, obb.ctypes.data, pts.ctypes.data, cols.ctypes.data, C.byref(tot))
        out, off = [], 0
        for k in range(n):
            m = int(npts[k])
            out.append(dict(id=int(ids[k]), class_id=int(cls[k]), points=pts[off:off + m], colors=cols[off:off + m],
                            confidence_min=float(cmin[k]), confidence_max=float(cmax[k]), obb_center=obb[k, 0:3],
                            obb_size=obb[k, 3:6], obb_quat_wxyz=obb[k, 6:10]))
            off += m
        return out

    def get_object_segments(self, min_count=1, min_confidence=0.0):
        return self._segments(0, min_count, min_confidence)

    def get_class_segments(self, min_count=1, min_confidence=0.0):
        return self._segments(1, min_count, min_confidence)

    def num_blocks(self):
        return int(self._L.refsem_num_blocks(self._h))

    def clear(self):
        self._L.refsem_clear(self._h)

    def dump_blocks(self, K=8):
        nb, nv = self.num_blocks(), 512
        d = dict(keys=np.zeros((nb, 3), np.int32), hashes=np.zeros(nb, np.uint64),
                 count=np.zeros((nb, nv), np.int32), pos_sum=np.zeros((nb, nv, 3), np.float64),
                 col_sum=np.zeros((nb, nv, 3), np.float32), object_id=np.zeros((nb, nv), np.int32),
                 class_id=np.zeros((nb, nv), np.int32), confidence=np.zeros((nb, nv), np.float32),
                 aux=np.zeros((nb, nv), np.int32), lab_obj=np.zeros((nb, nv, K), np.int32),
                 lab_cls=np.zeros((nb, nv, K), np.int32), lab_logp=np.zeros((nb, nv, K), np.float32))
        a = d
        self._L.refsem_dump_blocks(self._h, a["keys"].ctypes.data, a["hashes"].ctypes.data, a["count"].ctypes.data,
                                   a["pos_sum"].ctypes.data, a["col_sum"].ctypes.data, a["object_id"].ctypes.data,
                                   a["class_id"].ctypes.data, a["confidence"].ctypes.data, a["aux"].ctypes.data,
                                   int(K), a["lab_obj"].ctypes.data, a["lab_cls"].ctypes.data,
                                   a["lab_logp"].ctypes.data)
        return d

    def get_voxels(self, min_count=1, min_confidence=0.0):
        n = self._L.refsem_get_voxels(self._h, int(min_count), float(min_confidence), None, None, None, None, None)
        out = dict(points=np.zeros((n, 3), np.float64), colors=np.zeros((n, 3), np.float32),
                   class_ids=np.zeros(n, np.int32), object_ids=np.zeros(n, np.int32),
                   confidences=np.zeros(n, np.float32))
        if n:
            self._L.refsem_get_voxels(self._h, int(min_count), float(min_confidence), out["points"].ctypes.data,
                                      out["colors"].ctypes.data, out["class_ids"].ctypes.data,
                                      out["object_ids"].ctypes.data, out["confidences"].ctypes.data)
        return out

    def assign_object_ids_to_instance_ids(self, K, width, height, Tcw, depth_max, depth_min, class_image,
                                          instance_image, depth_image=None, depth_threshold=0.1, do_carving=False,
                                          min_vote_ratio=0.5, min_votes=3):
        """-> dict instance id -> object id (voxel_semantic_data_association.h:69-373)."""
        K4 = np.ascontiguousarray(K, np.float32)
        T = np.ascontiguousarray(np.asarray(Tcw, np.float64).reshape(16))
        ci = np.ascontiguousarray(class_image, np.int32)
        ii = np.ascontiguousarray(instance_image, np.int32)
        di = None if depth_image is None else np.ascontiguousarray(depth_image, np.float32)
        ids, objs = np.zeros(4096, np.int32), np.zeros(4096, np.int32)
        n = self._L.refsem_assign_object_ids(self._h, K4, int(width), int(height), T, float(depth_max),
                                             float(depth_min), ci, ii, None if di is None else di.ctypes.data,
                                             float(depth_threshold), int(bool(do_carving)), float(min_vote_ratio),
                                             int(min_votes), ids, objs, 4096)
        assert n <= 4096
        return {int(i): int(o) for i, o in zip(ids[:n], objs[:n])}

    def _query(self, K, width, height, Tcw, depth_max, depth_min, bbox, min_count, min_confidence):
        kp = tp = bp = None
        hold = []
        if K is not None:
            K4 = np.ascontiguousarray(K, np.float32)
            T = np.ascontiguousarray(np.asarray(Tcw, np.float64).reshape(16))
            hold += [K4, T]
            kp, tp = K4.ctypes.data, T.ctypes.data
        else:
            bb = np.ascontiguousarray(bbox, np.float64).reshape(6)
            hold.append(bb)
            bp = bb.ctypes.data
        args = (self._h, kp, int(width), int(height), tp, float(depth_max), float(depth_min), bp, int(min_count),
                float(min_confidence))
        n = self._L.refsem_query(*args, None, None, None, None, None)
        out = dict(points=np.zeros((n, 3), np.float64), colors=np.zeros((n, 3), np.float32),
                   class_ids=np.zeros(n, np.int32), object_ids=np.zeros(n, np.int32),
                   confidences=np.zeros(n, np.float32))
        if n:
            self._L.refsem_query(*args, out["points"].ctypes.data, out["colors"].ctypes.data,
                                 out["class_ids"].ctypes.data, out["object_ids"].ctypes.data,
                                 out["confidences"].ctypes.data)
        return out

    def get_voxels_in_camera_frustrum(self, K, width, height, Tcw, depth_max, depth_min, min_count=1,
                                      min_confidence=0.0):
        return self._query(K, width, height, Tcw, depth_max, depth_min, None, min_count, min_confidence)

    def get_voxels_in_bb(self, bbox, min_count=1, min_confidence=0.0):
        return self._query(None, 0, 0, None, 0.0, 0.0, bbox, min_count, min_confidence)

    def carve(self, K, width, height, Tcw, depth_max, depth_min, depth_image, depth_threshold):
        self._L.refsem_carve(self._h, np.ascontiguousarray(K, np.float32), int(width), int(height),
                             np.ascontiguousarray(np.asarray(Tcw, np.float64).reshape(16)), float(depth_max),
                             float(depth_min), np.ascontiguousarray(depth_image, np.float32), float(depth_threshold))

    @staticmethod
    def set_next_object_id(v):
        _sem().refsem_set_next_object_id(int(v))

    @staticmethod
    def get_next_object_id():
        return int(_sem().refsem_get_next_object_id())

    def remove_low_count_voxels(self, min_count):
        self._L.refsem_remove_low_count_voxels(self._h, int(min_count))

    def remove_low_confidence_segments(self, min_confidence):
        self._L.refsem_remove_low_confidence_segments(self._h, int(min_confidence))

    def merge_segments(self, a, b):
        self._L.refsem_merge_segments(self._h, int(a), int(b))

    def remove_segment(self, object_id):
        self._L.refsem_remove_segment(self._h, int(object_id))
