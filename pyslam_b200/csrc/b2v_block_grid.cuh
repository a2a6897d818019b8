// b2v_block_grid.cuh — device helpers of the two sparse block grids (b2v_grid.cu, b2v_semantic.cu): point keys, the
// RGBD back-projection, colour conversions and the spatial filter of the read-outs.  Bit for bit the reference's
// arithmetic; each grid keeps its own voxel update, mean and keep rule.
#pragma once

#include "b2v_internal.h"

namespace b2v {

// voxel coordinate of a point in its own precision: get_voxel_key_inv<Tpos, Tpos> (voxel_hashing.h:69-75) with the
// float32 inverse voxel size widened for float64 points (voxel_block_grid.hpp:473)
__device__ __forceinline__ int point_voxel_coord(float x, float inv_vs) { return voxel_coord(x, inv_vs); }
__device__ __forceinline__ int point_voxel_coord(double x, float inv_vs) {
    return __double2int_rd(__dmul_rn(x, static_cast<double>(inv_vs)));
}

// colour of a point as a voxel accumulates it: float passthrough, uint8 * (1.0f / 255.0f) (voxel_data.h:79-97)
__device__ __forceinline__ float color_value(float c) { return c; }
__device__ __forceinline__ float color_value(uint8_t c) { return __fmul_rn(static_cast<float>(c), 1.0f / 255.0f); }
// colour of an RGBD pixel: image / 255.0 in float64, then float32 (depth.py:76)
__device__ __forceinline__ float rgbd_color(uint8_t c) {
    return __double2float_rn(__ddiv_rn(static_cast<double>(c), 255.0));
}

// world point of pixel i, false where the depth is out of range (depth.py:62-73, then Twc and float32)
__device__ __forceinline__ bool rgbd_point(const RgbdParams &P, const float *__restrict__ depth, int64_t i,
                                           float pt[3]) {
    const float d = depth[i];
    if (!(d > P.min_depth && d < P.max_depth)) return false;  // depth.py:62
    const int row = static_cast<int>(i / P.W), col = static_cast<int>(i % P.W);
    const double z = static_cast<double>(d);
    const double x = __dmul_rn(__dmul_rn(__dsub_rn(static_cast<double>(col), P.cx), z), P.fx_inv);  // depth.py:72
    const double y = __dmul_rn(__dmul_rn(__dsub_rn(static_cast<double>(row), P.cy), z), P.fy_inv);  // depth.py:73
#pragma unroll
    for (int a = 0; a < 3; ++a)  // in float64, then ascontiguousarray(float32)
        pt[a] = __double2float_rn(__dadd_rn(
            __dadd_rn(__dadd_rn(__dmul_rn(x, P.R[3 * a]), __dmul_rn(y, P.R[3 * a + 1])), __dmul_rn(z, P.R[3 * a + 2])),
            P.t[a]));
    return true;
}

// ---- spatial filter of box and frustum queries ---------------------------------------------------------------
struct ImagePoint {
    float u, v, depth;
};

// false when no voxel of the block (side 1 << L) can lie in the query's key range
template <int L> __device__ __forceinline__ bool block_in_range(const GridQuery &Q, const int4 key) {
    const int k[3] = {key.x, key.y, key.z};
#pragma unroll
    for (int a = 0; a < 3; ++a)
        if (k[a] < grid_block_coord<L>(Q.min_key[a]) || k[a] > grid_block_coord<L>(Q.max_key[a])) return false;
    return true;
}

// voxel t (lx + B ly + B^2 lz) of the block lies in the query's key range
template <int L> __device__ __forceinline__ bool voxel_in_range(const GridQuery &Q, const int4 key, int t) {
    constexpr int kS = GridBlock<L>::kSide;
    const int vk[3] = {key.x * kS + (t & (kS - 1)), key.y * kS + ((t >> L) & (kS - 1)), key.z * kS + (t >> (2 * L))};
#pragma unroll
    for (int a = 0; a < 3; ++a)
        if (vk[a] < Q.min_key[a] || vk[a] > Q.max_key[a]) return false;
    return true;
}

// CameraFrustrum::contains (camera_frustrum.cpp:174-196): world point -> (inside?, pixel, depth)
__device__ __forceinline__ bool frustum_contains(const GridQuery &Q, const double p[3], ImagePoint *ip) {
    double pc[3];
#pragma unroll
    for (int a = 0; a < 3; ++a)
        pc[a] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(Q.R[3 * a], p[0]), __dmul_rn(Q.R[3 * a + 1], p[1])),
                                    __dmul_rn(Q.R[3 * a + 2], p[2])),
                          Q.t[a]);
    const float depth = static_cast<float>(pc[2]);
    if (!(depth >= Q.depth_min && depth <= Q.depth_max)) return false;
    const float u = static_cast<float>(__dadd_rn(__dmul_rn(static_cast<double>(Q.fx), __ddiv_rn(pc[0], pc[2])),
                                                 static_cast<double>(Q.cx)));
    const float v = static_cast<float>(__dadd_rn(__dmul_rn(static_cast<double>(Q.fy), __ddiv_rn(pc[1], pc[2])),
                                                 static_cast<double>(Q.cy)));
    ip->u = u;
    ip->v = v;
    ip->depth = depth;
    return u >= 0.0f && u < static_cast<float>(Q.W) && v >= 0.0f && v < static_cast<float>(Q.H);
}

// the fine test of a box or frustum query on a voxel's mean position: BoundingBox3D::contains
// (bounding_boxes_3d.cpp:207-210) or CameraFrustrum::contains
__device__ __forceinline__ bool region_contains(const GridQuery &Q, const double p[3], ImagePoint *ip) {
    if (Q.mode == kQueryBox)
        return p[0] >= Q.bb[0] && p[0] <= Q.bb[3] && p[1] >= Q.bb[1] && p[1] <= Q.bb[4] && p[2] >= Q.bb[2] &&
               p[2] <= Q.bb[5];
    return frustum_contains(Q, p, ip);
}

}  // namespace b2v
