// b2v_grid.cu — point-average voxel block grid (pySLAM's own `volumetric.VoxelBlockGrid`), sm_90a.
//
// Replaces VoxelBlockGridT<VoxelData>::integrate_raw / get_voxels / remove_low_count_voxels
// (cpp/volumetric/voxel_block_grid.hpp:115-136, 524-614, 625-647, 717-819).  Per voxel the
// reference keeps {count, position_sum[3], color_sum[3]} (cpp/volumetric/voxel_data.h:118-133);
// here each block stores the same seven fields as 512-wide planes so a warp's accesses coalesce.
//   keys: voxel = floor(p * inv_vs) (voxel_hashing.h:69-75), block = floor_div(voxel, 8),
//         local index lx + 8 ly + 64 lz (voxel_block.h:67-70) -- bit exact.
//   sums: float atomics => same values as the reference up to summation order; sub-normal addends are kept
//         (sum_add), as the reference's float adds keep them.
#include "b2v_internal.h"
#include "b2v_scan.cuh"

namespace b2v {

constexpr int kGridPlanes = 7;  // count(int32), px, py, pz, cr, cg, cb
constexpr int kGridBlockWords = kGridPlanes * kVox;

// ---- pass 1: make sure every point's block exists -------------------------------------------
// voxel coordinate of a point in its own precision: get_voxel_key_inv<Tpos, Tpos> (voxel_hashing.h:69-75) with the
// float32 inverse voxel size widened for float64 points (voxel_block_grid.hpp:473)
__device__ __forceinline__ int point_voxel_coord(float x, float inv_vs) { return voxel_coord(x, inv_vs); }
__device__ __forceinline__ int point_voxel_coord(double x, float inv_vs) {
    return __double2int_rd(__dmul_rn(x, static_cast<double>(inv_vs)));
}

template <typename Tp>
__global__ void __launch_bounds__(256)
grid_insert_kernel(const Tp *__restrict__ pts, const int64_t n, const float inv_vs,
                   const HashTable T, const GridMeta G) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    bool have = i < n;
    int bx = 0, by = 0, bz = 0;
    if (have) {
        bx = block_coord(point_voxel_coord(pts[3 * i + 0], inv_vs));
        by = block_coord(point_voxel_coord(pts[3 * i + 1], inv_vs));
        bz = block_coord(point_voxel_coord(pts[3 * i + 2], inv_vs));
    }
    // one probe per distinct block per warp (neighbouring pixels share blocks)
    const unsigned long long pk = have ? (static_cast<unsigned long long>(slot_hash(bx, by, bz)) << 32 |
                                          static_cast<uint32_t>(bx * 73856093 ^ by * 19349663 ^ bz * 83492791))
                                       : ((1ull << 63) | static_cast<unsigned long long>(lane) << 40 | 0xFFFFFFull);
    const unsigned grp = __match_any_sync(0xffffffffu, pk);
    // hash equality is not key equality: only skip when the leader's key really matches
    const int leader = __ffs(grp) - 1;
    const int lbx = __shfl_sync(0xffffffffu, bx, leader), lby = __shfl_sync(0xffffffffu, by, leader),
              lbz = __shfl_sync(0xffffffffu, bz, leader);
    if (!have) return;
    if (leader != lane && lbx == bx && lby == by && lbz == bz) return;
    bool is_new;
    const uint32_t slot = table_insert(T, bx, by, bz, &is_new);
    if (slot == kEmpty) {
        atomicOr(G.counters + kCtrError, 2u);
        return;
    }
    if (is_new) {
        const uint32_t idx = atomicAdd(G.counters + kCtrPool, 1u);
        uint32_t *w = reinterpret_cast<uint32_t *>(T.entries + slot) + 3;
        if (idx < G.capacity) {
            G.block_keys[idx] = make_int4(bx, by, bz, 0);
            *w = idx;
        } else {
            *w = kNoBlock;
            atomicOr(G.counters + kCtrError, 1u);
        }
    }
}

// ---- pass 2: accumulate ----------------------------------------------------------------------
// running float sum += x as the reference's float add does it.  Float atomics (red.global.add.f32) flush sub-normal
// operands and results to zero.  An addend of magnitude >= 2^-100 can neither make a sub-normal sum nor lose anything
// but a sub-normal sum that rounding would drop anyway, so it takes the atomic; smaller non-zero addends go through a
// compare-and-swap of an IEEE add.  Adding +-0 leaves every sum unchanged (sums start at +0).
__device__ __forceinline__ void sum_add(float *p, float x) {
    if (fabsf(x) >= 0x1p-100f) {
        atomicAdd(p, x);
    } else if (x != 0.0f) {
        unsigned int *u = reinterpret_cast<unsigned int *>(p);
        unsigned int old = *u, assumed;
        do {
            assumed = old;
            old = atomicCAS(u, assumed, __float_as_uint(__fadd_rn(__uint_as_float(assumed), x)));
        } while (old != assumed);
    }
}

// colour of a point as the voxel accumulates it: float passthrough, uint8 * (1.0f / 255.0f) (voxel_data.h:79-97)
__device__ __forceinline__ float color_value(float c) { return c; }
__device__ __forceinline__ float color_value(uint8_t c) { return __fmul_rn(static_cast<float>(c), 1.0f / 255.0f); }

// Only the points whose block has a pool index in [lo, hi) are accumulated: the first pass of a call covers the blocks
// with storage, [0, pool_capacity); after a growth the same pass is replayed over the blocks that just got storage.
// A voxel's observations of one call all belong to one block, so each voxel is updated in exactly one of the passes.
template <typename Tp, typename Tc>
__global__ void __launch_bounds__(256)
grid_accumulate_kernel(const Tp *__restrict__ pts, const Tc *__restrict__ cols, const int64_t n,
                       const float inv_vs, const HashTable T, const GridMeta G, const uint32_t lo, const uint32_t hi) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Tp xp = pts[3 * i + 0], yp = pts[3 * i + 1], zp = pts[3 * i + 2];
    const int vx = point_voxel_coord(xp, inv_vs), vy = point_voxel_coord(yp, inv_vs), vz = point_voxel_coord(zp, inv_vs);
    // position_sum += static_cast<float>(x) (voxel_data.h:53-57)
    const float x = static_cast<float>(xp), y = static_cast<float>(yp), z = static_cast<float>(zp);
    const uint32_t slot = table_find(T, block_coord(vx), block_coord(vy), block_coord(vz));
    if (slot == kEmpty) return;
    const uint32_t idx = T.entries[slot].w;
    if (idx < lo || idx >= hi) return;   // kNoBlock is past every window
    const int l = local_coord(vx) + (local_coord(vy) << 3) + (local_coord(vz) << 6);
    uint32_t *blk = G.pool + static_cast<size_t>(idx) * kGridBlockWords;
    float *fb = reinterpret_cast<float *>(blk);
    sum_add(fb + 1 * kVox + l, x);
    sum_add(fb + 2 * kVox + l, y);
    sum_add(fb + 3 * kVox + l, z);
    if (cols != nullptr) {
        sum_add(fb + 4 * kVox + l, color_value(cols[3 * i + 0]));
        sum_add(fb + 5 * kVox + l, color_value(cols[3 * i + 1]));
        sum_add(fb + 6 * kVox + l, color_value(cols[3 * i + 2]));
    }
    atomicAdd(reinterpret_cast<int *>(blk) + l, 1);
}

// ---- fused RGBD front-end: back-project + insert / accumulate ---------------------------------
__device__ __forceinline__ bool rgbd_point(const RgbdParams &P, const float *__restrict__ depth, int64_t i,
                                           float pt[3]) {
    const float d = depth[i];
    if (!(d > P.min_depth && d < P.max_depth)) return false;  // depth.py:62
    const int row = static_cast<int>(i / P.W), col = static_cast<int>(i % P.W);
    const double z = static_cast<double>(d);
    const double x = __dmul_rn(__dmul_rn(__dsub_rn(static_cast<double>(col), P.cx), z), P.fx_inv);  // depth.py:72
    const double y = __dmul_rn(__dmul_rn(__dsub_rn(static_cast<double>(row), P.cy), z), P.fy_inv);  // depth.py:73
#pragma unroll
    for (int a = 0; a < 3; ++a)  // voxel_grid.py:262-265, then ascontiguousarray(float32) :281
        pt[a] = __double2float_rn(__dadd_rn(
            __dadd_rn(__dadd_rn(__dmul_rn(x, P.R[3 * a]), __dmul_rn(y, P.R[3 * a + 1])), __dmul_rn(z, P.R[3 * a + 2])),
            P.t[a]));
    return true;
}

__global__ void __launch_bounds__(256)
grid_rgbd_insert_kernel(const RgbdParams P, const float *__restrict__ depth, const float inv_vs,
                        const HashTable T, const GridMeta G) {
    const int64_t n = static_cast<int64_t>(P.H) * P.W;
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    float pt[3];
    const bool have = i < n && rgbd_point(P, depth, i, pt);
    int bx = 0, by = 0, bz = 0;
    if (have) {
        bx = block_coord(voxel_coord(pt[0], inv_vs));
        by = block_coord(voxel_coord(pt[1], inv_vs));
        bz = block_coord(voxel_coord(pt[2], inv_vs));
    }
    const unsigned long long pk = have ? (static_cast<unsigned long long>(slot_hash(bx, by, bz)) << 32 |
                                          static_cast<uint32_t>(bx * 73856093 ^ by * 19349663 ^ bz * 83492791))
                                       : ((1ull << 63) | static_cast<unsigned long long>(lane) << 40 | 0xFFFFFFull);
    const unsigned grp = __match_any_sync(0xffffffffu, pk);
    const int leader = __ffs(grp) - 1;
    const int lbx = __shfl_sync(0xffffffffu, bx, leader), lby = __shfl_sync(0xffffffffu, by, leader),
              lbz = __shfl_sync(0xffffffffu, bz, leader);
    if (!have) return;
    if (leader != lane && lbx == bx && lby == by && lbz == bz) return;
    bool is_new;
    const uint32_t slot = table_insert(T, bx, by, bz, &is_new);
    if (slot == kEmpty) {
        atomicOr(G.counters + kCtrError, 2u);
        return;
    }
    if (is_new) {
        const uint32_t idx = atomicAdd(G.counters + kCtrPool, 1u);
        uint32_t *w = reinterpret_cast<uint32_t *>(T.entries + slot) + 3;
        if (idx < G.capacity) {
            G.block_keys[idx] = make_int4(bx, by, bz, 0);
            *w = idx;
        } else {
            *w = kNoBlock;
            atomicOr(G.counters + kCtrError, 1u);
        }
    }
}

__global__ void __launch_bounds__(256)
grid_rgbd_accumulate_kernel(const RgbdParams P, const float *__restrict__ depth, const uint8_t *__restrict__ rgb,
                            const float inv_vs, const HashTable T, const GridMeta G, const uint32_t lo,
                            const uint32_t hi) {
    const int64_t n = static_cast<int64_t>(P.H) * P.W;
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    float pt[3];
    if (i >= n || !rgbd_point(P, depth, i, pt)) return;
    const int vx = voxel_coord(pt[0], inv_vs), vy = voxel_coord(pt[1], inv_vs), vz = voxel_coord(pt[2], inv_vs);
    const uint32_t slot = table_find(T, block_coord(vx), block_coord(vy), block_coord(vz));
    if (slot == kEmpty) return;
    const uint32_t idx = T.entries[slot].w;
    if (idx < lo || idx >= hi) return;   // the window of grid_accumulate_kernel
    const int l = local_coord(vx) + (local_coord(vy) << 3) + (local_coord(vz) << 6);
    uint32_t *blk = G.pool + static_cast<size_t>(idx) * kGridBlockWords;
    float *fb = reinterpret_cast<float *>(blk);
    sum_add(fb + 1 * kVox + l, pt[0]);
    sum_add(fb + 2 * kVox + l, pt[1]);
    sum_add(fb + 3 * kVox + l, pt[2]);
#pragma unroll
    for (int c = 0; c < 3; ++c)  // image[valid] / 255.0 in float64, then float32 (depth.py:76, voxel_grid.py:271-273)
        sum_add(fb + (4 + c) * kVox + l, __double2float_rn(__ddiv_rn(static_cast<double>(rgb[3 * i + c]), 255.0)));
    atomicAdd(reinterpret_cast<int *>(blk) + l, 1);
}

cudaError_t launch_grid_integrate_rgbd(const RgbdParams &p, const float *depth, const uint8_t *rgb,
                                       float inv_vs, const HashTable &table, const GridMeta &meta,
                                       cudaStream_t stream) {
    const int64_t n = static_cast<int64_t>(p.H) * p.W;
    if (n <= 0) return cudaSuccess;
    const unsigned grid = static_cast<unsigned>((n + 255) / 256);
    grid_rgbd_insert_kernel<<<grid, 256, 0, stream>>>(p, depth, inv_vs, table, meta);
    grid_rgbd_accumulate_kernel<<<grid, 256, 0, stream>>>(p, depth, rgb, inv_vs, table, meta, 0u, meta.pool_capacity);
    return cudaGetLastError();
}

cudaError_t launch_grid_rgbd_accumulate(const RgbdParams &p, const float *depth, const uint8_t *rgb, float inv_vs,
                                        const HashTable &table, const GridMeta &meta, uint32_t lo, uint32_t hi,
                                        cudaStream_t stream) {
    const int64_t n = static_cast<int64_t>(p.H) * p.W;
    if (n <= 0) return cudaSuccess;
    grid_rgbd_accumulate_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(p, depth, rgb, inv_vs,
                                                                                            table, meta, lo, hi);
    return cudaGetLastError();
}

// ---- get_voxels: count -> scan -> emit -------------------------------------------------------
__global__ void __launch_bounds__(kVox)
grid_count_kernel(const GridMeta G, const int min_count, uint32_t *__restrict__ sums) {
    __shared__ uint32_t s_warp[16];
    const uint32_t b = blockIdx.x;
    const int t = threadIdx.x;
    const int c = reinterpret_cast<const int *>(G.pool + static_cast<size_t>(b) * kGridBlockWords)[t];
    uint32_t x = __reduce_add_sync(0xffffffffu, (c >= min_count) ? 1u : 0u);
    if ((t & 31) == 0) s_warp[t >> 5] = x;
    __syncthreads();
    if (t == 0) {
        uint32_t s = 0;
        for (int k = 0; k < 16; ++k) s += s_warp[k];
        sums[b] = s;
    }
}

__global__ void __launch_bounds__(kVox)
grid_emit_kernel(const GridMeta G, const int min_count, const uint32_t *__restrict__ offs,
                 float *__restrict__ out_pts, float *__restrict__ out_cols) {
    __shared__ uint32_t s_warp[16];
    const uint32_t b = blockIdx.x;
    const int t = threadIdx.x;
    const uint32_t *blk = G.pool + static_cast<size_t>(b) * kGridBlockWords;
    const float *fb = reinterpret_cast<const float *>(blk);
    const int c = reinterpret_cast<const int *>(blk)[t];
    const bool keep = c >= min_count;
    const uint32_t pos = offs[b] + block_excl_scan_512(keep ? 1u : 0u, s_warp);
    if (!keep) return;
    const float fc = static_cast<float>(c);  // voxel_data.h:64-67,104-107: sum / (T)count
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        out_pts[3 * static_cast<size_t>(pos) + k] = __fdiv_rn(fb[(1 + k) * kVox + t], fc);
        out_cols[3 * static_cast<size_t>(pos) + k] = __fdiv_rn(fb[(4 + k) * kVox + t], fc);
    }
}

__global__ void __launch_bounds__(kVox)
grid_remove_low_count_kernel(const GridMeta G, const int min_count) {
    uint32_t *blk = G.pool + static_cast<size_t>(blockIdx.x) * kGridBlockWords;
    const int t = threadIdx.x;
    if (reinterpret_cast<const int *>(blk)[t] < min_count) {  // voxel_block_grid.hpp:641-643 -> reset()
#pragma unroll
        for (int k = 0; k < kGridPlanes; ++k) blk[k * kVox + t] = 0u;
    }
}

// ---- spatial queries and carving ---------------------------------------------------------------
struct ImagePoint {
    float u, v, depth;
};

// CameraFrustrum::contains (camera_frustrum.cpp:174-196): world point -> (inside?, pixel, depth)
__device__ __forceinline__ bool frustum_contains(const GridQuery &Q, const float p[3], ImagePoint *ip) {
    const double x = p[0], y = p[1], z = p[2];
    double pc[3];
#pragma unroll
    for (int a = 0; a < 3; ++a)
        pc[a] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(Q.R[3 * a], x), __dmul_rn(Q.R[3 * a + 1], y)),
                                    __dmul_rn(Q.R[3 * a + 2], z)),
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

// the reference's per-voxel filter chain; returns true and the mean position if the voxel qualifies
__device__ __forceinline__ bool query_voxel(const GridQuery &Q, const uint32_t *blk, const int4 key, int t,
                                            float pos[3], ImagePoint *ip) {
    const int c = reinterpret_cast<const int *>(blk)[t];
    if (c < Q.min_count) return false;
    const int vk[3] = {key.x * kB + (t & 7), key.y * kB + ((t >> 3) & 7), key.z * kB + (t >> 6)};
#pragma unroll
    for (int a = 0; a < 3; ++a)
        if (vk[a] < Q.min_key[a] || vk[a] > Q.max_key[a]) return false;
    const float *fb = reinterpret_cast<const float *>(blk);
    const float fc = static_cast<float>(c);
#pragma unroll
    for (int a = 0; a < 3; ++a) pos[a] = __fdiv_rn(fb[(1 + a) * kVox + t], fc);  // voxel_data.h:58-69
    if (Q.mode == 0) {
        const double x = pos[0], y = pos[1], z = pos[2];  // BoundingBox3D::contains (bounding_boxes_3d.cpp:207-210)
        return x >= Q.bb[0] && x <= Q.bb[3] && y >= Q.bb[1] && y <= Q.bb[4] && z >= Q.bb[2] && z <= Q.bb[5];
    }
    return frustum_contains(Q, pos, ip);
}

__device__ __forceinline__ bool block_in_range(const GridQuery &Q, const int4 key) {
    const int k[3] = {key.x, key.y, key.z};
#pragma unroll
    for (int a = 0; a < 3; ++a)
        if (k[a] < block_coord(Q.min_key[a]) || k[a] > block_coord(Q.max_key[a])) return false;
    return true;
}

__global__ void __launch_bounds__(kVox)
grid_query_count_kernel(const GridMeta G, const GridQuery Q, uint32_t *__restrict__ sums) {
    __shared__ uint32_t s_warp[16];
    const uint32_t b = blockIdx.x;
    const int t = threadIdx.x;
    const int4 key = G.block_keys[b];
    float pos[3];
    ImagePoint ip;
    const bool keep = block_in_range(Q, key) &&
                      query_voxel(Q, G.pool + static_cast<size_t>(b) * kGridBlockWords, key, t, pos, &ip);
    const uint32_t x = __reduce_add_sync(0xffffffffu, keep ? 1u : 0u);
    if ((t & 31) == 0) s_warp[t >> 5] = x;
    __syncthreads();
    if (t == 0) {
        uint32_t s = 0;
        for (int k = 0; k < 16; ++k) s += s_warp[k];
        sums[b] = s;
    }
}

__global__ void __launch_bounds__(kVox)
grid_query_emit_kernel(const GridMeta G, const GridQuery Q, const uint32_t *__restrict__ offs,
                       float *__restrict__ out_pts, float *__restrict__ out_cols) {
    __shared__ uint32_t s_warp[16];
    const uint32_t b = blockIdx.x;
    const int t = threadIdx.x;
    const int4 key = G.block_keys[b];
    const uint32_t *blk = G.pool + static_cast<size_t>(b) * kGridBlockWords;
    float pos[3];
    ImagePoint ip;
    const bool keep = block_in_range(Q, key) && query_voxel(Q, blk, key, t, pos, &ip);
    const uint32_t o = offs[b] + block_excl_scan_512(keep ? 1u : 0u, s_warp);
    if (!keep) return;
    const float *fb = reinterpret_cast<const float *>(blk);
    const float fc = static_cast<float>(reinterpret_cast<const int *>(blk)[t]);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        out_pts[3 * static_cast<size_t>(o) + k] = pos[k];
        out_cols[3 * static_cast<size_t>(o) + k] = __fdiv_rn(fb[(4 + k) * kVox + t], fc);
    }
}

// carve (voxel_grid_carving.h:47-80): reset voxels that lie in front of the observed depth by more
// than the threshold.  The depth image is indexed with TRUNCATED pixel coordinates, like at<float>(v, u).
__global__ void __launch_bounds__(kVox)
grid_carve_kernel(const GridMeta G, const GridQuery Q, const float *__restrict__ depth, const float thr) {
    const uint32_t b = blockIdx.x;
    const int t = threadIdx.x;
    const int4 key = G.block_keys[b];
    if (!block_in_range(Q, key)) return;
    uint32_t *blk = G.pool + static_cast<size_t>(b) * kGridBlockWords;
    float pos[3];
    ImagePoint ip;
    if (!query_voxel(Q, blk, key, t, pos, &ip)) return;
    const float image_depth = depth[static_cast<size_t>(static_cast<int>(ip.v)) * Q.W + static_cast<int>(ip.u)];
    if (image_depth <= 0.0f || !isfinite(image_depth)) return;
    if (ip.depth < image_depth - thr) {
#pragma unroll
        for (int k = 0; k < kGridPlanes; ++k) blk[k * kVox + t] = 0u;
    }
}

cudaError_t launch_grid_query_count(const GridMeta &meta, uint32_t n_blocks, const GridQuery &q,
                                    uint32_t *sums, uint32_t *offs, uint32_t *total, cudaStream_t stream) {
    if (n_blocks == 0) return cudaMemsetAsync(total, 0, sizeof(uint32_t), stream);
    grid_query_count_kernel<<<n_blocks, kVox, 0, stream>>>(meta, q, sums);
    exclusive_scan_kernel<<<1, 1024, 0, stream>>>(sums, offs, total, n_blocks);
    return cudaGetLastError();
}

cudaError_t launch_grid_query_emit(const GridMeta &meta, uint32_t n_blocks, const GridQuery &q,
                                   const uint32_t *offs, float *out_pts, float *out_cols, cudaStream_t stream) {
    if (n_blocks == 0) return cudaSuccess;
    grid_query_emit_kernel<<<n_blocks, kVox, 0, stream>>>(meta, q, offs, out_pts, out_cols);
    return cudaGetLastError();
}

cudaError_t launch_grid_carve(const GridMeta &meta, uint32_t n_blocks, const GridQuery &q, const float *depth,
                              float depth_threshold, cudaStream_t stream) {
    if (n_blocks == 0) return cudaSuccess;
    grid_carve_kernel<<<n_blocks, kVox, 0, stream>>>(meta, q, depth, depth_threshold);
    return cudaGetLastError();
}

// ---- launchers -------------------------------------------------------------------------------
template <typename Tp>
static void launch_grid_accumulate_t(const Tp *p, const void *cols, bool cols_u8, int64_t n, float inv_vs,
                                     const HashTable &table, const GridMeta &meta, uint32_t lo, uint32_t hi,
                                     cudaStream_t stream) {
    const unsigned grid = static_cast<unsigned>((n + 255) / 256);
    if (cols_u8)
        grid_accumulate_kernel<Tp, uint8_t><<<grid, 256, 0, stream>>>(p, static_cast<const uint8_t *>(cols), n, inv_vs,
                                                                      table, meta, lo, hi);
    else
        grid_accumulate_kernel<Tp, float><<<grid, 256, 0, stream>>>(p, static_cast<const float *>(cols), n, inv_vs,
                                                                    table, meta, lo, hi);
}

cudaError_t launch_grid_accumulate(const void *pts, bool pts_f64, const void *cols, bool cols_u8, int64_t n,
                                   float inv_vs, const HashTable &table, const GridMeta &meta, uint32_t lo, uint32_t hi,
                                   cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    if (pts_f64)
        launch_grid_accumulate_t(static_cast<const double *>(pts), cols, cols_u8, n, inv_vs, table, meta, lo, hi, stream);
    else
        launch_grid_accumulate_t(static_cast<const float *>(pts), cols, cols_u8, n, inv_vs, table, meta, lo, hi, stream);
    return cudaGetLastError();
}

cudaError_t launch_grid_integrate(const void *pts, bool pts_f64, const void *cols, bool cols_u8, int64_t n, float inv_vs,
                                  const HashTable &table, const GridMeta &meta, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    const unsigned grid = static_cast<unsigned>((n + 255) / 256);
    if (pts_f64)
        grid_insert_kernel<double><<<grid, 256, 0, stream>>>(static_cast<const double *>(pts), n, inv_vs, table, meta);
    else
        grid_insert_kernel<float><<<grid, 256, 0, stream>>>(static_cast<const float *>(pts), n, inv_vs, table, meta);
    return launch_grid_accumulate(pts, pts_f64, cols, cols_u8, n, inv_vs, table, meta, 0u, meta.pool_capacity, stream);
}

cudaError_t launch_grid_count(const GridMeta &meta, uint32_t n_blocks, int min_count, uint32_t *sums,
                              uint32_t *offs, uint32_t *total, cudaStream_t stream) {
    if (n_blocks == 0) return cudaMemsetAsync(total, 0, sizeof(uint32_t), stream);
    grid_count_kernel<<<n_blocks, kVox, 0, stream>>>(meta, min_count, sums);
    exclusive_scan_kernel<<<1, 1024, 0, stream>>>(sums, offs, total, n_blocks);
    return cudaGetLastError();
}

cudaError_t launch_grid_emit(const GridMeta &meta, uint32_t n_blocks, int min_count,
                             const uint32_t *offs, float *out_pts, float *out_cols,
                             cudaStream_t stream) {
    if (n_blocks == 0) return cudaSuccess;
    grid_emit_kernel<<<n_blocks, kVox, 0, stream>>>(meta, min_count, offs, out_pts, out_cols);
    return cudaGetLastError();
}

cudaError_t launch_grid_remove_low_count(const GridMeta &meta, uint32_t n_blocks, int min_count,
                                         cudaStream_t stream) {
    if (n_blocks == 0) return cudaSuccess;
    grid_remove_low_count_kernel<<<n_blocks, kVox, 0, stream>>>(meta, min_count);
    return cudaGetLastError();
}

}  // namespace b2v
