// b2v_grid.cu — point-average voxel block grid (pySLAM's own `volumetric.VoxelBlockGrid`), sm_90a, and the block
// grid core it shares with the semantic grids (b2v_semantic.cu): the warp-deduplicated block insert and the host
// half (BlockGridCore: table, block index, counters, growth, read-out scans, query builders).
//
// Replaces VoxelBlockGridT<VoxelData>::integrate_raw / get_voxels / remove_low_count_voxels
// (cpp/volumetric/voxel_block_grid.hpp:115-136, 524-614, 625-647, 717-819).  Per voxel the
// reference keeps {count, position_sum[3], color_sum[3]} (cpp/volumetric/voxel_data.h:118-133);
// here each block stores the same seven fields as B^3-wide planes so a warp's accesses coalesce.
//   keys: voxel = floor(p * inv_vs) (voxel_hashing.h:69-75), block = floor_div(voxel, B),
//         local index lx + B ly + B^2 lz (voxel_block.h:67-70) -- bit exact, for B = 1 << L (1, 2, 8, 16) a template
//         parameter of every kernel that keys or walks voxels (with_grid_block picks the instantiation).
//   sums: float atomics => same values as the reference up to summation order; sub-normal addends are kept
//         (sum_add), as the reference's float adds keep them.  With input-order sums (b2v_grid_set_input_order_sums)
//         each voxel instead adds its points in input order with IEEE float32 adds (voxel sort -> grid_runs_kernel),
//         the sequential reference's sums bit for bit.
#include <cub/device/device_radix_sort.cuh>

#include <cmath>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "b2v_block_grid.cuh"
#include "b2v_scan.cuh"

namespace b2v {

constexpr int kGridPlanes = 7;  // count(int32), px, py, pz, cr, cg, cb
template <int L> constexpr int kGridBlockWords = kGridPlanes * GridBlock<L>::kVox;

struct GridMeta {
    uint32_t *pool;     // [pool_capacity][7][B^3] planes: count(int32), px, py, pz, cr, cg, cb (float32)
    BlockIndex index;
};

// ---- block insert (both grids) ---------------------------------------------------------------
// Make sure block (bx, by, bz) of every thread with `have` exists: one probe per distinct block per warp
// (neighbouring points share blocks).  A new block gets the next pool index, or kNoBlock past index.capacity.
// A sharded grid inserts only the blocks its rank owns; every pass that writes voxels finds its block with
// table_find and skips the points whose block is absent, so this one test partitions both grids.
__device__ __forceinline__ void block_insert(bool have, int bx, int by, int bz, const HashTable &T,
                                             const BlockIndex &B) {
    const int lane = threadIdx.x & 31;
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
    // after the warp vote, which needs every lane: one owner test per distinct block
    if (B.shard_count > 1u && block_owner(bx, by, bz, B.shard_count) != B.shard_rank) return;
    bool is_new;
    const uint32_t slot = table_insert(T, bx, by, bz, &is_new);
    if (slot == kEmpty) {
        atomicOr(B.counters + kBgError, 2u);
        return;
    }
    if (is_new) {
        const uint32_t idx = atomicAdd(B.counters + kBgPool, 1u);
        uint32_t *w = reinterpret_cast<uint32_t *>(T.entries + slot) + 3;
        if (idx < B.capacity) {
            B.block_keys[idx] = make_int4(bx, by, bz, 0);
            *w = idx;
        } else {
            *w = kNoBlock;
            atomicOr(B.counters + kBgError, 1u);
        }
    }
}

template <typename Tp, int L>
__global__ void __launch_bounds__(256)
point_insert_kernel(const Tp *__restrict__ pts, const uint8_t *__restrict__ valid, const int64_t n,
                    const float inv_vs, const HashTable T, const BlockIndex B) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    const bool have = i < n && (valid == nullptr || valid[i]);
    int bx = 0, by = 0, bz = 0;
    if (have) {
        bx = grid_block_coord<L>(point_voxel_coord(pts[3 * i + 0], inv_vs));
        by = grid_block_coord<L>(point_voxel_coord(pts[3 * i + 1], inv_vs));
        bz = grid_block_coord<L>(point_voxel_coord(pts[3 * i + 2], inv_vs));
    }
    block_insert(have, bx, by, bz, T, B);
}

// block upload: one thread per uploaded key, through the same insert (and owner test) as the points' blocks
__global__ void __launch_bounds__(256)
block_import_kernel(const int4 *__restrict__ keys, const uint32_t n, const HashTable T, const BlockIndex B) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool have = i < n;
    const int4 k = have ? keys[i] : make_int4(0, 0, 0, 0);
    block_insert(have, k.x, k.y, k.z, T, B);
}

cudaError_t launch_point_insert(const void *pts, bool pts_f64, const uint8_t *valid, int64_t n, float inv_vs,
                                int log2_block, const HashTable &table, const BlockIndex &index, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    const unsigned grid = static_cast<unsigned>((n + 255) / 256);
    with_grid_block(log2_block, [&](auto l) {
        constexpr int L = decltype(l)::value;
        if (pts_f64)
            point_insert_kernel<double, L><<<grid, 256, 0, stream>>>(static_cast<const double *>(pts), valid, n,
                                                                     inv_vs, table, index);
        else
            point_insert_kernel<float, L><<<grid, 256, 0, stream>>>(static_cast<const float *>(pts), valid, n,
                                                                    inv_vs, table, index);
    });
    return cudaGetLastError();
}

// ---- accumulate ------------------------------------------------------------------------------
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

// Only the points whose block has a pool index in [lo, hi) are accumulated: the first pass of a call covers the blocks
// with storage, [0, pool_capacity); after a growth the same pass is replayed over the blocks that just got storage.
// A voxel's observations of one call all belong to one block, so each voxel is updated in exactly one of the passes.
template <typename Tp, typename Tc, int L>
__global__ void __launch_bounds__(256)
grid_accumulate_kernel(const Tp *__restrict__ pts, const Tc *__restrict__ cols, const int64_t n,
                       const float inv_vs, const HashTable T, const GridMeta G, const uint32_t lo, const uint32_t hi) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Tp xp = pts[3 * i + 0], yp = pts[3 * i + 1], zp = pts[3 * i + 2];
    const int vx = point_voxel_coord(xp, inv_vs), vy = point_voxel_coord(yp, inv_vs), vz = point_voxel_coord(zp, inv_vs);
    // position_sum += static_cast<float>(x) (voxel_data.h:53-57)
    const float x = static_cast<float>(xp), y = static_cast<float>(yp), z = static_cast<float>(zp);
    const uint32_t slot = table_find(T, grid_block_coord<L>(vx), grid_block_coord<L>(vy), grid_block_coord<L>(vz));
    if (slot == kEmpty) return;
    const uint32_t idx = T.entries[slot].w;
    if (idx < lo || idx >= hi) return;   // kNoBlock is past every window
    constexpr int kV = GridBlock<L>::kVox;
    const int l = grid_local_index<L>(vx, vy, vz);
    uint32_t *blk = G.pool + static_cast<size_t>(idx) * kGridBlockWords<L>;
    float *fb = reinterpret_cast<float *>(blk);
    sum_add(fb + 1 * kV + l, x);
    sum_add(fb + 2 * kV + l, y);
    sum_add(fb + 3 * kV + l, z);
    if (cols != nullptr) {
        sum_add(fb + 4 * kV + l, color_value(cols[3 * i + 0]));
        sum_add(fb + 5 * kV + l, color_value(cols[3 * i + 1]));
        sum_add(fb + 6 * kV + l, color_value(cols[3 * i + 2]));
    }
    atomicAdd(reinterpret_cast<int *>(blk) + l, 1);
}

// ---- fused RGBD front-end: back-project + insert / accumulate ---------------------------------
template <int L>
__global__ void __launch_bounds__(256)
grid_rgbd_insert_kernel(const RgbdParams P, const float *__restrict__ depth, const float inv_vs,
                        const HashTable T, const BlockIndex B) {
    const int64_t n = static_cast<int64_t>(P.H) * P.W;
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    float pt[3];
    const bool have = i < n && rgbd_point(P, depth, i, pt);
    int bx = 0, by = 0, bz = 0;
    if (have) {
        bx = grid_block_coord<L>(voxel_coord(pt[0], inv_vs));
        by = grid_block_coord<L>(voxel_coord(pt[1], inv_vs));
        bz = grid_block_coord<L>(voxel_coord(pt[2], inv_vs));
    }
    block_insert(have, bx, by, bz, T, B);
}

template <int L>
__global__ void __launch_bounds__(256)
grid_rgbd_accumulate_kernel(const RgbdParams P, const float *__restrict__ depth, const uint8_t *__restrict__ rgb,
                            const float inv_vs, const HashTable T, const GridMeta G, const uint32_t lo,
                            const uint32_t hi) {
    const int64_t n = static_cast<int64_t>(P.H) * P.W;
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    float pt[3];
    if (i >= n || !rgbd_point(P, depth, i, pt)) return;
    const int vx = voxel_coord(pt[0], inv_vs), vy = voxel_coord(pt[1], inv_vs), vz = voxel_coord(pt[2], inv_vs);
    const uint32_t slot = table_find(T, grid_block_coord<L>(vx), grid_block_coord<L>(vy), grid_block_coord<L>(vz));
    if (slot == kEmpty) return;
    const uint32_t idx = T.entries[slot].w;
    if (idx < lo || idx >= hi) return;   // the window of grid_accumulate_kernel
    constexpr int kV = GridBlock<L>::kVox;
    const int l = grid_local_index<L>(vx, vy, vz);
    uint32_t *blk = G.pool + static_cast<size_t>(idx) * kGridBlockWords<L>;
    float *fb = reinterpret_cast<float *>(blk);
    sum_add(fb + 1 * kV + l, pt[0]);
    sum_add(fb + 2 * kV + l, pt[1]);
    sum_add(fb + 3 * kV + l, pt[2]);
#pragma unroll
    for (int c = 0; c < 3; ++c)  // voxel_grid.py:271-273
        sum_add(fb + (4 + c) * kV + l, rgbd_color(rgb[3 * i + c]));
    atomicAdd(reinterpret_cast<int *>(blk) + l, 1);
}

// ---- voxel-order sort (both grids' input-order updates: BlockGridCore::sort_voxels) -------------------------
// sort key of point i: pool index * B^3 + local index when its block has a pool index in [lo, hi), else kBadVid (also
// for points masked out by `valid`); value: i.  A pass over [lo, hi) updates each voxel of those blocks once.
template <typename T, int L>
__global__ void __launch_bounds__(256)
voxel_keys_kernel(const T *__restrict__ pts, const uint8_t *__restrict__ valid, const int64_t n, const float inv_vs,
                  const HashTable H, const uint32_t lo, const uint32_t hi, uint32_t *__restrict__ vid,
                  uint32_t *__restrict__ order) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int vx = point_voxel_coord(pts[3 * i + 0], inv_vs), vy = point_voxel_coord(pts[3 * i + 1], inv_vs),
              vz = point_voxel_coord(pts[3 * i + 2], inv_vs);
    uint32_t key = kBadVid;
    const uint32_t slot = (valid == nullptr || valid[i])
                              ? table_find(H, grid_block_coord<L>(vx), grid_block_coord<L>(vy), grid_block_coord<L>(vz))
                              : kEmpty;
    if (slot != kEmpty) {
        const uint32_t idx = H.entries[slot].w;
        if (idx >= lo && idx < hi)   // kNoBlock is past every window
            key = idx * GridBlock<L>::kVox + static_cast<uint32_t>(grid_local_index<L>(vx, vy, vz));
    }
    vid[i] = key;
    order[i] = static_cast<uint32_t>(i);
}

// ---- input-order sums (b2v_grid_set_input_order_sums) ------------------------------------------------------
// After the voxel-order sort each voxel's points of the pass are one run of equal keys, in input order (the sort is
// stable).  The head of a run walks it from the voxel's stored values with the reference's per-point update
// (voxel_data.h:53-57, 79-90): count + 1, position_sum += float32(x), color_sum += colour, each an IEEE float32 add
// (--ftz=false keeps sub-normal addends), and writes each plane once.  The three sums of a group are independent
// chains.  kBadVid ends the keys of the pass.  No colours (cols == nullptr): the colour sums are left as they are.
template <typename Tp, typename Tc, int L>
__global__ void __launch_bounds__(256)
grid_runs_kernel(const uint32_t *__restrict__ vid, const uint32_t *__restrict__ order, const int64_t n,
                 const Tp *__restrict__ pts, const Tc *__restrict__ cols, const GridMeta G) {
    const int64_t j0 = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (j0 >= n) return;
    const uint32_t v = vid[j0];
    if (v == kBadVid || (j0 > 0 && vid[j0 - 1] == v)) return;  // not the head of a run
    constexpr int kV = GridBlock<L>::kVox;
    const int l = static_cast<int>(v & (kV - 1));
    uint32_t *blk = G.pool + static_cast<size_t>(v >> (3 * L)) * kGridBlockWords<L>;
    float *fb = reinterpret_cast<float *>(blk);
    int count = reinterpret_cast<const int *>(blk)[l];
    float px = fb[1 * kV + l], py = fb[2 * kV + l], pz = fb[3 * kV + l];
    float cr = 0.0f, cg = 0.0f, cb = 0.0f;
    if (cols != nullptr) cr = fb[4 * kV + l], cg = fb[5 * kV + l], cb = fb[6 * kV + l];
    for (int64_t j = j0; j < n && vid[j] == v; ++j) {
        const size_t i = order[j];
        ++count;
        px = __fadd_rn(px, static_cast<float>(pts[3 * i + 0]));
        py = __fadd_rn(py, static_cast<float>(pts[3 * i + 1]));
        pz = __fadd_rn(pz, static_cast<float>(pts[3 * i + 2]));
        if (cols != nullptr) {
            cr = __fadd_rn(cr, color_value(cols[3 * i + 0]));
            cg = __fadd_rn(cg, color_value(cols[3 * i + 1]));
            cb = __fadd_rn(cb, color_value(cols[3 * i + 2]));
        }
    }
    reinterpret_cast<int *>(blk)[l] = count;
    fb[1 * kV + l] = px;
    fb[2 * kV + l] = py;
    fb[3 * kV + l] = pz;
    if (cols != nullptr) {
        fb[4 * kV + l] = cr;
        fb[5 * kV + l] = cg;
        fb[6 * kV + l] = cb;
    }
}

// integrate_rgbd with input-order sums: one thread per pixel writes the point record the front-end makes of it, from
// the rgbd_point / rgbd_color of the atomic path, and a valid mask.  Invalid pixels are masked, not compacted, so each
// voxel's run follows the row-major pixel order, the reference's point order.
__global__ void __launch_bounds__(256)
grid_rgbd_points_kernel(const RgbdParams P, const float *__restrict__ depth, const uint8_t *__restrict__ rgb,
                        float *__restrict__ pts, float *__restrict__ cols, uint8_t *__restrict__ valid) {
    const int64_t n = static_cast<int64_t>(P.H) * P.W;
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float pt[3];
    const bool ok = rgbd_point(P, depth, i, pt);
    valid[i] = ok ? 1 : 0;
    if (!ok) return;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        pts[3 * i + a] = pt[a];
        cols[3 * i + a] = rgbd_color(rgb[3 * i + a]);
    }
}

// Per-voxel passes: one 512-thread CTA per 512 pool voxels (cta_voxel); nb, the blocks in use, bounds the last CTA
// when B < 8 (at B >= 8 the CTAs cover whole blocks and it is not read).
template <int L>
__global__ void __launch_bounds__(kVox)
grid_remove_low_count_kernel(const GridMeta G, const int min_count, const uint32_t nb) {
    uint32_t b;
    int t;
    cta_voxel<L>(&b, &t);
    if (3 * L < 9 && b >= nb) return;
    uint32_t *blk = G.pool + static_cast<size_t>(b) * kGridBlockWords<L>;
    if (reinterpret_cast<const int *>(blk)[t] < min_count) {  // voxel_block_grid.hpp:641-643 -> reset()
#pragma unroll
        for (int k = 0; k < kGridPlanes; ++k) blk[k * GridBlock<L>::kVox + t] = 0u;
    }
}

// ---- read-outs (count -> scan -> emit) and carving ---------------------------------------------
// mean position of a voxel with count c: sum / (float)count (voxel_data.h:58-69)
template <int L> __device__ __forceinline__ void grid_mean(const uint32_t *blk, int t, int c, float pos[3]) {
    const float *fb = reinterpret_cast<const float *>(blk);
    const float fc = static_cast<float>(c);
#pragma unroll
    for (int a = 0; a < 3; ++a) pos[a] = __fdiv_rn(fb[(1 + a) * GridBlock<L>::kVox + t], fc);
}

// the reference's per-voxel filter chain: count >= min_count, then (box, frustum) the key range and the fine test on
// the float32 mean widened to double.  pos: the mean, computed here in box and frustum mode only.  A voxel of a block
// past nb (the last CTA of a pass at B < 8) is never kept.
template <int L>
__device__ __forceinline__ bool grid_keep(const GridMeta &G, const GridQuery &Q, uint32_t b, int t, uint32_t nb,
                                          float pos[3], ImagePoint *ip) {
    if (3 * L < 9 && b >= nb) return false;
    const bool spatial = Q.mode != kQueryAll;
    const int4 key = spatial ? G.index.block_keys[b] : make_int4(0, 0, 0, 0);
    if (spatial && !block_in_range<L>(Q, key)) return false;
    const uint32_t *blk = G.pool + static_cast<size_t>(b) * kGridBlockWords<L>;
    const int c = reinterpret_cast<const int *>(blk)[t];
    if (c < Q.min_count) return false;
    if (!spatial) return true;
    if (!voxel_in_range<L>(Q, key, t)) return false;
    grid_mean<L>(blk, t, c, pos);
    const double p[3] = {pos[0], pos[1], pos[2]};
    return region_contains(Q, p, ip);
}

// count -> scan -> emit per CTA: the read-out is in pool order, then voxel order
template <int L>
__global__ void __launch_bounds__(kVox)
grid_query_count_kernel(const GridMeta G, const GridQuery Q, uint32_t *__restrict__ sums, const uint32_t nb) {
    __shared__ uint32_t s_warp[16];
    float pos[3];
    ImagePoint ip;
    uint32_t b;
    int t;
    cta_voxel<L>(&b, &t);
    block_count_512(grid_keep<L>(G, Q, b, t, nb, pos, &ip), s_warp, sums + blockIdx.x);
}

template <int L>
__global__ void __launch_bounds__(kVox)
grid_query_emit_kernel(const GridMeta G, const GridQuery Q, const uint32_t *__restrict__ offs,
                       float *__restrict__ out_pts, float *__restrict__ out_cols, const uint32_t nb) {
    __shared__ uint32_t s_warp[16];
    uint32_t b;
    int t;
    cta_voxel<L>(&b, &t);
    float pos[3];
    ImagePoint ip;
    const bool keep = grid_keep<L>(G, Q, b, t, nb, pos, &ip);
    const uint32_t o = offs[blockIdx.x] + block_excl_scan_512(keep ? 1u : 0u, s_warp);
    if (!keep) return;
    const uint32_t *blk = G.pool + static_cast<size_t>(b) * kGridBlockWords<L>;
    const float *fb = reinterpret_cast<const float *>(blk);
    const int c = reinterpret_cast<const int *>(blk)[t];
    if (Q.mode == kQueryAll) grid_mean<L>(blk, t, c, pos);
    const float fc = static_cast<float>(c);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        out_pts[3 * static_cast<size_t>(o) + k] = pos[k];
        out_cols[3 * static_cast<size_t>(o) + k] = __fdiv_rn(fb[(4 + k) * GridBlock<L>::kVox + t], fc);
    }
}

// carve (voxel_grid_carving.h:47-80): reset voxels that lie in front of the observed depth by more
// than the threshold.  The depth image is indexed with TRUNCATED pixel coordinates, like at<float>(v, u).
template <int L>
__global__ void __launch_bounds__(kVox)
grid_carve_kernel(const GridMeta G, const GridQuery Q, const float *__restrict__ depth, const float thr,
                  const uint32_t nb) {
    uint32_t b;
    int t;
    cta_voxel<L>(&b, &t);
    float pos[3];
    ImagePoint ip;
    if (!grid_keep<L>(G, Q, b, t, nb, pos, &ip)) return;
    const float image_depth = depth[static_cast<size_t>(static_cast<int>(ip.v)) * Q.W + static_cast<int>(ip.u)];
    if (image_depth <= 0.0f || !isfinite(image_depth)) return;
    if (ip.depth < image_depth - thr) {
        uint32_t *blk = G.pool + static_cast<size_t>(b) * kGridBlockWords<L>;
#pragma unroll
        for (int k = 0; k < kGridPlanes; ++k) blk[k * GridBlock<L>::kVox + t] = 0u;
    }
}

// block upload (BlockGridCore::scatter_blocks): one CTA per uploaded block copies every array's run of the block, one
// word W per thread and step, over its pool block's run.  W = uint4 where every run is a multiple of 16 bytes, else
// uint32_t.  A block without a table entry (another shard owns it) or storage (the pool is full) is skipped.  The keys
// went through block_import_kernel in an earlier launch, so the table holds their final entries.
template <typename W>
__global__ void __launch_bounds__(256)
block_scatter_kernel(const int4 *__restrict__ keys, const BlockArrays A, const HashTable T, const uint32_t pool_capacity) {
    __shared__ uint32_t s_idx;
    if (threadIdx.x == 0) {
        const int4 key = keys[blockIdx.x];
        const uint32_t slot = table_find(T, key.x, key.y, key.z);
        const uint32_t idx = slot == kEmpty ? kNoBlock : T.entries[slot].w;
        s_idx = idx < pool_capacity ? idx : kNoBlock;
    }
    __syncthreads();
    const uint32_t idx = s_idx;
    if (idx == kNoBlock) return;
    for (int k = 0; k < A.n_arrays; ++k) {
        const uint32_t words = A.block_bytes[k] / static_cast<uint32_t>(sizeof(W));
        const W *src = static_cast<const W *>(A.src[k]) + static_cast<size_t>(blockIdx.x) * words;
        W *dst = static_cast<W *>(A.dst[k]) + static_cast<size_t>(idx) * words;
        for (uint32_t w = threadIdx.x; w < words; w += blockDim.x) dst[w] = src[w];
    }
}

// ====================================================================================================================
// host side: the block grid core (both grids)
// ====================================================================================================================

RgbdParams rgbd_params(const double K[4], const double Twc[16], float min_depth, float max_depth, int H, int W) {
    RgbdParams P;
    P.fx_inv = 1.0 / K[0];
    P.fy_inv = 1.0 / K[1];
    P.cx = K[2];
    P.cy = K[3];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) P.R[3 * i + j] = Twc[4 * i + j];
        P.t[i] = Twc[4 * i + 3];
    }
    P.min_depth = min_depth;
    P.max_depth = max_depth;
    P.H = H;
    P.W = W;
    return P;
}

int BlockGridCore::log2_block_size(int32_t block_size) {
    for (int l = 0; l <= kMaxGridLog2B; ++l)
        if (block_size == (1 << l) && grid_log2_block_supported(l)) return l;
    return -1;
}

bool BlockGridCore::valid_args(double voxel_size, int32_t block_size, uint32_t capacity_blocks,
                               uint32_t max_capacity_blocks) {
    const int l = log2_block_size(block_size);
    return l >= 0 && voxel_size > 0.0 && capacity_blocks != 0 &&
           (max_capacity_blocks == 0 || (max_capacity_blocks >= capacity_blocks && max_capacity_blocks <= max_blocks(l)));
}

int BlockGridCore::create(double voxel_size, int32_t block_size, uint32_t capacity_blocks, uint32_t max_capacity_blocks,
                          int32_t dev) {
    inv_voxel_size = 1.0f / static_cast<float>(voxel_size);
    log2_block = log2_block_size(block_size);
    device = dev;
    const uint32_t cap = std::max(capacity_blocks, max_capacity_blocks);
    growable = cap > capacity_blocks;
    index.capacity = cap;
    B2V_CUDA(this, cudaSetDevice(device));
    B2V_CUDA(this, cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    const uint32_t tcap = next_pow2(static_cast<uint64_t>(cap) * 2);
    table.mask = tcap - 1;
    B2V_CUDA(this, table_mem.reserve(tcap));
    B2V_CUDA(this, block_keys.reserve(cap));
    B2V_CUDA(this, counters.reserve(kBgNumCounters));
    B2V_CUDA(this, d_total.reserve(1));
    table.entries = table_mem.get();
    index.block_keys = block_keys.get();
    index.counters = counters.get();
    B2V_CUDA(this, cudaMallocHost(&h_counters, kBgNumCounters * sizeof(uint32_t)));
    return B2V_OK;
}

void BlockGridCore::destroy() {
    cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);
    cudaFreeHost(h_counters);
    if (stream) cudaStreamDestroy(stream);
}

int BlockGridCore::fetch_counters() {
    B2V_CUDA(this, cudaSetDevice(device));
    B2V_CUDA(this, cudaMemcpyAsync(h_counters, index.counters, kBgNumCounters * sizeof(uint32_t),
                                   cudaMemcpyDeviceToHost, stream));
    B2V_CUDA(this, cudaStreamSynchronize(stream));
    return B2V_OK;
}

int BlockGridCore::read_counters() {
    const int rc = fetch_counters();
    if (rc != B2V_OK) return rc;
    if (h_counters[kBgError]) {
        err = (h_counters[kBgError] & 2u) ? "hash table full: raise capacity_blocks"
                                          : "block pool full: raise capacity_blocks";
        return B2V_ERR_CAPACITY;
    }
    return B2V_OK;
}

int BlockGridCore::capacity(int64_t *capacity_blocks, int64_t *growths_out) {
    B2V_CUDA(this, cudaSetDevice(device));
    B2V_CUDA(this, cudaStreamSynchronize(stream));
    if (capacity_blocks) *capacity_blocks = index.pool_capacity;
    if (growths_out) *growths_out = growths;
    return B2V_OK;
}

int BlockGridCore::set_shard(int32_t rank, int32_t count) {
    if (count < 1 || rank < 0 || rank >= count) {
        err = "set_shard: need shard_count >= 1 and 0 <= shard_rank < shard_count";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    const int rc = fetch_counters();
    if (rc != B2V_OK) return rc;
    if (h_counters[kBgPool] != 0) {   // blocks of another partition may already be in the table
        err = "set_shard: the grid holds blocks (clear it first)";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    index.shard_rank = static_cast<uint32_t>(rank);
    index.shard_count = static_cast<uint32_t>(count);
    return B2V_OK;
}

int BlockGridCore::clear_index() {
    B2V_CUDA(this, cudaMemsetAsync(table.entries, 0xFF, (static_cast<size_t>(table.mask) + 1) * sizeof(uint4), stream));
    B2V_CUDA(this, cudaMemsetAsync(index.counters, 0, kBgNumCounters * sizeof(uint32_t), stream));
    return B2V_OK;
}

int BlockGridCore::insert_keys(int64_t n, const int32_t *keys4, DeviceBuffer<int4> *d_keys) {
    B2V_CUDA(this, d_keys->reserve(static_cast<size_t>(n)));
    B2V_CUDA(this, cudaMemcpyAsync(d_keys->get(), keys4, static_cast<size_t>(n) * sizeof(int4), cudaMemcpyHostToDevice,
                                   stream));
    block_import_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(
        d_keys->get(), static_cast<uint32_t>(n), table, index);
    B2V_CUDA(this, cudaGetLastError());
    return B2V_OK;
}

int BlockGridCore::scatter_blocks(int64_t n, const int4 *d_keys, const BlockArrays &arrays) {
    BlockArrays A = arrays;   // with src[k] staged on the device, one array after the other
    size_t bytes = 0;
    bool runs16 = true;
    for (int k = 0; k < A.n_arrays; ++k) {
        bytes += static_cast<size_t>(n) * A.block_bytes[k];
        runs16 = runs16 && A.block_bytes[k] % 16 == 0;
    }
    DeviceBuffer<uint8_t> d_src;
    B2V_CUDA(this, d_src.reserve(bytes));
    size_t off = 0;
    for (int k = 0; k < A.n_arrays; ++k) {
        const size_t run = static_cast<size_t>(n) * A.block_bytes[k];
        B2V_CUDA(this, cudaMemcpyAsync(d_src.get() + off, arrays.src[k], run, cudaMemcpyHostToDevice, stream));
        A.src[k] = d_src.get() + off;
        off += run;
    }
    if (runs16)
        block_scatter_kernel<uint4><<<static_cast<unsigned>(n), 256, 0, stream>>>(d_keys, A, table,
                                                                                 index.pool_capacity);
    else
        block_scatter_kernel<uint32_t><<<static_cast<unsigned>(n), 256, 0, stream>>>(d_keys, A, table,
                                                                                    index.pool_capacity);
    B2V_CUDA(this, cudaGetLastError());
    B2V_CUDA(this, cudaStreamSynchronize(stream));
    return B2V_OK;
}

int BlockGridCore::reserve_sort(size_t cap) {
    size_t tmp = 0;
    B2V_CUDA(this, cub::DeviceRadixSort::SortPairs(nullptr, tmp, sort.vid[0].get(), sort.vid[1].get(), sort.ord[0].get(),
                                                  sort.ord[1].get(), static_cast<int64_t>(cap), 0, 32, stream));
    B2V_CUDA(this, sort.tmp.reserve(tmp));
    for (int k = 0; k < 2; ++k) {   // ord[1] last: it holds cap only once every buffer does
        B2V_CUDA(this, sort.vid[k].reserve(cap));
        B2V_CUDA(this, sort.ord[k].reserve(cap));
    }
    return B2V_OK;
}

cudaError_t BlockGridCore::sort_voxels(const void *pts, bool pts_f64, const uint8_t *valid, int64_t n, uint32_t lo,
                                       uint32_t hi) {
    if (n <= 0) return cudaSuccess;
    const unsigned grid = static_cast<unsigned>((n + 255) / 256);
    dispatch([&](auto l) {
        constexpr int L = decltype(l)::value;
        if (pts_f64)
            voxel_keys_kernel<double, L><<<grid, 256, 0, stream>>>(static_cast<const double *>(pts), valid, n,
                                                                   inv_voxel_size, table, lo, hi, sort.vid[0].get(),
                                                                   sort.ord[0].get());
        else
            voxel_keys_kernel<float, L><<<grid, 256, 0, stream>>>(static_cast<const float *>(pts), valid, n,
                                                                  inv_voxel_size, table, lo, hi, sort.vid[0].get(),
                                                                  sort.ord[0].get());
    });
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    size_t tmp = sort.tmp.size();  // all 32 key bits: kBadVid (points without storage) must sort last
    return cub::DeviceRadixSort::SortPairs(sort.tmp.get(), tmp, sort.vid[0].get(), sort.vid[1].get(), sort.ord[0].get(),
                                           sort.ord[1].get(), n, 0, 32, stream);
}

int BlockGridCore::ensure_scan(uint32_t n) {
    // room for twice the CTAs, so a growing map rarely reallocates
    if (n > d_sums.size()) B2V_CUDA(this, d_sums.reserve(static_cast<size_t>(n) * 2));
    if (n > d_offs.size()) B2V_CUDA(this, d_offs.reserve(static_cast<size_t>(n) * 2));
    return B2V_OK;
}

cudaError_t BlockGridCore::scan_total(uint32_t n, uint32_t *total) {
    *total = 0;
    if (n == 0) return cudaSuccess;
    exclusive_scan_kernel<<<1, 1024, 0, stream>>>(d_sums.get(), d_offs.get(), d_total.get(), n);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(total, d_total.get(), sizeof(uint32_t), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    return e;
}

GridQuery BlockGridCore::all_query(int min_count) const {
    GridQuery q;
    std::memset(&q, 0, sizeof(q));
    q.mode = kQueryAll;
    q.min_count = min_count;
    return q;
}

static void key_bounds(GridQuery *q, float inv_vs) {
    for (int a = 0; a < 3; ++a) {
        q->min_key[a] = static_cast<int32_t>(std::floor(q->bb[a] * static_cast<double>(inv_vs)));
        q->max_key[a] = static_cast<int32_t>(std::floor(q->bb[3 + a] * static_cast<double>(inv_vs)));
    }
}

GridQuery BlockGridCore::box_query(const double bbox[6], int min_count) const {
    GridQuery q = all_query(min_count);
    q.mode = kQueryBox;
    for (int a = 0; a < 6; ++a) q.bb[a] = bbox[a];
    key_bounds(&q, inv_voxel_size);
    return q;
}

GridQuery BlockGridCore::frustum_query(const float K[4], int W, int H, const double Tcw[16], float depth_max,
                                       float depth_min, int min_count) const {
    GridQuery q = all_query(min_count);
    q.mode = kQueryFrustum;
    q.fx = K[0];
    q.fy = K[1];
    q.cx = K[2];
    q.cy = K[3];
    q.depth_min = depth_min;
    q.depth_max = depth_max;
    q.W = W;
    q.H = H;
    double Rwc[9], twc[3];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) {
            q.R[3 * i + j] = Tcw[4 * i + j];
            Rwc[3 * i + j] = Tcw[4 * j + i];
        }
        q.t[i] = Tcw[4 * i + 3];
    }
    for (int i = 0; i < 3; ++i) twc[i] = -(Rwc[3 * i] * q.t[0] + Rwc[3 * i + 1] * q.t[1] + Rwc[3 * i + 2] * q.t[2]);
    for (int a = 0; a < 3; ++a) {
        q.bb[a] = 1e300;
        q.bb[3 + a] = -1e300;
    }
    const double us[4] = {0.0, static_cast<double>(W), static_cast<double>(W), 0.0};
    const double vs[4] = {0.0, 0.0, static_cast<double>(H), static_cast<double>(H)};
    for (int c = 0; c < 4; ++c) {
        const double xn = (us[c] - static_cast<double>(q.cx)) / static_cast<double>(q.fx);
        const double yn = (vs[c] - static_cast<double>(q.cy)) / static_cast<double>(q.fy);
        for (int far = 0; far < 2; ++far) {
            const double d = far ? static_cast<double>(depth_max) : static_cast<double>(depth_min);
            const double pc[3] = {xn * d, yn * d, d};
            for (int a = 0; a < 3; ++a) {
                const double w = Rwc[3 * a] * pc[0] + Rwc[3 * a + 1] * pc[1] + Rwc[3 * a + 2] * pc[2] + twc[a];
                q.bb[a] = std::min(q.bb[a], w);
                q.bb[3 + a] = std::max(q.bb[3 + a], w);
            }
        }
    }
    key_bounds(&q, inv_voxel_size);
    return q;
}

int BlockGridCore::stage_input(const char *fn, int H, int W, bool filter_shadow_points, const float **depth,
                               const uint8_t **rgb, const int32_t **cls, const int32_t **obj) {
    if (filter_shadow_points && (H <= 2 || W <= 2)) {
        err = std::string(fn) + ": image too small for the shadow filter";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    B2V_CUDA(this, cudaSetDevice(device));
    const size_t pixels = static_cast<size_t>(H) * W;
    auto on_host = [](auto **p) { return p && *p && !is_device_pointer(*p); };
    // Each group below synchronises when the last buffer it reserves is short: that buffer only ever held what
    // the ones before it were reserved for, so no buffer that holds memory is reallocated without the wait.
    if (filter_shadow_points || on_host(depth) || on_host(rgb)) {
        if (pixels * 3 > input.rgb.size()) B2V_CUDA(this, cudaStreamSynchronize(stream));
        B2V_CUDA(this, input.depth.reserve(pixels));
        B2V_CUDA(this, input.filtered.reserve(pixels));
        B2V_CUDA(this, input.shadow_scratch.reserve(kShadowScratchBytes));
        B2V_CUDA(this, input.rgb.reserve(pixels * 3));
    }
    if (on_host(cls) || on_host(obj)) {
        if (pixels > input.obj.size()) B2V_CUDA(this, cudaStreamSynchronize(stream));
        B2V_CUDA(this, input.cls.reserve(pixels));
        B2V_CUDA(this, input.obj.reserve(pixels));
    }
    cudaError_t e = cudaSuccess;
    auto upload = [&](auto **p, void *buf, size_t bytes) {
        if (e != cudaSuccess || !on_host(p)) return;
        e = cudaMemcpyAsync(buf, *p, bytes, cudaMemcpyHostToDevice, stream);
        *p = static_cast<std::remove_reference_t<decltype(*p)>>(buf);
    };
    upload(depth, input.depth.get(), pixels * sizeof(float));
    upload(rgb, input.rgb.get(), pixels * 3);
    upload(cls, input.cls.get(), pixels * sizeof(int32_t));
    upload(obj, input.obj.get(), pixels * sizeof(int32_t));
    if (e == cudaSuccess && filter_shadow_points) {
        e = launch_filter_shadow_points(*depth, H, W, 2, 2, -1.0f, input.filtered.get(), input.shadow_scratch.get(),
                                        stream);
        *depth = input.filtered.get();
    }
    if (e != cudaSuccess) {
        err = std::string(fn) + ": " + cudaGetErrorString(e);
        return B2V_ERR_CUDA;
    }
    return B2V_OK;
}

int BlockGridCore::set_rectification(const float *map_x, const float *map_y, int H, int W, int swap_rb) {
    if (map_x && map_y && (H <= 0 || W <= 0)) {
        err = "set_rectification: bad image size";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    B2V_CUDA(this, cudaSetDevice(device));
    B2V_CUDA(this, cudaStreamSynchronize(stream));
    frame.mapx = {};
    frame.mapy = {};
    frame.map_h = frame.map_w = 0;
    frame.swap_rb = swap_rb;
    if (!map_x || !map_y) return B2V_OK;
    const size_t pixels = static_cast<size_t>(H) * W;
    B2V_CUDA(this, frame.mapx.reserve(pixels));
    B2V_CUDA(this, frame.mapy.reserve(pixels));
    B2V_CUDA(this, cudaMemcpy(frame.mapx.get(), map_x, pixels * sizeof(float), cudaMemcpyDefault));
    B2V_CUDA(this, cudaMemcpy(frame.mapy.get(), map_y, pixels * sizeof(float), cudaMemcpyDefault));
    frame.map_h = H;
    frame.map_w = W;
    return B2V_OK;
}

int BlockGridCore::set_frame(const void *depth, bool depth_u16, float depth_scale, const uint8_t *color,
                             const int32_t *cls, const int32_t *inst, int H, int W, bool filter_shadow_points,
                             b2v_frame *out) {
    const char *bad = nullptr;
    if (!depth || !color || !out || H <= 0 || W <= 0) bad = "set_frame: bad arguments";
    else if (depth_u16 && !(depth_scale > 0.0f)) bad = "set_frame: uint16 depth needs a positive depth_scale";
    else if (inst && !cls) bad = "set_frame: an instance image needs a class image";
    else if (frame.mapx.get() && (H != frame.map_h || W != frame.map_w))
        bad = "set_frame: rectification maps were installed for a different image size";
    else if (filter_shadow_points && (H <= 2 || W <= 2)) bad = "set_frame: image too small for the shadow filter";
    frame_store.begin_call(1);   // (also when the call fails)
    if (bad) {
        err = bad;
        return B2V_ERR_INVALID_ARGUMENT;
    }
    B2V_CUDA(this, cudaSetDevice(device));
    const size_t pixels = static_cast<size_t>(H) * W;
    {
        const int rc = reserve_frame(pixels, cls != nullptr);
        if (rc != B2V_OK) return rc;
    }
    cudaStream_t s = stream;
    const bool rect = frame.mapx.get() != nullptr;
    void *const raw = frame.raw.get();
    cudaError_t e = cudaSuccess;
    // a host image is uploaded into `dst`, a device image is read in place.  Uploads through frame.raw are ordered
    // after the kernels that read the previous one (one stream).
    auto input = [&](const void *src, size_t bytes, void *dst) -> const void * {
        if (e != cudaSuccess || is_device_pointer(src)) return src;
        e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s);
        return dst;
    };
    // 32-bit image (depth, labels) into its staged buffer: nearest remap, or a copy without maps
    auto place_b32 = [&](const void *src, void *dst) {
        if (e != cudaSuccess) return;
        if (rect)
            e = launch_remap_b32_nearest(src, H, W, frame.mapx.get(), frame.mapy.get(), dst, s);
        else if (src != dst)
            e = cudaMemcpyAsync(dst, src, pixels * 4, cudaMemcpyDeviceToDevice, s);
    };
    // depth: upload -> widen (uint16; into `filtered`, free until the filter runs, when the remap follows) -> remap
    const void *d = input(depth, pixels * (depth_u16 ? 2 : 4), (depth_u16 || rect) ? raw : frame.depth.get());
    if (depth_u16 && e == cudaSuccess) {
        float *wide = rect ? frame.filtered.get() : frame.depth.get();
        e = launch_depth_u16_to_f32(static_cast<const uint16_t *>(d), wide, pixels, depth_scale, s);
        d = wide;
    }
    place_b32(d, frame.depth.get());
    const void *c = input(color, pixels * 3, rect ? raw : frame.rgb.get());
    if (e == cudaSuccess) {
        if (rect)
            e = launch_remap_u8c3_linear(static_cast<const uint8_t *>(c), H, W, frame.mapx.get(), frame.mapy.get(),
                                         frame.rgb.get(), frame.swap_rb, s);
        else if (c != frame.rgb.get())
            e = cudaMemcpyAsync(frame.rgb.get(), c, pixels * 3, cudaMemcpyDeviceToDevice, s);
    }
    if (cls) place_b32(input(cls, pixels * 4, rect ? raw : frame.cls.get()), frame.cls.get());
    if (inst) place_b32(input(inst, pixels * 4, rect ? raw : frame.inst.get()), frame.inst.get());
    if (e == cudaSuccess && filter_shadow_points)
        e = launch_filter_shadow_points(frame.depth.get(), H, W, 2, 2, -1.0f, frame.filtered.get(),
                                        frame.shadow_scratch.get(), s);
    // the frame store: the staged images into the next slot, before the synchronise below
    int32_t stored = -1;
    if (e == cudaSuccess && frame_store.max > 0) {
        frame_store.assign(1, H, W, grid_record_pitch(pixels, frame_labels), device, s);
        if (frame_store.last[0] >= 0) {
            e = launch_grid_frame_pack(frame.depth.get(), filter_shadow_points ? frame.filtered.get() : nullptr,
                                       frame.rgb.get(), cls ? frame.cls.get() : nullptr,
                                       inst ? frame.inst.get() : nullptr, pixels, frame_labels,
                                       frame_store.slot(frame_store.last[0]), s);
            if (e == cudaSuccess) stored = frame_store.last[0];
        }
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
        frame_store.drop_unfilled();
        err = std::string("set_frame: ") + cudaGetErrorString(e);
        return B2V_ERR_CUDA;
    }
    if (stored >= 0) {
        frame_store.filled(stored);
        store_flags.resize(static_cast<size_t>(frame_store.count));
        store_flags[stored] = static_cast<uint8_t>((cls ? kStoredClass : 0) | (inst ? kStoredInstance : 0) |
                                                   (filter_shadow_points ? kStoredFiltered : 0));
    }
    finish_frame(H, W, filter_shadow_points, cls != nullptr, inst != nullptr, out);
    return B2V_OK;
}

int BlockGridCore::reserve_frame(size_t pixels, bool labels) {
    frame.staged = b2v_frame{};
    // synchronise when the last buffer of a group is short, as stage_input does
    if (pixels * 3 > frame.rgb.size()) B2V_CUDA(this, cudaStreamSynchronize(stream));
    B2V_CUDA(this, frame.raw.reserve(pixels));
    B2V_CUDA(this, frame.depth.reserve(pixels));
    B2V_CUDA(this, frame.filtered.reserve(pixels));
    B2V_CUDA(this, frame.shadow_scratch.reserve(kShadowScratchBytes));
    B2V_CUDA(this, frame.rgb.reserve(pixels * 3));
    if (labels) {
        if (pixels > frame.obj.size()) B2V_CUDA(this, cudaStreamSynchronize(stream));
        B2V_CUDA(this, frame.cls.reserve(pixels));
        B2V_CUDA(this, frame.inst.reserve(pixels));
        B2V_CUDA(this, frame.obj.reserve(pixels));
    }
    return B2V_OK;
}

void BlockGridCore::finish_frame(int H, int W, bool filtered, bool cls, bool inst, b2v_frame *out) {
    frame.staged.depth = frame.depth.get();
    frame.staged.filtered_depth = filtered ? frame.filtered.get() : frame.depth.get();
    frame.staged.color = frame.rgb.get();
    frame.staged.class_image = cls ? frame.cls.get() : nullptr;
    frame.staged.instance_image = inst ? frame.inst.get() : nullptr;
    frame.staged.height = H;
    frame.staged.width = W;
    *out = frame.staged;
}

int BlockGridCore::set_frame_store(int32_t max_frames) {
    if (max_frames < 0) {
        err = "set_frame_store: max_frames must be >= 0";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    B2V_CUDA(this, cudaSetDevice(device));
    B2V_CUDA(this, cudaStreamSynchronize(stream));
    frame_store.release();
    store_flags.clear();
    frame_store.max = max_frames;
    return B2V_OK;
}

int BlockGridCore::stage_stored(int32_t slot, b2v_frame *out) {
    if (!out || !frame_store.holds(slot)) {
        err = "stage_stored: slot " + std::to_string(slot) + " holds no frame (the store holds " +
              std::to_string(frame_store.count) + ")";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    B2V_CUDA(this, cudaSetDevice(device));
    const size_t pixels = static_cast<size_t>(frame_store.H) * frame_store.W;
    const uint8_t fl = store_flags[slot];
    const bool filtered = fl & kStoredFiltered, cls = fl & kStoredClass, inst = fl & kStoredInstance;
    {
        const int rc = reserve_frame(pixels, cls);
        if (rc != B2V_OK) return rc;
    }
    cudaError_t e = launch_grid_frame_unpack(frame_store.slot(slot), pixels, frame_labels, frame.depth.get(),
                                             filtered ? frame.filtered.get() : nullptr, frame.rgb.get(),
                                             cls ? frame.cls.get() : nullptr, inst ? frame.inst.get() : nullptr,
                                             stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) {
        err = std::string("stage_stored: ") + cudaGetErrorString(e);
        return B2V_ERR_CUDA;
    }
    finish_frame(frame_store.H, frame_store.W, filtered, cls, inst, out);
    return B2V_OK;
}

}  // namespace b2v

// ====================================================================================================================
// host side: the C ABI of the point-average grid (b2v_grid_*)
// ====================================================================================================================
using namespace b2v;

struct b2v_grid : BlockGridCore {
    // the pool is a reservation for index.capacity blocks with storage mapped for index.pool_capacity (a fixed grid
    // maps it whole at create); a growable grid maps more inside the integrate call that needs it
    VmmRange pool;
    DeviceBuffer<float> d_pts, d_cols, d_out_pts, d_out_cols;   // staging of host points, read-out
    int64_t last_n = 0;
    bool input_order = false;   // b2v_grid_set_input_order_sums
    // point records and mask of an input-order integrate_rgbd; d_valid's size is their capacity
    DeviceBuffer<float> d_rec_pts, d_rec_cols;
    DeviceBuffer<uint8_t> d_valid;

    GridMeta meta() const { return GridMeta{reinterpret_cast<uint32_t *>(pool.va), index}; }
    size_t block_bytes() const { return static_cast<size_t>(kGridPlanes) * block_voxels() * sizeof(uint32_t); }
};

extern "C" const char *b2v_grid_last_error(const b2v_grid *g) { return g ? g->err.c_str() : "null grid"; }

// map storage for at least `blocks` blocks; index.pool_capacity becomes what the mapping holds.  False if it failed.
static bool grid_map_storage(b2v_grid *g, uint64_t blocks, std::string *err) {
    const bool ok = vmm_map(&g->pool, static_cast<size_t>(blocks) * g->block_bytes(), g->stream, err);
    g->index.pool_capacity =
        static_cast<uint32_t>(std::min<size_t>(g->index.capacity, g->pool.mapped / g->block_bytes()));
    return ok;
}

// the storage growth of BlockGridCore::resolve / upload_blocks
static auto grid_grow_storage(b2v_grid *g) {
    return [g](uint64_t blocks) {
        std::string map_err;   // a failed mapping surfaces as "block pool full"
        grid_map_storage(g, blocks, &map_err);
    };
}

static int grid_clear_device(b2v_grid *g, uint32_t used_blocks) {
    const int rc = g->clear_index();
    if (rc != B2V_OK) return rc;
    B2V_CUDA(g, cudaMemsetAsync(reinterpret_cast<void *>(g->pool.va), 0, static_cast<size_t>(used_blocks) * g->block_bytes(),
                                g->stream));
    return B2V_OK;
}

extern "C" int b2v_grid_create_ex(float voxel_size, int32_t block_size, uint32_t capacity_blocks,
                                  uint32_t max_capacity_blocks, int32_t device, b2v_grid **out) {
    if (!out) return B2V_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    if (!BlockGridCore::valid_args(voxel_size, block_size, capacity_blocks, max_capacity_blocks))
        return B2V_ERR_INVALID_ARGUMENT;
    b2v_grid *g = new (std::nothrow) b2v_grid();
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    *out = g;
    int rc = g->create(voxel_size, block_size, capacity_blocks, max_capacity_blocks, device);
    if (rc != B2V_OK) return rc;
    if (!vmm_reserve(&g->pool, static_cast<size_t>(g->index.capacity) * g->block_bytes(), device, &g->err) ||
        !grid_map_storage(g, capacity_blocks, &g->err))
        return B2V_ERR_CUDA;
    g->index.pool_capacity = capacity_blocks;   // the rest of the last granule is used only after a growth
    rc = grid_clear_device(g, capacity_blocks);
    if (rc != B2V_OK) return rc;
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    return B2V_OK;
}

extern "C" int b2v_grid_destroy(b2v_grid *g) {
    if (!g) return B2V_OK;
    g->destroy();
    delete g;
    return B2V_OK;
}

extern "C" int b2v_grid_capacity(b2v_grid *g, int64_t *capacity_blocks, int64_t *growths) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->capacity(capacity_blocks, growths);
}

extern "C" int b2v_grid_set_shard(b2v_grid *g, int32_t shard_rank, int32_t shard_count) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->set_shard(shard_rank, shard_count);
}

extern "C" int b2v_grid_clear(b2v_grid *g) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    int rc = g->read_counters();
    if (rc == B2V_ERR_CUDA) return rc;
    rc = grid_clear_device(g, g->block_count());
    if (rc != B2V_OK) return rc;
    g->err.clear();
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    return B2V_OK;
}

// the accumulate pass over the points whose block's pool index lies in [lo, hi)
template <typename Tp>
static cudaError_t grid_accumulate_t(const b2v_grid *g, const Tp *p, const void *cols, bool cols_u8, int64_t n,
                                     uint32_t lo, uint32_t hi) {
    const unsigned grid = static_cast<unsigned>((n + 255) / 256);
    g->dispatch([&](auto l) {
        constexpr int L = decltype(l)::value;
        if (cols_u8)
            grid_accumulate_kernel<Tp, uint8_t, L><<<grid, 256, 0, g->stream>>>(
                p, static_cast<const uint8_t *>(cols), n, g->inv_voxel_size, g->table, g->meta(), lo, hi);
        else
            grid_accumulate_kernel<Tp, float, L><<<grid, 256, 0, g->stream>>>(
                p, static_cast<const float *>(cols), n, g->inv_voxel_size, g->table, g->meta(), lo, hi);
    });
    return cudaGetLastError();
}

static cudaError_t grid_accumulate(const b2v_grid *g, const void *pts, bool pts_f64, const void *cols, bool cols_u8,
                                   int64_t n, uint32_t lo, uint32_t hi) {
    if (pts_f64) return grid_accumulate_t(g, static_cast<const double *>(pts), cols, cols_u8, n, lo, hi);
    return grid_accumulate_t(g, static_cast<const float *>(pts), cols, cols_u8, n, lo, hi);
}

// an input-order call takes at most this many points: the sort's values are uint32 point indices (as the semantic
// grids' b2v_sgrid_integrate)
constexpr int64_t kMaxOrderedPoints = 0x7FFFFFF0LL;

extern "C" int b2v_grid_set_input_order_sums(b2v_grid *g, int32_t enable) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (enable && g->index.capacity > BlockGridCore::max_blocks(g->log2_block)) {
        g->err = "b2v_grid_set_input_order_sums: the grid holds more than 2^31 voxels";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    g->input_order = enable != 0;
    return B2V_OK;
}

// Room for n points of an input-order pass: the voxel sort and, with `records`, the point records of integrate_rgbd.
// Queued passes may still read these buffers, so a reallocation waits for the stream.
static int grid_reserve_ordered(b2v_grid *g, size_t n, bool records) {
    const bool sort_short = n > g->sort.ord[1].size(), rec_short = records && n > g->d_valid.size();
    if (!sort_short && !rec_short) return B2V_OK;
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    const size_t cap = n + n / 4 + 1024;
    if (rec_short) {
        B2V_CUDA(g, g->d_rec_pts.reserve(cap * 3));
        B2V_CUDA(g, g->d_rec_cols.reserve(cap * 3));
        B2V_CUDA(g, g->d_valid.reserve(cap));
    }
    return sort_short ? g->reserve_sort(cap) : B2V_OK;
}

// the input-order pass over the points whose block's pool index lies in [lo, hi): keys -> sort -> runs
template <typename Tp>
static cudaError_t grid_sum_in_order_t(b2v_grid *g, const Tp *p, const void *cols, bool cols_u8,
                                       const uint8_t *valid, int64_t n, uint32_t lo, uint32_t hi) {
    cudaError_t e = g->sort_voxels(p, sizeof(Tp) == sizeof(double), valid, n, lo, hi);
    if (e != cudaSuccess) return e;
    const unsigned grid = static_cast<unsigned>((n + 255) / 256);
    const uint32_t *vid = g->sort.vid[1].get(), *ord = g->sort.ord[1].get();
    g->dispatch([&](auto l) {
        constexpr int L = decltype(l)::value;
        if (cols_u8)
            grid_runs_kernel<Tp, uint8_t, L><<<grid, 256, 0, g->stream>>>(vid, ord, n, p,
                                                                          static_cast<const uint8_t *>(cols), g->meta());
        else
            grid_runs_kernel<Tp, float, L><<<grid, 256, 0, g->stream>>>(vid, ord, n, p,
                                                                        static_cast<const float *>(cols), g->meta());
    });
    return cudaGetLastError();
}

static cudaError_t grid_sum_in_order(b2v_grid *g, const void *pts, bool pts_f64, const void *cols, bool cols_u8,
                                     const uint8_t *valid, int64_t n, uint32_t lo, uint32_t hi) {
    if (pts_f64)
        return grid_sum_in_order_t(g, static_cast<const double *>(pts), cols, cols_u8, valid, n, lo, hi);
    return grid_sum_in_order_t(g, static_cast<const float *>(pts), cols, cols_u8, valid, n, lo, hi);
}

extern "C" int b2v_grid_integrate_ex(b2v_grid *g, const void *points, int32_t points_f64, const void *colors,
                                     int32_t colors_u8, int64_t n_points) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (n_points < 0 || (n_points > 0 && !points)) {
        g->err = "b2v_grid_integrate_ex: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    if (g->input_order && n_points > kMaxOrderedPoints) {
        g->err = "b2v_grid_integrate_ex: more than 0x7FFFFFF0 points in one call with input-order sums";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    if (n_points == 0) return B2V_OK;  // voxel_block_grid.hpp:22-24,121-123
    B2V_CUDA(g, cudaSetDevice(g->device));
    const bool f64 = points_f64 != 0, u8 = colors_u8 != 0;
    if (g->input_order) {
        const int rc = grid_reserve_ordered(g, static_cast<size_t>(n_points), false);
        if (rc != B2V_OK) return rc;
    }
    const void *d_p = points;
    const void *d_c = colors;
    const bool dev_p = is_device_pointer(points);
    const bool dev_c = colors ? is_device_pointer(colors) : true;
    if (!dev_p || !dev_c) {
        const size_t n = static_cast<size_t>(n_points);
        if (n * 3 > g->d_cols.size()) B2V_CUDA(g, cudaStreamSynchronize(g->stream));   // reserved last
        B2V_CUDA(g, g->d_pts.reserve(n * 3 * 2));  // room for float64 points
        B2V_CUDA(g, g->d_cols.reserve(n * 3));
        if (!dev_p) {
            B2V_CUDA(g, cudaMemcpyAsync(g->d_pts.get(), points, static_cast<size_t>(n_points) * 3 * (f64 ? sizeof(double) : sizeof(float)),
                                        cudaMemcpyHostToDevice, g->stream));
            d_p = g->d_pts.get();
        }
        if (colors && !dev_c) {
            B2V_CUDA(g, cudaMemcpyAsync(g->d_cols.get(), colors, static_cast<size_t>(n_points) * 3 * (u8 ? 1 : sizeof(float)),
                                        cudaMemcpyHostToDevice, g->stream));
            d_c = g->d_cols.get();
        }
    }
    B2V_CUDA(g, launch_point_insert(d_p, f64, nullptr, n_points, g->inv_voxel_size, g->log2_block, g->table, g->index,
                                    g->stream));
    // a voxel's run is its only update in a pass, so the growth replay over the new blocks is exact in either mode
    const bool ordered = g->input_order;
    auto pass = [&](uint32_t lo, uint32_t hi) {
        return ordered ? grid_sum_in_order(g, d_p, f64, d_c, u8, nullptr, n_points, lo, hi)
                       : grid_accumulate(g, d_p, f64, d_c, u8, n_points, lo, hi);
    };
    B2V_CUDA(g, pass(0u, g->index.pool_capacity));
    if (!g->growable) return B2V_OK;
    return g->resolve(grid_grow_storage(g), [&](uint32_t lo, uint32_t hi) {
        B2V_CUDA(g, pass(lo, hi));
        return B2V_OK;
    });
}

extern "C" int b2v_grid_integrate_rgbd(b2v_grid *g, const float *depth, const uint8_t *color, int32_t height,
                                       int32_t width, const double K[4], const double Twc[16], float max_depth,
                                       float min_depth, int32_t filter_shadow_points) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (!depth || !color || !K || !Twc || height <= 0 || width <= 0) {
        g->err = "b2v_grid_integrate_rgbd: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    const int64_t n = static_cast<int64_t>(height) * width;
    if (g->input_order && n > kMaxOrderedPoints) {
        g->err = "b2v_grid_integrate_rgbd: more than 0x7FFFFFF0 pixels with input-order sums";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    const float *d_depth = depth;
    const uint8_t *d_color = color;
    // voxel_grid.py:238-245: depth2pointcloud sees the filtered depth
    int rc = g->stage_input("b2v_grid_integrate_rgbd", height, width, filter_shadow_points != 0, &d_depth, &d_color);
    if (rc != B2V_OK) return rc;
    const RgbdParams P = rgbd_params(K, Twc, min_depth, max_depth, height, width);
    if (g->input_order) {   // point records -> the input-order path of b2v_grid_integrate_ex
        rc = grid_reserve_ordered(g, static_cast<size_t>(n), true);
        if (rc != B2V_OK) return rc;
        const float *pts = g->d_rec_pts.get(), *cols = g->d_rec_cols.get();
        const uint8_t *valid = g->d_valid.get();
        grid_rgbd_points_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, g->stream>>>(
            P, d_depth, d_color, g->d_rec_pts.get(), g->d_rec_cols.get(), g->d_valid.get());
        B2V_CUDA(g, cudaGetLastError());
        B2V_CUDA(g, launch_point_insert(pts, false, valid, n, g->inv_voxel_size, g->log2_block, g->table, g->index,
                                        g->stream));
        B2V_CUDA(g, grid_sum_in_order(g, pts, false, cols, false, valid, n, 0u, g->index.pool_capacity));
        if (!g->growable) return B2V_OK;
        return g->resolve(grid_grow_storage(g), [&](uint32_t lo, uint32_t hi) {
            B2V_CUDA(g, grid_sum_in_order(g, pts, false, cols, false, valid, n, lo, hi));
            return B2V_OK;
        });
    }
    const unsigned grid = static_cast<unsigned>((static_cast<size_t>(height) * width + 255) / 256);
    auto accumulate = [&](uint32_t lo, uint32_t hi) {
        g->dispatch([&](auto l) {
            grid_rgbd_accumulate_kernel<decltype(l)::value><<<grid, 256, 0, g->stream>>>(
                P, d_depth, d_color, g->inv_voxel_size, g->table, g->meta(), lo, hi);
        });
    };
    g->dispatch([&](auto l) {
        grid_rgbd_insert_kernel<decltype(l)::value><<<grid, 256, 0, g->stream>>>(P, d_depth, g->inv_voxel_size,
                                                                                g->table, g->index);
    });
    accumulate(0u, g->index.pool_capacity);
    B2V_CUDA(g, cudaGetLastError());
    if (!g->growable) return B2V_OK;
    return g->resolve(grid_grow_storage(g), [&](uint32_t lo, uint32_t hi) {
        accumulate(lo, hi);
        B2V_CUDA(g, cudaGetLastError());
        return B2V_OK;
    });
}

extern "C" int b2v_grid_set_rectification(b2v_grid *g, const float *map_x, const float *map_y, int32_t height,
                                          int32_t width, int32_t swap_rb) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->set_rectification(map_x, map_y, height, width, swap_rb);
}

extern "C" int b2v_grid_set_frame(b2v_grid *g, const void *depth, int32_t depth_u16, float depth_scale,
                                  const uint8_t *color, int32_t height, int32_t width, int32_t filter_shadow_points,
                                  b2v_frame *out) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->set_frame(depth, depth_u16 != 0, depth_scale, color, nullptr, nullptr, height, width,
                        filter_shadow_points != 0, out);
}

extern "C" int b2v_grid_set_frame_store(b2v_grid *g, int32_t max_frames) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->set_frame_store(max_frames);
}

extern "C" int b2v_grid_frame_store_clear(b2v_grid *g) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->set_frame_store(g->frame_store.max);
}

extern "C" int b2v_grid_frame_store_last(b2v_grid *g, int32_t *slot) {
    if (!g || !slot) return B2V_ERR_INVALID_ARGUMENT;
    *slot = g->frame_store.last.empty() ? -1 : g->frame_store.last[0];
    return B2V_OK;
}

extern "C" int b2v_grid_frame_store_stats(b2v_grid *g, int64_t *frames, int64_t *bytes) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (frames) *frames = g->frame_store.count;
    if (bytes) *bytes = static_cast<int64_t>(g->frame_store.range.mapped);
    return B2V_OK;
}

extern "C" int b2v_grid_stage_stored(b2v_grid *g, int32_t slot, b2v_frame *out) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->stage_stored(slot, out);
}

extern "C" int b2v_grid_synchronize(b2v_grid *g) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->read_counters();
}

extern "C" int64_t b2v_grid_num_blocks(b2v_grid *g) {
    if (!g) return -1;
    if (g->read_counters() == B2V_ERR_CUDA) return -1;
    return g->block_count();
}

// count -> scan (-> emit into the read-out buffers, unless count_only) of the voxels the query keeps
static int64_t grid_run_query(b2v_grid *g, const GridQuery &q, bool count_only = false) {
    if (g->read_counters() == B2V_ERR_CUDA) return -1;
    const uint32_t nb = g->block_count(), nc = g->voxel_ctas(nb);
    if (g->ensure_scan(nc) != B2V_OK) return -1;
    if (nc)
        g->dispatch([&](auto l) {
            grid_query_count_kernel<decltype(l)::value><<<nc, kVox, 0, g->stream>>>(g->meta(), q, g->d_sums.get(), nb);
        });
    uint32_t total = 0;
    if (cudaGetLastError() != cudaSuccess || g->scan_total(nc, &total) != cudaSuccess) return -1;
    if (count_only) return total;
    if (g->d_out_pts.reserve(static_cast<size_t>(total) * 3) != cudaSuccess ||
        g->d_out_cols.reserve(static_cast<size_t>(total) * 3) != cudaSuccess)
        return -1;
    if (nc)
        g->dispatch([&](auto l) {
            grid_query_emit_kernel<decltype(l)::value><<<nc, kVox, 0, g->stream>>>(
                g->meta(), q, g->d_offs.get(), g->d_out_pts.get(), g->d_out_cols.get(), nb);
        });
    if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(g->stream) != cudaSuccess) return -1;
    g->last_n = total;
    return total;
}

extern "C" int64_t b2v_grid_size(b2v_grid *g) {
    if (!g) return -1;
    return grid_run_query(g, g->all_query(1), true);
}

extern "C" int64_t b2v_grid_get_voxels(b2v_grid *g, int32_t min_count) {
    if (!g) return -1;
    return grid_run_query(g, g->all_query(min_count));
}

extern "C" int64_t b2v_grid_get_voxels_in_frustum(b2v_grid *g, const float K[4], int32_t width, int32_t height,
                                                  const double Tcw[16], float depth_max, float depth_min,
                                                  int32_t min_count) {
    if (!g || !K || !Tcw || width <= 0 || height <= 0) return -1;
    return grid_run_query(g, g->frustum_query(K, width, height, Tcw, depth_max, depth_min, min_count));
}

extern "C" int64_t b2v_grid_get_voxels_in_bb(b2v_grid *g, const double bbox[6], int32_t min_count) {
    if (!g || !bbox) return -1;
    return grid_run_query(g, g->box_query(bbox, min_count));
}

extern "C" int b2v_grid_copy_voxels(b2v_grid *g, float *points, float *colors) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    const size_t n = static_cast<size_t>(g->last_n);
    if (points && n) B2V_CUDA(g, cudaMemcpy(points, g->d_out_pts.get(), n * 3 * sizeof(float), cudaMemcpyDeviceToHost));
    if (colors && n) B2V_CUDA(g, cudaMemcpy(colors, g->d_out_cols.get(), n * 3 * sizeof(float), cudaMemcpyDeviceToHost));
    return B2V_OK;
}

extern "C" int b2v_grid_remove_low_count_voxels(b2v_grid *g, int32_t min_count) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    const int rc = g->read_counters();
    if (rc == B2V_ERR_CUDA) return rc;
    const uint32_t nb = g->block_count();
    if (nb)
        g->dispatch([&](auto l) {
            grid_remove_low_count_kernel<decltype(l)::value><<<g->voxel_ctas(nb), kVox, 0, g->stream>>>(g->meta(),
                                                                                                   min_count, nb);
        });
    B2V_CUDA(g, cudaGetLastError());
    return B2V_OK;
}

extern "C" int b2v_grid_carve(b2v_grid *g, const float K[4], int32_t width, int32_t height, const double Tcw[16],
                              float depth_max, float depth_min, const float *depth, float depth_threshold) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (!K || !Tcw || !depth || width <= 0 || height <= 0) {
        g->err = "b2v_grid_carve: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    int rc = g->read_counters();
    if (rc == B2V_ERR_CUDA) return rc;
    const uint32_t nb = g->block_count();
    if (nb == 0) return B2V_OK;
    const float *d_depth = depth;
    rc = g->stage_input("b2v_grid_carve", height, width, false, &d_depth);
    if (rc != B2V_OK) return rc;
    const GridQuery q = g->frustum_query(K, width, height, Tcw, depth_max, depth_min, 1);
    g->dispatch([&](auto l) {
        grid_carve_kernel<decltype(l)::value><<<g->voxel_ctas(nb), kVox, 0, g->stream>>>(g->meta(), q, d_depth,
                                                                                       depth_threshold, nb);
    });
    B2V_CUDA(g, cudaGetLastError());
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    return B2V_OK;
}

extern "C" int64_t b2v_grid_export_blocks(b2v_grid *g, int32_t *keys4, uint32_t *blocks) {
    if (!g) return -1;
    if (g->read_counters() == B2V_ERR_CUDA) return -1;
    const uint32_t nb = g->block_count();
    cudaError_t e = cudaSuccess;
    if (nb && keys4)
        e = cudaMemcpyAsync(keys4, g->index.block_keys, nb * sizeof(int4), cudaMemcpyDeviceToHost, g->stream);
    if (nb && blocks && e == cudaSuccess)
        e = cudaMemcpyAsync(blocks, reinterpret_cast<const void *>(g->pool.va), nb * g->block_bytes(),
                            cudaMemcpyDeviceToHost, g->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(g->stream);
    if (e != cudaSuccess) {
        g->err = std::string("b2v_grid_export_blocks: ") + cudaGetErrorString(e);
        return -1;
    }
    return nb;
}

extern "C" int b2v_grid_upload_blocks(b2v_grid *g, int64_t n_blocks, const int32_t *keys4, const uint32_t *blocks) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (n_blocks < 0 || n_blocks > INT32_MAX || (n_blocks > 0 && (!keys4 || !blocks))) {
        g->err = "b2v_grid_upload_blocks: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    if (n_blocks == 0) return B2V_OK;
    B2V_CUDA(g, cudaSetDevice(g->device));
    BlockArrays a{};
    a.n_arrays = 1;
    a.dst[0] = reinterpret_cast<void *>(g->pool.va);
    a.src[0] = blocks;
    a.block_bytes[0] = static_cast<uint32_t>(g->block_bytes());
    // new storage is mapped zeroed, which is the cleared state of a voxel: nothing to fill
    const int rc = g->upload_blocks(n_blocks, keys4, a, grid_grow_storage(g),
                                    [](uint32_t, uint32_t) { return B2V_OK; });
    return rc == B2V_OK ? g->read_counters() : rc;
}
