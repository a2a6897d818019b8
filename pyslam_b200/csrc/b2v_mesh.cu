// b2v_mesh.cu — per-block marching-cubes triangle emission (sm_90a).
//
// Replaces Open3D ScalableTSDFVolume::ExtractTriangleMesh / ExtractPointCloud, called from
// pyslam/dense/volumetric_integrator_tsdf.py:239,246,260,267.  Semantics (SURVEY.md A.4):
//   - a cube is rooted at every voxel; its 8 corners may live in up to 7 neighbouring blocks;
//     a cube with any zero-weight (or missing) corner is skipped; cases 0 / 255 emit nothing
//   - a vertex lives on an edge identified by (lower-corner voxel, axis) and is shared by every
//     cube around that edge (welding): position = voxel centre + |f0| vs / (|f0| + |f1|) along axis
//   - triangles come from the classic 256-case table with winding (i, i+2, i+1)
// Deterministic three-pass structure: classify -> exclusive scan -> emit.  Output order is
// (pool block, voxel index, axis) for vertices and (pool block, voxel index, case order) for
// triangles.
#include "b2v_internal.h"
#include "b2v_scan.cuh"
#include "mc_tables.h"

namespace b2v {

__constant__ unsigned short c_halo[217];   // the 9^3 - 8^3 tile cells outside the own block: x | y << 4 | z << 8
// the marching-cubes tables live in global memory: their index differs per lane, and a divergent constant-bank read
// is serialised per distinct address, while these go through the L1
__device__ signed char g_tri_table[256][16];
__device__ unsigned char g_num_tris[256];
__device__ uchar4 g_edge_shift[12];

// cube edge e -> owner voxel offset and axis: MC_EDGE_SHIFT as compile-time constants (checked at table upload)
#define B2V_MC_EDGES(X) \
    X(0, 0, 0, 0, 0) X(1, 1, 0, 0, 1) X(2, 0, 1, 0, 0) X(3, 0, 0, 0, 1) X(4, 0, 0, 1, 0) X(5, 1, 0, 1, 1) \
    X(6, 0, 1, 1, 0) X(7, 0, 0, 1, 1) X(8, 0, 0, 0, 2) X(9, 1, 0, 0, 2) X(10, 1, 1, 0, 2) X(11, 0, 1, 0, 2)

static cudaError_t upload_tables_once() {
    static bool done = false;
    static int done_device = -1;
    int dev = 0;
    cudaGetDevice(&dev);
    if (done && done_device == dev) return cudaSuccess;
    cudaError_t e;
    if ((e = cudaMemcpyToSymbol(g_tri_table, MC_TRI_TABLE, sizeof(MC_TRI_TABLE))) != cudaSuccess) return e;
    if ((e = cudaMemcpyToSymbol(g_num_tris, MC_NUM_TRIS, sizeof(MC_NUM_TRIS))) != cudaSuccess) return e;
    static_assert(sizeof(MC_EDGE_SHIFT) == 12 * 4, "edge shift table is 12 x {dx, dy, dz, axis}");
    {   // the classify kernel carries the same table as compile-time constants, and derives the edge mask of a case
        // from its corner bits: both must agree with the generated tables
#define B2V_CHECK(e, sx, sy, sz, ax)                                                                          \
    if (MC_EDGE_SHIFT[e][0] != sx || MC_EDGE_SHIFT[e][1] != sy || MC_EDGE_SHIFT[e][2] != sz || MC_EDGE_SHIFT[e][3] != ax) \
        return cudaErrorInvalidValue;
        B2V_MC_EDGES(B2V_CHECK)
#undef B2V_CHECK
        for (unsigned cube = 0; cube < 256; ++cube) {
            const unsigned lo = cube & 15u, hi = cube >> 4;
            const unsigned em = (lo ^ ((lo >> 1) | ((lo & 1u) << 3))) | ((hi ^ ((hi >> 1) | ((hi & 1u) << 3))) << 4) | ((lo ^ hi) << 8);
            if (em != MC_EDGE_TABLE[cube]) return cudaErrorInvalidValue;
        }
    }
    if ((e = cudaMemcpyToSymbol(g_edge_shift, MC_EDGE_SHIFT, sizeof(MC_EDGE_SHIFT))) != cudaSuccess) return e;
    unsigned short halo[217];
    int nh = 0;
    for (int z = 0; z < 9; ++z)
        for (int y = 0; y < 9; ++y)
            for (int x = 0; x < 9; ++x)
                if (x == 8 || y == 8 || z == 8) halo[nh++] = static_cast<unsigned short>(x | (y << 4) | (z << 8));
    if ((e = cudaMemcpyToSymbol(c_halo, halo, sizeof(halo))) != cudaSuccess) return e;
    done = true;
    done_device = dev;
    return cudaSuccess;
}

// ---- pass 0: neighbour block indices --------------------------------------------------------

// pool index of the block at +(o&1, o>>1&1, o>>2&1) of block b, -1 if it does not exist
__device__ __forceinline__ int32_t neighbor_block(const HashTable &T, const PoolMeta &M, uint32_t b, uint32_t o) {
    if (o == 0) return static_cast<int32_t>(b);
    const int4 k = M.block_keys[b];
    const uint32_t s = table_find(T, k.x + (o & 1), k.y + ((o >> 1) & 1), k.z + ((o >> 2) & 1));
    if (s == kEmpty) return -1;
    const uint32_t w = T.entries[s].w;
    return w < M.capacity ? static_cast<int32_t>(w) : -1;
}

// pass 0: one thread per (block, neighbour) - a separate, massively parallel launch so that the two dependent memory
// hops of a table probe are not on the critical path of every classify CTA.  The eight lanes of a block also OR the
// sign summaries of the tile's blocks (PoolMeta::block_flags): a tile holds a surface crossing only if it has an
// observed negative AND an observed non-negative voxel, and the summaries are supersets of the signs present, so a
// tile whose union misses a bit is dropped without reading a voxel.  Candidate tiles go to work[2][*]; their ownership
// masks are cleared here (a vertex owner and the far end of its edge have opposite signs and lie in the owner's tile,
// so every block that receives an ownership bit is a candidate).
__global__ void __launch_bounds__(256)
mesh_neighbors_kernel(const HashTable T, const PoolMeta M, const MeshBuffers mb) {
    __shared__ uint32_t s_n, s_base;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    const bool live = i < mb.n_blocks * 8u;
    const uint32_t b = i >> 3, o = i & 7u;
    int32_t nb = -1;
    if (live) {
        nb = neighbor_block(T, M, b, o);
        mb.nbr[i] = nb;
    }
    uint32_t f = nb >= 0 ? M.block_flags[nb] : 0u;
    f |= __shfl_xor_sync(0xffffffffu, f, 1);
    f |= __shfl_xor_sync(0xffffffffu, f, 2);
    f |= __shfl_xor_sync(0xffffffffu, f, 4);
    const bool cand = live && (f & 3u) == 3u;
    uint32_t pos = 0;
    if (cand && o == 0) pos = atomicAdd(&s_n, 1u);
    __syncthreads();
    if (threadIdx.x == 0 && s_n) s_base = atomicAdd(mb.totals + kMtCandidates, s_n);
    __syncthreads();
    if (cand) {
        if (o == 0) mb.work[2 * static_cast<size_t>(mb.n_blocks) + s_base + pos] = b;
        uint4 *em = reinterpret_cast<uint4 *>(mb.edge_mask + static_cast<size_t>(b) * (kVox / 4));
#pragma unroll
        for (int k = 0; k < 4; ++k) em[o + 8 * k] = make_uint4(0u, 0u, 0u, 0u);
    }
}

// owner voxel of cube edge e rooted at local (lx,ly,lz): flat index into the per-voxel arrays + the edge's axis
__device__ __forceinline__ bool edge_owner(const int *nbr, int lx, int ly, int lz, int sx, int sy, int sz,
                                           size_t *flat) {
    const int ox = lx + sx, oy = ly + sy, oz = lz + sz;
    const int ob = nbr[(ox >> 3) | ((oy >> 3) << 1) | ((oz >> 3) << 2)];
    if (ob < 0) return false;
    *flat = static_cast<size_t>(ob) * kVox + ((ox & 7) + ((oy & 7) << 3) + ((oz & 7) << 6));
    return true;
}

// ---- pass 1a: marching-cubes case + vertex ownership (mesh) ---------------------------------

constexpr int kClsThreads = 128;   // 4 voxels per thread
constexpr int kClsCtasPerSm = 10;  // 48 registers: the persistent grid is exactly one resident wave

// Persistent over the candidate tiles.  The 9^3 tile is kept as two bit planes (row y + 9 z, bit x): "tsdf < 0" and
// "observed"; a cube's case is assembled from four row words instead of sixteen shared-memory reads.  Ownership bits
// of voxels inside the block are collected in shared memory (the four cubes around an edge all set the same bit) and
// merged into the global masks with one atomic per non-zero word; owners in a neighbouring block are set directly.
// The own voxels of the CTA's next tile are loaded while the current one is classified.

template <typename TC>
__device__ __forceinline__ void mesh_classify_kernel_body(const PoolMeta M, const MeshBuffers mb) {
    __shared__ uint32_t s_neg[81], s_val[81];
    __shared__ uint32_t s_cube[kVox / 4];
    __shared__ uint32_t s_own[kVox / 4];
    __shared__ int s_nbr[8];
    const int t = threadIdx.x, lane = t & 31;
    const int lx = t & 7, ly = (t >> 3) & 7, lz0 = t >> 6;   // voxel k of the thread: index t + 128 k, lz = lz0 + 2 k
    const uint32_t n = mb.totals[kMtCandidates];
    const uint32_t *__restrict__ cand = mb.work + 2 * static_cast<size_t>(mb.n_blocks);
    uint32_t it = blockIdx.x;
    uint32_t b = 0;
    int nbr_t = -1;
    float f0[4], w0[4];
    if (it < n) {
        b = cand[it];
        if (t < 8) nbr_t = mb.nbr[b * 8 + t];
        const float *own = M.pool + static_cast<size_t>(b) * TsdfBlock<TC>::kFloats;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            f0[k] = own[t + kClsThreads * k];
            w0[k] = own[kVox + t + kClsThreads * k];
        }
    }
    while (it < n) {
        if (t < 8) s_nbr[t] = nbr_t;
        if (t < 17) {   // the rows that hold halo cells only
            const int row = t < 9 ? 72 + t : 8 + 9 * (t - 9);
            s_neg[row] = 0;
            s_val[row] = 0;
        }
        s_own[t] = 0;
        bool neg = false, pos = false;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const unsigned bn = __ballot_sync(0xffffffffu, f0[k] < 0.0f);
            const unsigned bv = __ballot_sync(0xffffffffu, w0[k] != 0.0f);
            if (lx == 0) {   // the 8 lanes lane & 24 .. + 7 are one x row
                const int row = ly + 9 * (lz0 + 2 * k);
                s_neg[row] = (bn >> (lane & 24)) & 0xFFu;
                s_val[row] = (bv >> (lane & 24)) & 0xFFu;
            }
            neg |= w0[k] != 0.0f && f0[k] < 0.0f;
            pos |= w0[k] != 0.0f && !(f0[k] < 0.0f);
        }
        // the next tile of this CTA: its own voxels are in flight while this one is classified
        const uint32_t it_next = it + gridDim.x;
        uint32_t b_next = 0;
        if (it_next < n) {
            b_next = cand[it_next];
            if (t < 8) nbr_t = mb.nbr[b_next * 8 + t];
            const float *own = M.pool + static_cast<size_t>(b_next) * TsdfBlock<TC>::kFloats;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                f0[k] = own[t + kClsThreads * k];
                w0[k] = own[kVox + t + kClsThreads * k];
            }
        }
        __syncthreads();
        // the 217 halo cells of the 9^3 tile
        for (int i = t; i < 217; i += kClsThreads) {
            const int h = c_halo[i];
            const int x = h & 15, y = (h >> 4) & 15, z = h >> 8;
            const int pb = s_nbr[(x >> 3) | ((y >> 3) << 1) | ((z >> 3) << 2)];
            if (pb >= 0) {
                const float *blk = M.pool + static_cast<size_t>(pb) * TsdfBlock<TC>::kFloats;
                const int v = (x & 7) + ((y & 7) << 3) + ((z & 7) << 6);
                const float f = blk[v], w = blk[kVox + v];
                if (f < 0.0f) atomicOr(&s_neg[y + 9 * z], 1u << x);
                if (w != 0.0f) atomicOr(&s_val[y + 9 * z], 1u << x);
                neg |= w != 0.0f && f < 0.0f;
                pos |= w != 0.0f && !(f < 0.0f);
            }
        }
        // a tile whose observed voxels all lie on one side of the surface has no cube to emit
        const int has_neg = __syncthreads_or(neg);
        const int has_pos = __syncthreads_or(pos);
        if (has_neg && has_pos) {   // uniform over the CTA
#pragma unroll 1   // (twelve inlined edge cases per voxel: unrolled x4 the kernel needs 121 registers)
            for (int k = 0; k < 4; ++k) {
                const int lz = lz0 + 2 * k;
                const int r = ly + 9 * lz;
                // corner order {000,100,110,010,001,101,111,011} (SURVEY.md A.4 `shift`)
                const uint32_t n00 = s_neg[r] >> lx, n10 = s_neg[r + 1] >> lx;
                const uint32_t n01 = s_neg[r + 9] >> lx, n11 = s_neg[r + 10] >> lx;
                const uint32_t ok = (s_val[r] & s_val[r + 1] & s_val[r + 9] & s_val[r + 10]) >> lx;
                uint32_t cube = (n00 & 3u) | ((n10 & 2u) << 1) | ((n10 & 1u) << 3) | ((n01 & 3u) << 4) |
                                ((n11 & 2u) << 5) | ((n11 & 1u) << 7);
                if ((ok & 3u) != 3u || cube == 255u) cube = 0;   // an unobserved corner, or nothing to emit
                reinterpret_cast<uint8_t *>(s_cube)[t + kClsThreads * k] = static_cast<uint8_t>(cube);
                if (cube) {
                    // edges with a sign change: e0..3 = corners i, i+1 of the bottom face, e4..7 the top face,
                    // e8..11 the verticals (the classic edge table, tests/test_mc_tables.py)
                    const uint32_t lo = cube & 15u, hi = cube >> 4;
                    const uint32_t em = (lo ^ ((lo >> 1) | ((lo & 1u) << 3))) | ((hi ^ ((hi >> 1) | ((hi & 1u) << 3))) << 4) |
                                        ((lo ^ hi) << 8);
#define B2V_OWN(e, sx, sy, sz, ax)                                                                                   \
    if (em & (1u << e)) {                                                                                            \
        const int ox = lx + sx, oy = ly + sy, oz = lz + sz;                                                          \
        const int ov = (ox & 7) + ((oy & 7) << 3) + ((oz & 7) << 6);                                                 \
        if ((sx | sy | sz) && ((ox | oy | oz) & 8)) {                                                                \
            const int ob = s_nbr[(ox >> 3) | ((oy >> 3) << 1) | ((oz >> 3) << 2)];                                   \
            if (ob >= 0)                                                                                             \
                atomicOr(mb.edge_mask + static_cast<size_t>(ob) * (kVox / 4) + (ov >> 2), (1u << ax) << ((ov & 3) * 8)); \
        } else {                                                                                                     \
            atomicOr(&s_own[ov >> 2], (1u << ax) << ((ov & 3) * 8));                                                 \
        }                                                                                                            \
    }
                    B2V_MC_EDGES(B2V_OWN)
#undef B2V_OWN
                }
            }
            __syncthreads();
            reinterpret_cast<uint32_t *>(mb.cube)[static_cast<size_t>(b) * (kVox / 4) + t] = s_cube[t];
            // other tiles set bits of this block's halo-side voxels concurrently: merge, do not store
            const uint32_t own_bits = s_own[t];
            if (own_bits) atomicOr(mb.edge_mask + static_cast<size_t>(b) * (kVox / 4) + t, own_bits);
            if (t == 0) mb.work[3 * static_cast<size_t>(mb.n_blocks) + atomicAdd(mb.totals + kMtTiles, 1u)] = b;
        }
        __syncthreads();   // the tile's shared arrays are rewritten by the next iteration
        it = it_next;
        b = b_next;
    }
}

__global__ void __launch_bounds__(kClsThreads, kClsCtasPerSm)
mesh_classify_kernel(const PoolMeta M, const MeshBuffers mb) {
    mesh_classify_kernel_body<float>(M, mb);
}
// the float64-colour instantiation
__global__ void __launch_bounds__(kClsThreads, kClsCtasPerSm)
mesh_classify_kernel_c64(const PoolMeta M, const MeshBuffers mb) {
    mesh_classify_kernel_body<double>(M, mb);
}

// ---- pass 1b: zero-crossing masks (point cloud) ---------------------------------------------

template <typename TC>
__device__ __forceinline__ void point_masks_kernel_body(const PoolMeta M, const MeshBuffers mb) {
    __shared__ int s_nbr[8];
    __shared__ uint8_t s_m[kVox];
    const int t = threadIdx.x;
    const uint32_t n = mb.totals[kMtCandidates];
    const uint32_t *__restrict__ cand = mb.work + 2 * static_cast<size_t>(mb.n_blocks);
    for (uint32_t it = blockIdx.x; it < n; it += gridDim.x) {
        const uint32_t b = cand[it];
        if (t < 8) s_nbr[t] = mb.nbr[b * 8 + t];
        __syncthreads();
        const float *blk = M.pool + static_cast<size_t>(b) * TsdfBlock<TC>::kFloats;
        const float f0 = blk[t], w0 = blk[kVox + t];
        const int l[3] = {t & 7, (t >> 3) & 7, t >> 6};
        unsigned m = 0;
        if (w0 != 0.0f && f0 < 0.98f && f0 >= -0.98f) {
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                int q[3] = {l[0], l[1], l[2]};
                q[a] += 1;
                const int pb = s_nbr[(q[0] >> 3) | ((q[1] >> 3) << 1) | ((q[2] >> 3) << 2)];
                if (pb < 0) continue;
                const float *nb = M.pool + static_cast<size_t>(pb) * TsdfBlock<TC>::kFloats;
                const int v = (q[0] & 7) + ((q[1] & 7) << 3) + ((q[2] & 7) << 6);
                const float f1 = nb[v], w1 = nb[kVox + v];
                if (w1 != 0.0f && f1 < 0.98f && f1 >= -0.98f && f0 * f1 < 0.0f) m |= 1u << a;
            }
        }
        s_m[t] = static_cast<uint8_t>(m);
        const int any = __syncthreads_or(m != 0);
        if (any) {
            if (t < kVox / 4) {
                mb.edge_mask[static_cast<size_t>(b) * (kVox / 4) + t] = reinterpret_cast<const uint32_t *>(s_m)[t];
                reinterpret_cast<uint32_t *>(mb.cube)[static_cast<size_t>(b) * (kVox / 4) + t] = 0;
            }
            if (t == 0) mb.work[3 * static_cast<size_t>(mb.n_blocks) + atomicAdd(mb.totals + kMtTiles, 1u)] = b;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kVox)
point_masks_kernel(const PoolMeta M, const MeshBuffers mb) {
    point_masks_kernel_body<float>(M, mb);
}
// the float64-colour instantiation
__global__ void __launch_bounds__(kVox)
point_masks_kernel_c64(const PoolMeta M, const MeshBuffers mb) {
    point_masks_kernel_body<double>(M, mb);
}

// ---- pass 2: per-block sums and their exclusive scans ---------------------------------------

// persistent over the tiles pass 1 kept; the sums of every other block stay at the launcher's zero
__global__ void __launch_bounds__(128, 16)
mesh_block_sums_kernel(const MeshBuffers mb) {
    __shared__ uint32_t s_v[4], s_t[4];
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    const uint32_t n = mb.totals[kMtTiles];
    const uint32_t *__restrict__ tiles = mb.work + 3 * static_cast<size_t>(mb.n_blocks);
    uint32_t b = 0, m4 = 0, c4 = 0;
    if (blockIdx.x < n) {
        b = tiles[blockIdx.x];
        m4 = mb.edge_mask[static_cast<size_t>(b) * 128 + t];
        c4 = reinterpret_cast<const uint32_t *>(mb.cube)[static_cast<size_t>(b) * 128 + t];
    }
    for (uint32_t it = blockIdx.x; it < n; it += gridDim.x) {
        // the next tile's words are in flight during this one
        uint32_t b_next = 0, m4_next = 0, c4_next = 0;
        if (it + gridDim.x < n) {
            b_next = tiles[it + gridDim.x];
            m4_next = mb.edge_mask[static_cast<size_t>(b_next) * 128 + t];
            c4_next = reinterpret_cast<const uint32_t *>(mb.cube)[static_cast<size_t>(b_next) * 128 + t];
        }
        uint32_t pv[4], pt[4];   // vertices / triangles of the thread's four voxels
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            pv[k] = __popc((m4 >> (8 * k)) & 7u);
            const uint32_t cube = (c4 >> (8 * k)) & 0xFFu;
            pt[k] = cube ? g_num_tris[cube] : 0u;
        }
        const uint32_t nv = pv[0] + pv[1] + pv[2] + pv[3], nt = pt[0] + pt[1] + pt[2] + pt[3];
        // exclusive scan over the 128 threads (vertices in the low half, triangles in the high half: <= 1536 / 2560)
        uint32_t x = nv | (nt << 16);
        const uint32_t mine = x;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
            if (lane >= d) x += y;
        }
        if (lane == 31) {
            s_v[wid] = x & 0xFFFFu;
            s_t[wid] = x >> 16;
        }
        __syncthreads();
        uint32_t ov = 0, ot = 0;
        for (int w = 0; w < wid; ++w) {
            ov += s_v[w];
            ot += s_t[w];
        }
        const uint32_t sv = s_v[0] + s_v[1] + s_v[2] + s_v[3], st = s_t[0] + s_t[1] + s_t[2] + s_t[3];
        if (sv | st) {  // per-voxel position inside the block: the emit kernels need no scan of their own
            uint32_t bv = ov + ((x - mine) & 0xFFFFu), bt = ot + ((x - mine) >> 16);
            uint4 out;
            uint32_t *o = &out.x;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                o[k] = bv | (bt << 16);
                bv += pv[k];
                bt += pt[k];
            }
            reinterpret_cast<uint4 *>(mb.local)[static_cast<size_t>(b) * 128 + t] = out;
        }
        if (t == 0) {
            mb.sums[b] = sv;
            mb.sums[mb.n_blocks + b] = st;
            // the emit kernels run over the blocks that have output only (list order does not matter: positions
            // come from the scan of the sums)
            if (sv) mb.work[atomicAdd(mb.totals + kMtVertexBlocks, 1u)] = b;
            if (st) mb.work[mb.n_blocks + atomicAdd(mb.totals + kMtTriangleBlocks, 1u)] = b;
        }
        __syncthreads();   // s_v / s_t are rewritten by the next iteration
        b = b_next;
        m4 = m4_next;
        c4 = c4_next;
    }
}

// ---- pass 3a: vertices -----------------------------------------------------------------------

// points = false: ScalableTSDFVolume::ExtractTriangleMesh vertex / colour formulas (float64):
//     pt = vl/2 + vl * e;  pt[a] += |f0| vl / (|f0| + |f1|);  colour (|f1| c0/255 + |f0| c1/255) / (|f0| + |f1|)
// points = true: ExtractPointCloud: p0 = (vl/2 + vl * x_in_unit) + unit * L, p1 = p0 + vl on the axis,
//     p = (p0 r1 + p1 r0) / (r0 + r1) with float32 r0 = |f0|, r1 = |f1| (their sum in float32), colour
//     ((c0 r1 + c1 r0) / (r0 + r1)) / 255 in float32, widened.  With float64 colour (TC = double) the colour terms
//     are float64: c r widens r, the sum r0 + r1 is widened after its float32 add, and 255 is widened.
// One CTA per block with output.  The block's vertices are first listed in shared memory at the positions pass 2 gave
// them, then every lane emits one listed vertex: no lane idles on a voxel without output, stores are consecutive.
constexpr int kEmitThreads = 128;

template <typename TC, bool kPoints>
__device__ __forceinline__ void mesh_vertices_kernel_body(const PoolMeta M, const MeshBuffers mb, const double vl,
                                                          const int unit_shift) {
    __shared__ unsigned short s_list[3 * kVox];   // voxel << 2 | axis
    const uint32_t b = mb.work[blockIdx.x];       // blocks with at least one vertex
    const int t = threadIdx.x;
    {
        const uint32_t m4 = mb.edge_mask[static_cast<size_t>(b) * (kVox / 4) + t];
        const uint4 lc = reinterpret_cast<const uint4 *>(mb.local)[static_cast<size_t>(b) * (kVox / 4) + t];
        const uint32_t l4[4] = {lc.x, lc.y, lc.z, lc.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const unsigned m = (m4 >> (8 * k)) & 7u;
            uint32_t pos = l4[k] & 0xFFFFu;
#pragma unroll
            for (int a = 0; a < 3; ++a)
                if ((m >> a) & 1u) s_list[pos++] = static_cast<unsigned short>(((4 * t + k) << 2) | a);
        }
    }
    __syncthreads();
    const uint32_t nv = mb.sums[b];
    const uint32_t vbase = mb.offs[b];
    const int *nbr = mb.nbr + static_cast<size_t>(b) * 8;
    const float *blk = M.pool + static_cast<size_t>(b) * TsdfBlock<TC>::kFloats;
    const int4 key = M.block_keys[b];
    const double half = __dmul_rn(vl, 0.5);
    for (uint32_t i = t; i < nv; i += kEmitThreads) {
        const int en = s_list[i];
        const int v0 = en >> 2, a = en & 3;
        const float r0 = fabsf(blk[v0]);
        const TC c0[3] = {TsdfBlock<TC>::color_at(blk, 0, v0), TsdfBlock<TC>::color_at(blk, 1, v0),
                          TsdfBlock<TC>::color_at(blk, 2, v0)};
        const int l[3] = {v0 & 7, (v0 >> 3) & 7, v0 >> 6};
        const int g[3] = {key.x * kB + l[0], key.y * kB + l[1], key.z * kB + l[2]};
        double p[3];
        if (kPoints) {
            const int kk[3] = {key.x, key.y, key.z};
            const double L = __dmul_rn(vl, static_cast<double>(kB << unit_shift));  // volume_unit_length_
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const int u = kk[c] >> unit_shift;
                const int x = (kk[c] - (u << unit_shift)) * kB + l[c];
                p[c] = __dadd_rn(__dadd_rn(half, __dmul_rn(vl, static_cast<double>(x))), __dmul_rn(static_cast<double>(u), L));
            }
        } else {
#pragma unroll
            for (int c = 0; c < 3; ++c) p[c] = __dadd_rn(half, __dmul_rn(vl, static_cast<double>(g[c])));
        }
        const int q[3] = {l[0] + (a == 0), l[1] + (a == 1), l[2] + (a == 2)};
        const int pb = nbr[(q[0] >> 3) | ((q[1] >> 3) << 1) | ((q[2] >> 3) << 2)];
        const float *nb = M.pool + static_cast<size_t>(pb) * TsdfBlock<TC>::kFloats;
        const int v1 = (q[0] & 7) + ((q[1] & 7) << 3) + ((q[2] & 7) << 6);
        const float r1 = fabsf(nb[v1]);
        const double pa = a == 0 ? p[0] : (a == 1 ? p[1] : p[2]);
        double pn, col[3];
        if (kPoints) {
            const float rs = __fadd_rn(r0, r1);
            const double p1 = __dadd_rn(pa, vl);
            pn = __ddiv_rn(__dadd_rn(__dmul_rn(pa, static_cast<double>(r1)), __dmul_rn(p1, static_cast<double>(r0))),
                           static_cast<double>(rs));
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const TC c1 = TsdfBlock<TC>::color_at(nb, k, v1);
                if constexpr (std::is_same<TC, float>::value) {
                    const float num = __fadd_rn(__fmul_rn(c0[k], r1), __fmul_rn(c1, r0));
                    col[k] = static_cast<double>(__fdiv_rn(__fdiv_rn(num, rs), 255.0f));
                } else {
                    const double num = __dadd_rn(__dmul_rn(c0[k], static_cast<double>(r1)),
                                                 __dmul_rn(c1, static_cast<double>(r0)));
                    col[k] = __ddiv_rn(__ddiv_rn(num, static_cast<double>(rs)), 255.0);
                }
            }
        } else {
            const double f0 = static_cast<double>(r0), f1 = static_cast<double>(r1);
            const double fs = __dadd_rn(f0, f1);
            pn = __dadd_rn(pa, __ddiv_rn(__dmul_rn(f0, vl), fs));
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const double d0 = __ddiv_rn(static_cast<double>(c0[k]), 255.0);
                const double d1 = __ddiv_rn(static_cast<double>(TsdfBlock<TC>::color_at(nb, k, v1)), 255.0);
                col[k] = __ddiv_rn(__dadd_rn(__dmul_rn(f1, d0), __dmul_rn(f0, d1)), fs);
            }
        }
        if (a == 0) p[0] = pn;
        else if (a == 1) p[1] = pn;
        else p[2] = pn;
        const size_t vid = static_cast<size_t>(vbase) + i;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            mb.vertices[3 * vid + k] = p[k];
            mb.colors[3 * vid + k] = col[k];
        }
        reinterpret_cast<int4 *>(mb.edge_ids)[vid] = make_int4(g[0], g[1], g[2], a);
    }
}

template <bool kPoints>
__global__ void __launch_bounds__(kEmitThreads)
mesh_vertices_kernel(const PoolMeta M, const MeshBuffers mb, const double vl, const int unit_shift) {
    mesh_vertices_kernel_body<float, kPoints>(M, mb, vl, unit_shift);
}
// the float64-colour instantiation
template <bool kPoints>
__global__ void __launch_bounds__(kEmitThreads)
mesh_vertices_kernel_c64(const PoolMeta M, const MeshBuffers mb, const double vl, const int unit_shift) {
    mesh_vertices_kernel_body<double, kPoints>(M, mb, vl, unit_shift);
}

// ---- pass 3b: triangles ----------------------------------------------------------------------

// One CTA per block with output; the block's triangles are listed in shared memory first, then every lane emits one.
__global__ void __launch_bounds__(kEmitThreads)
mesh_triangles_kernel(const MeshBuffers mb) {
    __shared__ unsigned short s_list[5 * kVox];   // voxel << 3 | triangle of its cube
    __shared__ uint32_t s_cube[kVox / 4];
    const uint32_t b = mb.work[mb.n_blocks + blockIdx.x];  // blocks with at least one triangle
    const int t = threadIdx.x;
    {
        const uint32_t c4 = reinterpret_cast<const uint32_t *>(mb.cube)[static_cast<size_t>(b) * (kVox / 4) + t];
        s_cube[t] = c4;
        const uint4 lc = reinterpret_cast<const uint4 *>(mb.local)[static_cast<size_t>(b) * (kVox / 4) + t];
        const uint32_t l4[4] = {lc.x, lc.y, lc.z, lc.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t cube = (c4 >> (8 * k)) & 0xFFu;
            if (cube == 0) continue;
            const uint32_t nt = g_num_tris[cube];
            const uint32_t pos = l4[k] >> 16;
            for (uint32_t j = 0; j < nt; ++j) s_list[pos + j] = static_cast<unsigned short>(((4 * t + k) << 3) | j);
        }
    }
    __syncthreads();
    const uint32_t nt = mb.sums[mb.n_blocks + b];
    const uint32_t tbase = mb.offs[mb.n_blocks + b];
    const int *nbr = mb.nbr + static_cast<size_t>(b) * 8;
    for (uint32_t i = t; i < nt; i += kEmitThreads) {
        const int en = s_list[i];
        const int v0 = en >> 3, j = en & 7;
        const int cube = (s_cube[v0 >> 2] >> ((v0 & 3) * 8)) & 0xFF;
        const int lx = v0 & 7, ly = (v0 >> 3) & 7, lz = v0 >> 6;
        int vid[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int e = g_tri_table[cube][3 * j + c];
            const uchar4 sh = g_edge_shift[e];
            size_t flat;
            vid[c] = -1;
            if (edge_owner(nbr, lx, ly, lz, sh.x, sh.y, sh.z, &flat)) {
                const unsigned m = (mb.edge_mask[flat >> 2] >> ((flat & 3) * 8)) & 7u;
                vid[c] = static_cast<int>(mb.offs[flat >> 9] + (mb.local[flat] & 0xFFFFu) + __popc(m & ((1u << sh.w) - 1u)));
            }
        }
        int32_t *tri = mb.triangles + 3 * (static_cast<size_t>(tbase) + i);
        tri[0] = vid[0];
        tri[1] = vid[2];  // winding (i, i+2, i+1)
        tri[2] = vid[1];
    }
}

// ---- launchers -------------------------------------------------------------------------------

// pass 0 for both extractions: counters, the sums of the blocks no later pass visits, neighbours + candidate tiles
static cudaError_t launch_mesh_front(const HashTable &table, const PoolMeta &meta, const MeshBuffers &mb,
                                     cudaStream_t stream) {
    cudaError_t e = upload_tables_once();
    if (e != cudaSuccess) return e;
    e = cudaMemsetAsync(mb.totals, 0, kNumMeshTotals * sizeof(uint32_t), stream);
    if (e != cudaSuccess || mb.n_blocks == 0) return e;
    e = cudaMemsetAsync(mb.sums, 0, 2 * static_cast<size_t>(mb.n_blocks) * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    mesh_neighbors_kernel<<<(mb.n_blocks * 8u + 255u) / 256u, 256, 0, stream>>>(table, meta, mb);
    return cudaGetLastError();
}

cudaError_t launch_mesh_classify(const HashTable &table, const PoolMeta &meta, const MeshBuffers &mb, int sms,
                                 cudaStream_t stream, bool color_f64) {
    cudaError_t e = launch_mesh_front(table, meta, mb, stream);
    if (e != cudaSuccess || mb.n_blocks == 0) return e;
    const unsigned grid = min(mb.n_blocks, static_cast<unsigned>(sms) * kClsCtasPerSm);
    (color_f64 ? mesh_classify_kernel_c64 : mesh_classify_kernel)<<<grid, kClsThreads, 0, stream>>>(meta, mb);
    return cudaGetLastError();
}

cudaError_t launch_point_masks(const HashTable &table, const PoolMeta &meta, const MeshBuffers &mb, int sms,
                               cudaStream_t stream, bool color_f64) {
    cudaError_t e = launch_mesh_front(table, meta, mb, stream);
    if (e != cudaSuccess || mb.n_blocks == 0) return e;
    const unsigned grid = min(mb.n_blocks, static_cast<unsigned>(sms) * (2048u / kVox));
    (color_f64 ? point_masks_kernel_c64 : point_masks_kernel)<<<grid, kVox, 0, stream>>>(meta, mb);
    return cudaGetLastError();
}

cudaError_t launch_mesh_scan(const MeshBuffers &mb, int sms, cudaStream_t stream) {
    if (mb.n_blocks == 0) return cudaSuccess;
    const unsigned grid = min(mb.n_blocks, static_cast<unsigned>(sms) * 16u);
    mesh_block_sums_kernel<<<grid, 128, 0, stream>>>(mb);
    const dim3 chunks((mb.n_blocks + 1023u) / 1024u, 2);
    scan_reduce_kernel<<<chunks, 1024, 0, stream>>>(mb.sums, mb.partials, mb.n_blocks);
    scan_apply_kernel<<<chunks, 1024, 0, stream>>>(mb.sums, mb.offs, mb.partials, mb.totals, mb.n_blocks);
    return cudaGetLastError();
}

cudaError_t launch_mesh_vertices(const PoolMeta &meta, const MeshBuffers &mb, double voxel_length, int unit_shift,
                                 bool points, uint32_t work_blocks, cudaStream_t stream, bool color_f64) {
    if (work_blocks == 0) return cudaSuccess;
    const auto kernel = points ? (color_f64 ? mesh_vertices_kernel_c64<true> : mesh_vertices_kernel<true>)
                               : (color_f64 ? mesh_vertices_kernel_c64<false> : mesh_vertices_kernel<false>);
    kernel<<<work_blocks, kEmitThreads, 0, stream>>>(meta, mb, voxel_length, unit_shift);
    return cudaGetLastError();
}

cudaError_t launch_mesh_triangles(const MeshBuffers &mb, uint32_t work_blocks, cudaStream_t stream) {
    if (work_blocks == 0) return cudaSuccess;
    mesh_triangles_kernel<<<work_blocks, kEmitThreads, 0, stream>>>(mb);
    return cudaGetLastError();
}

}  // namespace b2v
