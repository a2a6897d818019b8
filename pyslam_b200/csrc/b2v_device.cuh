// b2v_device.cuh — device-side building blocks shared by the sm_90a kernels.
//
// Key arithmetic follows pySLAM's cpp/volumetric bit for bit:
//   voxel coord  v = (int32)floor(x * inv_voxel_size)            voxel_hashing.h:69-75
//   block coord  b = floor_div(v, 8), local l = v - 8 b          voxel_hashing.h:139-161
//   voxel index  lx + 8 ly + 64 lz                                voxel_block.h:67-70
//   BlockKeyHash h1 ^ (h2 << 1) ^ (h3 << 2) on sign-extended u64  voxel_hashing.h:106-113
// The open-addressing table probes with a separate strong mix (the reference hash is reported
// and used for sharding, but clusters far too much to probe with).
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

namespace b2v {

constexpr int kB = 8;              // block side
constexpr int kLog2B = 3;
constexpr int kVox = 512;          // voxels per block
constexpr int kPlanes = 5;         // tsdf, weight, r, g, b
constexpr int kBlockFloats = kVox * kPlanes;

constexpr uint32_t kEmpty = 0xFFFFFFFFu;    // entry.w of an empty slot (whole entry is 0xFF..)
constexpr uint32_t kPending = 0xFFFFFFFEu;  // inserted in this launch, pool index not yet assigned
constexpr uint32_t kNoBlock = 0xFFFFFFFDu;  // pool overflowed: key present but no storage

// Open-addressing table: entry = {key.x, key.y, key.z, pool index}.  16-byte entries are read
// with one LDG.128 and inserted with one 128-bit CAS (ATOMG.E.CAS.128 on sm_90a).
struct HashTable {
    uint4 *entries;
    uint32_t mask;    // capacity - 1 (capacity is a power of two)
};

__host__ __device__ __forceinline__ uint64_t block_key_hash(int x, int y, int z) {
    const uint64_t h1 = static_cast<uint64_t>(static_cast<int64_t>(x));
    const uint64_t h2 = static_cast<uint64_t>(static_cast<int64_t>(y));
    const uint64_t h3 = static_cast<uint64_t>(static_cast<int64_t>(z));
    return h1 ^ (h2 << 1) ^ (h3 << 2);
}

// owner rank of a block: BlockKeyHash % n (SURVEY.md 8e).  64-bit division is emulated (~60 instructions); the
// allocate kernels test ~1000 candidate keys per tile, so a power-of-two rank count takes the mask instead
__host__ __device__ __forceinline__ uint32_t block_owner(int x, int y, int z, uint32_t n) {
    const uint64_t h = block_key_hash(x, y, z);
    return (n & (n - 1u)) == 0u ? static_cast<uint32_t>(h) & (n - 1u) : static_cast<uint32_t>(h % static_cast<uint64_t>(n));
}

__host__ __device__ __forceinline__ uint32_t mix32(uint32_t h) {
    h ^= h >> 16;
    h *= 0x85ebca6bu;
    h ^= h >> 13;
    h *= 0xc2b2ae35u;
    h ^= h >> 16;
    return h;
}

__host__ __device__ __forceinline__ uint32_t slot_hash(int x, int y, int z) {
    uint32_t h = mix32(static_cast<uint32_t>(x) * 0x9E3779B1u + 0x7F4A7C15u);
    h = mix32(h ^ (static_cast<uint32_t>(y) * 0x85EBCA77u));
    h = mix32(h ^ (static_cast<uint32_t>(z) * 0xC2B2AE3Du));
    return h;
}

// floor division by the block side (arithmetic shift == floor_div for a power of two)
__host__ __device__ __forceinline__ int block_coord(int v) { return v >> kLog2B; }
__host__ __device__ __forceinline__ int local_coord(int v) { return v & (kB - 1); }

// ---- the sparse block grids (b2v_grid.cu, b2v_semantic.cu): block side B = 1 << L, L in [0, kMaxGridLog2B] ----
// The same key rules with B a compile-time power of two: block key floor_div(v, B) = v >> L, local key v - B b =
// v & (B - 1), voxel index lx + B ly + B^2 lz (voxel_hashing.h:139-161, voxel_block.h:67-70).  The TSDF volume keeps
// kB above.  At L = 3 each of these is the expression of the helpers above.
constexpr int kMaxGridLog2B = 4;   // B = 16
template <int L> struct GridBlock {
    static constexpr int kSide = 1 << L;
    static constexpr int kVox = 1 << (3 * L);   // voxels per block
};
template <int L> __host__ __device__ __forceinline__ int grid_block_coord(int v) { return v >> L; }
template <int L> __host__ __device__ __forceinline__ int grid_local_coord(int v) { return v & ((1 << L) - 1); }
template <int L> __host__ __device__ __forceinline__ int grid_local_index(int vx, int vy, int vz) {
    return grid_local_coord<L>(vx) + (grid_local_coord<L>(vy) << L) + (grid_local_coord<L>(vz) << (2 * L));
}

#ifdef __CUDACC__
// Voxel-range CTA mapping of the grids' per-voxel passes: CTA c covers the 512 consecutive voxels [512 c, 512 c + 512)
// of the pool, where voxel id = pool index * B^3 + local index.  *b: the pool index, *t: the local index of this
// thread's voxel.  B = 8: one CTA per block (b = blockIdx.x, t = threadIdx.x); B = 16: eight CTAs per block; B < 8: a
// CTA spans 512 / B^3 blocks, and the last CTA may reach past the blocks in use (callers bound b).
template <int L> __device__ __forceinline__ void cta_voxel(uint32_t *b, int *t) {
    if constexpr (3 * L >= 9) {
        *b = blockIdx.x >> (3 * L - 9);
        *t = static_cast<int>(((blockIdx.x & ((1u << (3 * L - 9)) - 1u)) << 9) + threadIdx.x);
    } else {
        *b = (blockIdx.x << (9 - 3 * L)) + (threadIdx.x >> (3 * L));
        *t = static_cast<int>(threadIdx.x & ((1u << (3 * L)) - 1u));
    }
}
#endif

#ifdef __CUDACC__

// (int32)floorf(x * inv_vs) with the multiply rounded on its own (never contracted)
__device__ __forceinline__ int voxel_coord(float x, float inv_vs) {
    return __float2int_rd(__fmul_rn(x, inv_vs));
}

__device__ __forceinline__ uint4 ld_entry(const uint4 *p) {
    return __ldcg(p);  // L2: entries are written by other SMs during the same launch
}

__device__ __forceinline__ uint4 cas_entry(uint4 *addr, uint4 cmp, uint4 val) {
    const uint64_t clo = static_cast<uint64_t>(cmp.x) | (static_cast<uint64_t>(cmp.y) << 32);
    const uint64_t chi = static_cast<uint64_t>(cmp.z) | (static_cast<uint64_t>(cmp.w) << 32);
    const uint64_t vlo = static_cast<uint64_t>(val.x) | (static_cast<uint64_t>(val.y) << 32);
    const uint64_t vhi = static_cast<uint64_t>(val.z) | (static_cast<uint64_t>(val.w) << 32);
    uint64_t olo, ohi;
    asm volatile(
        "{\n\t.reg .b128 c, v, o;\n\t"
        "mov.b128 c, {%2, %3};\n\t"
        "mov.b128 v, {%4, %5};\n\t"
        "atom.global.relaxed.gpu.cas.b128 o, [%6], c, v;\n\t"
        "mov.b128 {%0, %1}, o;\n\t}"
        : "=l"(olo), "=l"(ohi)
        : "l"(clo), "l"(chi), "l"(vlo), "l"(vhi), "l"(addr)
        : "memory");
    return make_uint4(static_cast<uint32_t>(olo), static_cast<uint32_t>(olo >> 32),
                      static_cast<uint32_t>(ohi), static_cast<uint32_t>(ohi >> 32));
}

// Find the slot of a key; kEmpty if absent.
__device__ __forceinline__ uint32_t table_find(const HashTable &t, int x, int y, int z) {
    uint32_t s = slot_hash(x, y, z) & t.mask;
    for (uint32_t probe = 0; probe <= t.mask; ++probe) {
        const uint4 e = ld_entry(t.entries + s);
        if (e.w == kEmpty) return kEmpty;
        if (static_cast<int>(e.x) == x && static_cast<int>(e.y) == y && static_cast<int>(e.z) == z)
            return s;
        s = (s + 1) & t.mask;
    }
    return kEmpty;
}

// Find-or-insert.  A fresh entry carries kPending until its pool index is assigned.
// Returns the slot (kEmpty when the table is full); *is_new says whether this call inserted it.
__device__ __forceinline__ uint32_t table_insert(const HashTable &t, int x, int y, int z,
                                                 bool *is_new) {
    const uint4 empty = make_uint4(kEmpty, kEmpty, kEmpty, kEmpty);
    const uint4 fresh = make_uint4(static_cast<uint32_t>(x), static_cast<uint32_t>(y),
                                   static_cast<uint32_t>(z), kPending);
    uint32_t s = slot_hash(x, y, z) & t.mask;
    *is_new = false;
    for (uint32_t probe = 0; probe <= t.mask; ++probe) {
        uint4 e = ld_entry(t.entries + s);
        if (e.w == kEmpty) {
            e = cas_entry(t.entries + s, empty, fresh);
            if (e.w == kEmpty) {
                *is_new = true;
                return s;
            }
        }
        if (static_cast<int>(e.x) == x && static_cast<int>(e.y) == y && static_cast<int>(e.z) == z)
            return s;
        s = (s + 1) & t.mask;
    }
    return kEmpty;
}

#endif  // __CUDACC__

}  // namespace b2v
