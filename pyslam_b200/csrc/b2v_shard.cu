// b2v_shard.cu — face-halo exchange of a hash-sharded volume (sm_90a): each rank meshes its own blocks.
//
// A cube rooted in block B reads B and its seven +x/+y/+z neighbours B+o, o in {1..7} (bit 0 = x).  From B+o it needs
// only the voxels whose local coordinate is 0 on every axis where o is 1: a 64-voxel face, an 8-voxel line or one
// corner voxel.  A rank therefore sends, for each owned block H and each rank r != own owning some H-o, ONE record:
// the header {key.x, key.y, key.z, mask} (bit o-1 of the 7-bit mask: r owns H-o) and the union of the needed voxels
// in increasing voxel index (at most 169 voxels of HaloVoxel<TC>::kWords float32 words each: tsdf, weight, r, g, b,
// the colour as float32 or, in a float64-colour volume, as float64 with kHaloColorF64 set in the mask).  Records are grouped
// by destination, and inside a destination ordered by the sender's pool index (count -> scan -> emit).
//
// The receiver imports its own blocks (pool indices [0, n_owned)) and the records as zero-filled halo blocks after
// them into an extraction scratch, and runs the unchanged marching-cubes kernels.  Every cube rooted in a halo block
// has a corner with all local coordinates >= 1, outside every imported plane, so it has weight 0 and emits nothing:
// the ranks' triangles partition the single-volume mesh.  Vertices of seam edges may be emitted on several ranks
// (same voxel values, same arithmetic, same float64 result); the weld below keeps one per edge id.
#include "b2v_internal.h"
#include "b2v_scan.cuh"

namespace b2v {

__device__ unsigned short g_halo_vox[128][kHaloMaxVoxels];   // voxels of each mask's union, increasing index
__device__ unsigned char g_halo_cnt[128];

static void halo_shape(uint32_t mask, unsigned short *vox, uint32_t *count) {
    uint32_t n = 0;
    for (int v = 0; v < kVox; ++v) {
        const int x = v & 7, y = (v >> 3) & 7, z = v >> 6;
        bool need = false;
        for (int o = 1; o < 8; ++o)
            if (((mask >> (o - 1)) & 1u) && (!(o & 1) || x == 0) && (!(o & 2) || y == 0) && (!(o & 4) || z == 0))
                need = true;
        if (need) vox[n++] = static_cast<unsigned short>(v);
    }
    *count = n;
}

static cudaError_t upload_halo_tables_once() {
    static int done_device = -1;
    int dev = 0;
    cudaGetDevice(&dev);
    if (done_device == dev) return cudaSuccess;
    static unsigned short vox[128][kHaloMaxVoxels];
    static unsigned char cnt[128];
    for (uint32_t m = 0; m < 128; ++m) {
        uint32_t n = 0;
        halo_shape(m, vox[m], &n);
        cnt[m] = static_cast<unsigned char>(n);
    }
    cudaError_t e = cudaMemcpyToSymbol(g_halo_vox, vox, sizeof(vox));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_halo_cnt, cnt, sizeof(cnt));
    if (e == cudaSuccess) done_device = dev;
    return e;
}

// owners of H - o for o = 1..7; bit o-1 of the returned masks[k] belongs to the k-th distinct foreign owner dest[k]
// (in order of first appearance over o); returns the number of distinct foreign owners
__device__ __forceinline__ int halo_dests(const int4 k, const uint32_t world, uint32_t dest[7], uint32_t masks[7]) {
    const uint32_t own = block_owner(k.x, k.y, k.z, world);
    int n = 0;
#pragma unroll
    for (int o = 1; o < 8; ++o) {
        const uint32_t r = block_owner(k.x - (o & 1), k.y - ((o >> 1) & 1), k.z - ((o >> 2) & 1), world);
        if (r == own) continue;
        int j = 0;
        while (j < n && dest[j] != r) ++j;
        if (j == n) {
            dest[n] = r;
            masks[n] = 0;
            ++n;
        }
        masks[j] |= 1u << (o - 1);
    }
    return n;
}

// counts[r * nb + b] = 1 if block b sends a record to rank r; counts[world * nb + r * nb + b] = its voxel count
__global__ void halo_count_kernel(const int4 *__restrict__ keys, uint32_t nb, uint32_t world,
                                  uint32_t *__restrict__ counts) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    uint32_t dest[7], masks[7];
    const int n = halo_dests(keys[b], world, dest, masks);
    const size_t plane = static_cast<size_t>(world) * nb;
    for (int j = 0; j < n; ++j) {
        const size_t i = static_cast<size_t>(dest[j]) * nb + b;
        counts[i] = 1u;
        counts[plane + i] = g_halo_cnt[masks[j]];
    }
}

// per-destination starts of the records / payload voxels: out[0][r], out[1][r] for r <= world (r = world: totals)
__global__ void halo_dest_offsets_kernel(const uint32_t *__restrict__ offs, const uint32_t *__restrict__ totals,
                                         uint32_t nb, uint32_t world, uint32_t *__restrict__ out) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r > world) return;
    const size_t plane = static_cast<size_t>(world) * nb;
    out[r] = r < world ? offs[static_cast<size_t>(r) * nb] : totals[0];
    out[world + 1 + r] = r < world ? offs[plane + static_cast<size_t>(r) * nb] : totals[1];
}

// one voxel of a float64-colour block as a halo payload record {tsdf, weight, r, g, b as float64} and back (the
// default volume's kernels copy its five float32 planes in place)
__device__ __forceinline__ void halo_put_f64(float *out, const float *blk, const int v) {
    out[0] = blk[v];
    out[1] = blk[kVox + v];
#pragma unroll
    for (int c = 0; c < 3; ++c) reinterpret_cast<double *>(out + 2)[c] = TsdfBlock<double>::color(blk, c)[v];
}
// voxel q of a record's payload `in` into voxel v of the block at blk
__device__ __forceinline__ void halo_get_f64(float *blk, const float *in, const uint32_t q, const int v) {
    constexpr int kWords = HaloVoxel<double>::kWords;
    blk[v] = in[q * kWords];
    blk[kVox + v] = in[q * kWords + 1];
#pragma unroll
    for (int c = 0; c < 3; ++c)
        TsdfBlock<double>::color(blk, c)[v] = reinterpret_cast<const double *>(in + q * kWords + 2)[c];
}

// one CTA per owned block: its records' headers and voxels at the positions the scan gave them
template <typename TC>   // TC = double: the float64-colour kernel
__device__ __forceinline__ void halo_emit_kernel_body(const PoolMeta M, uint32_t nb, uint32_t world,
                                                      const uint32_t *__restrict__ offs, int4 *__restrict__ headers,
                                                      float *__restrict__ payload) {
    constexpr int kWords = HaloVoxel<TC>::kWords;
    const uint32_t b = blockIdx.x;
    const int4 k = M.block_keys[b];
    uint32_t dest[7], masks[7];
    const int n = halo_dests(k, world, dest, masks);
    const size_t plane = static_cast<size_t>(world) * nb;
    const float *blk = M.pool + static_cast<size_t>(b) * TsdfBlock<TC>::kFloats;
    for (int j = 0; j < n; ++j) {
        const size_t i = static_cast<size_t>(dest[j]) * nb + b;
        const uint32_t rec = offs[i];
        const size_t voff = offs[plane + i];
        if (threadIdx.x == 0)
            headers[rec] = make_int4(k.x, k.y, k.z, static_cast<int>(masks[j]) | HaloVoxel<TC>::kMaskFlag);
        const uint32_t cnt = g_halo_cnt[masks[j]];
        for (uint32_t q = threadIdx.x; q < cnt; q += blockDim.x) {
            const int v = g_halo_vox[masks[j]][q];
            halo_put_f64(payload + (voff + q) * kWords, blk, v);
        }
    }
}

// the default volume's kernel, written out (as an inlined body it would compile to different SASS)
__global__ void __launch_bounds__(128)
halo_emit_kernel(const PoolMeta M, uint32_t nb, uint32_t world, const uint32_t *__restrict__ offs,
                 int4 *__restrict__ headers, float *__restrict__ payload) {
    const uint32_t b = blockIdx.x;
    const int4 k = M.block_keys[b];
    uint32_t dest[7], masks[7];
    const int n = halo_dests(k, world, dest, masks);
    const size_t plane = static_cast<size_t>(world) * nb;
    const float *blk = M.pool + static_cast<size_t>(b) * kBlockFloats;
    for (int j = 0; j < n; ++j) {
        const size_t i = static_cast<size_t>(dest[j]) * nb + b;
        const uint32_t rec = offs[i];
        const size_t voff = offs[plane + i];
        if (threadIdx.x == 0) headers[rec] = make_int4(k.x, k.y, k.z, static_cast<int>(masks[j]));
        const uint32_t cnt = g_halo_cnt[masks[j]];
        for (uint32_t q = threadIdx.x; q < cnt; q += blockDim.x) {
            const int v = g_halo_vox[masks[j]][q];
            float *out = payload + (voff + q) * kPlanes;
#pragma unroll
            for (int c = 0; c < kPlanes; ++c) out[c] = blk[c * kVox + v];
        }
    }
}
// the float64-colour instantiation
__global__ void __launch_bounds__(128)
halo_emit_kernel_c64(const PoolMeta M, uint32_t nb, uint32_t world, const uint32_t *__restrict__ offs,
                 int4 *__restrict__ headers, float *__restrict__ payload) {
    halo_emit_kernel_body<double>(M, nb, world, offs, headers, payload);
}

cudaError_t launch_halo_count(const PoolMeta &meta, uint32_t nb, uint32_t world, uint32_t *counts, uint32_t *offs,
                              uint32_t *partials, uint32_t *totals, uint32_t *dest_offs, cudaStream_t stream) {
    cudaError_t e = upload_halo_tables_once();
    if (e != cudaSuccess) return e;
    const size_t n = static_cast<size_t>(world) * nb;
    e = cudaMemsetAsync(counts, 0, 2 * n * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    e = cudaMemsetAsync(totals, 0, 2 * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    if (n) {
        halo_count_kernel<<<(nb + 255) / 256, 256, 0, stream>>>(meta.block_keys, nb, world, counts);
        const dim3 chunks(static_cast<unsigned>((n + 1023) / 1024), 2);
        scan_reduce_kernel<<<chunks, 1024, 0, stream>>>(counts, partials, static_cast<uint32_t>(n));
        scan_apply_kernel<<<chunks, 1024, 0, stream>>>(counts, offs, partials, totals, static_cast<uint32_t>(n));
    }
    halo_dest_offsets_kernel<<<(world + 1 + 255) / 256, 256, 0, stream>>>(offs, totals, nb, world, dest_offs);
    return cudaGetLastError();
}

cudaError_t launch_halo_emit(const PoolMeta &meta, uint32_t nb, uint32_t world, const uint32_t *offs, int32_t *headers,
                             float *payload, cudaStream_t stream, bool color_f64) {
    if (nb == 0) return cudaSuccess;
    (color_f64 ? halo_emit_kernel_c64 : halo_emit_kernel)<<<nb, 128, 0, stream>>>(
        meta, nb, world, offs, reinterpret_cast<int4 *>(headers), payload);
    return cudaGetLastError();
}

// ---- import into the extraction scratch ---------------------------------------------------------------------------

// insert a key that must be new with a given pool index
__device__ __forceinline__ void insert_at(const HashTable &T, const PoolMeta &D, int4 k, uint32_t idx) {
    bool is_new;
    const uint32_t s = table_insert(T, k.x, k.y, k.z, &is_new);
    if (s == kEmpty || !is_new) {   // table full / a key imported twice
        atomicOr(D.counters + kCtrError, s == kEmpty ? 2u : 8u);
        return;
    }
    reinterpret_cast<uint32_t *>(T.entries + s)[3] = idx;
    D.block_keys[idx] = make_int4(k.x, k.y, k.z, 0);
}

// one CTA per owned block: the live block b becomes scratch block b (voxels, sign summary, table entry)
template <typename TC>
__device__ __forceinline__ void halo_copy_owned_kernel_body(const PoolMeta S, const HashTable T, const PoolMeta D) {
    constexpr int kFloats = TsdfBlock<TC>::kFloats;
    const uint32_t b = blockIdx.x;
    const float4 *src = reinterpret_cast<const float4 *>(S.pool + static_cast<size_t>(b) * kFloats);
    float4 *dst = reinterpret_cast<float4 *>(D.pool + static_cast<size_t>(b) * kFloats);
    for (int i = threadIdx.x; i < kFloats / 4; i += blockDim.x) dst[i] = src[i];
    if (threadIdx.x == 0) {
        D.block_flags[b] = S.block_flags[b];
        insert_at(T, D, S.block_keys[b], b);
    }
}

__global__ void __launch_bounds__(128)
halo_copy_owned_kernel(const PoolMeta S, const HashTable T, const PoolMeta D) {
    halo_copy_owned_kernel_body<float>(S, T, D);
}
// the float64-colour instantiation
__global__ void __launch_bounds__(128)
halo_copy_owned_kernel_c64(const PoolMeta S, const HashTable T, const PoolMeta D) {
    halo_copy_owned_kernel_body<double>(S, T, D);
}

// counts[j] = voxels of record j (the receiver's payload offsets come from their scan); a bad mask counts 0 and is
// reported by the import.  A record of the other colour type (kHaloColorF64 set or missing) has a bad mask.
template <typename TC>
__device__ __forceinline__ void halo_record_sizes_kernel_body(const int4 *__restrict__ headers, uint32_t n,
                                                              uint32_t *__restrict__ counts) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int m = headers[j].w - HaloVoxel<TC>::kMaskFlag;
    counts[j] = (m > 0 && m < 128) ? g_halo_cnt[m] : 0u;
}

__global__ void
halo_record_sizes_kernel(const int4 *__restrict__ headers, uint32_t n, uint32_t *__restrict__ counts) {
    halo_record_sizes_kernel_body<float>(headers, n, counts);
}
// the float64-colour instantiation
__global__ void
halo_record_sizes_kernel_c64(const int4 *__restrict__ headers, uint32_t n, uint32_t *__restrict__ counts) {
    halo_record_sizes_kernel_body<double>(headers, n, counts);
}

// one CTA per record: a zero-filled block at pool index base + j with the record's voxels scattered into it; its sign
// summary is computed from what was written
template <typename TC>   // TC = double: the float64-colour kernel
__device__ __forceinline__ void halo_import_kernel_body(const int4 *__restrict__ headers,
                                                        const float *__restrict__ payload,
                                                        const uint32_t *__restrict__ offs, uint32_t base,
                                                        const HashTable T, const PoolMeta D) {
    constexpr int kFloats = TsdfBlock<TC>::kFloats, kWords = HaloVoxel<TC>::kWords;
    const uint32_t j = blockIdx.x;
    const int4 h = headers[j];
    const int hm = h.w - HaloVoxel<TC>::kMaskFlag;
    const uint32_t idx = base + j;
    float *blk = D.pool + static_cast<size_t>(idx) * kFloats;
    float4 *b4 = reinterpret_cast<float4 *>(blk);
    for (int i = threadIdx.x; i < kFloats / 4; i += blockDim.x) b4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    const bool ok = hm > 0 && hm < 128;
    bool neg = false, pos = false;
    if (ok) {
        const uint32_t cnt = g_halo_cnt[hm];
        const float *in = payload + static_cast<size_t>(offs[j]) * kWords;
        for (uint32_t q = threadIdx.x; q < cnt; q += blockDim.x) {
            const int v = g_halo_vox[hm][q];
            halo_get_f64(blk, in, q, v);
            const float f = in[q * kWords], w = in[q * kWords + 1];
            neg |= w != 0.0f && f < 0.0f;
            pos |= w != 0.0f && !(f < 0.0f);
        }
    }
    const int any_neg = __syncthreads_or(neg);
    const int any_pos = __syncthreads_or(pos);
    if (threadIdx.x == 0) {
        if (!ok) atomicOr(D.counters + kCtrError, 4u);
        D.block_flags[idx] = (any_neg ? 1u : 0u) | (any_pos ? 2u : 0u);
        insert_at(T, D, make_int4(h.x, h.y, h.z, 0), idx);
    }
}

// the default volume's kernel, written out (as an inlined body it would compile to different SASS)
__global__ void __launch_bounds__(128)
halo_import_kernel(const int4 *__restrict__ headers, const float *__restrict__ payload, const uint32_t *__restrict__ offs,
                   uint32_t base, const HashTable T, const PoolMeta D) {
    const uint32_t j = blockIdx.x;
    const int4 h = headers[j];
    const uint32_t idx = base + j;
    float *blk = D.pool + static_cast<size_t>(idx) * kBlockFloats;
    float4 *b4 = reinterpret_cast<float4 *>(blk);
    for (int i = threadIdx.x; i < kBlockFloats / 4; i += blockDim.x) b4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    const bool ok = h.w > 0 && h.w < 128;
    bool neg = false, pos = false;
    if (ok) {
        const uint32_t cnt = g_halo_cnt[h.w];
        const float *in = payload + static_cast<size_t>(offs[j]) * kPlanes;
        for (uint32_t q = threadIdx.x; q < cnt; q += blockDim.x) {
            const int v = g_halo_vox[h.w][q];
#pragma unroll
            for (int c = 0; c < kPlanes; ++c) blk[c * kVox + v] = in[q * kPlanes + c];
            const float f = in[q * kPlanes], w = in[q * kPlanes + 1];
            neg |= w != 0.0f && f < 0.0f;
            pos |= w != 0.0f && !(f < 0.0f);
        }
    }
    const int any_neg = __syncthreads_or(neg);
    const int any_pos = __syncthreads_or(pos);
    if (threadIdx.x == 0) {
        if (!ok) atomicOr(D.counters + kCtrError, 4u);
        D.block_flags[idx] = (any_neg ? 1u : 0u) | (any_pos ? 2u : 0u);
        insert_at(T, D, make_int4(h.x, h.y, h.z, 0), idx);
    }
}
// the float64-colour instantiation
__global__ void __launch_bounds__(128)
halo_import_kernel_c64(const int4 *__restrict__ headers, const float *__restrict__ payload, const uint32_t *__restrict__ offs,
                   uint32_t base, const HashTable T, const PoolMeta D) {
    halo_import_kernel_body<double>(headers, payload, offs, base, T, D);
}

cudaError_t launch_halo_import(const PoolMeta &src, uint32_t n_owned, const int32_t *headers, const float *payload,
                               uint32_t n_records, uint32_t *sizes, uint32_t *offs, uint32_t *partials,
                               uint32_t *totals, const HashTable &table, const PoolMeta &dst, cudaStream_t stream,
                               bool color_f64) {
    cudaError_t e = upload_halo_tables_once();
    if (e != cudaSuccess) return e;
    if (n_owned)
        (color_f64 ? halo_copy_owned_kernel_c64 : halo_copy_owned_kernel)<<<n_owned, 128, 0, stream>>>(src, table, dst);
    if (n_records) {
        const int4 *h4 = reinterpret_cast<const int4 *>(headers);
        (color_f64 ? halo_record_sizes_kernel_c64 : halo_record_sizes_kernel)<<<(n_records + 255) / 256, 256, 0,
                                                                                stream>>>(h4, n_records, sizes);
        const dim3 chunks((n_records + 1023) / 1024, 1);
        scan_reduce_kernel<<<chunks, 1024, 0, stream>>>(sizes, partials, n_records);
        scan_apply_kernel<<<chunks, 1024, 0, stream>>>(sizes, offs, partials, totals, n_records);
        (color_f64 ? halo_import_kernel_c64 : halo_import_kernel)<<<n_records, 128, 0, stream>>>(h4, payload, offs,
                                                                                                 n_owned, table, dst);
    }
    return cudaGetLastError();
}

// ---- weld ------------------------------------------------------------------------------------------------------------

// A set of 128-bit keys (edge ids {x, y, z, axis}) in an open-addressing table of uint4: an empty slot is all ones
// (axis is 0..2, so no key is), a key is inserted with one 128-bit CAS like the block table's entries.  first[slot]
// keeps the smallest concatenated vertex index with that key.
__device__ __forceinline__ uint32_t edge_slot(const HashTable &T, const int4 k) {
    const uint4 key = make_uint4(static_cast<uint32_t>(k.x), static_cast<uint32_t>(k.y), static_cast<uint32_t>(k.z),
                                 static_cast<uint32_t>(k.w));
    const uint4 empty = make_uint4(kEmpty, kEmpty, kEmpty, kEmpty);
    uint32_t s = (slot_hash(k.x, k.y, k.z) ^ mix32(key.w + 0x9E3779B9u)) & T.mask;
    for (uint32_t probe = 0; probe <= T.mask; ++probe) {
        uint4 e = ld_entry(T.entries + s);
        if (e.x == kEmpty && e.y == kEmpty && e.z == kEmpty && e.w == kEmpty) {
            e = cas_entry(T.entries + s, empty, key);
            if (e.x == kEmpty && e.y == kEmpty && e.z == kEmpty && e.w == kEmpty) return s;
        }
        if (e.x == key.x && e.y == key.y && e.z == key.z && e.w == key.w) return s;
        s = (s + 1) & T.mask;
    }
    return kEmpty;
}

__global__ void weld_insert_kernel(const int4 *__restrict__ edge_ids, uint32_t nv, const HashTable T,
                                   uint32_t *__restrict__ slot_of, uint32_t *__restrict__ first, uint32_t *error) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nv) return;
    const uint32_t s = edge_slot(T, edge_ids[i]);
    slot_of[i] = s;
    if (s == kEmpty) {
        atomicOr(error, 1u);
        return;
    }
    atomicMin(first + s, i);
}

__global__ void weld_keep_kernel(const uint32_t *__restrict__ slot_of, const uint32_t *__restrict__ first, uint32_t nv,
                                 uint32_t *__restrict__ keep) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nv) keep[i] = first[slot_of[i]] == i ? 1u : 0u;
}

__global__ void weld_emit_kernel(const double *__restrict__ V, const double *__restrict__ Cc, const int4 *__restrict__ E,
                                 const uint32_t *__restrict__ keep, const uint32_t *__restrict__ newidx, uint32_t nv,
                                 double *__restrict__ oV, double *__restrict__ oC, int4 *__restrict__ oE) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nv || !keep[i]) return;
    const size_t o = newidx[i];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        oV[3 * o + c] = V[3 * static_cast<size_t>(i) + c];
        oC[3 * o + c] = Cc[3 * static_cast<size_t>(i) + c];
    }
    oE[o] = E[i];
}

// triangle t of piece p (tri_base[p] <= t < tri_base[p + 1]) holds indices local to the piece's vertices
__global__ void weld_triangles_kernel(const int32_t *__restrict__ tri, uint32_t nt, const uint32_t *__restrict__ vbase,
                                      const uint32_t *__restrict__ tbase, int n_pieces,
                                      const uint32_t *__restrict__ slot_of, const uint32_t *__restrict__ first,
                                      const uint32_t *__restrict__ newidx, int32_t *__restrict__ out) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    int p = 0;
    while (p + 1 < n_pieces && tbase[p + 1] <= t) ++p;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const uint32_t g = vbase[p] + static_cast<uint32_t>(tri[3 * static_cast<size_t>(t) + c]);
        out[3 * static_cast<size_t>(t) + c] = static_cast<int32_t>(newidx[first[slot_of[g]]]);
    }
}

cudaError_t launch_weld(const WeldArgs &a, cudaStream_t stream) {
    const unsigned gv = (a.nv + 255) / 256, gt = (a.nt + 255) / 256;
    cudaError_t e = cudaMemsetAsync(a.set.entries, 0xFF, (static_cast<size_t>(a.set.mask) + 1) * sizeof(uint4), stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(a.first, 0xFF, (static_cast<size_t>(a.set.mask) + 1) * sizeof(uint32_t), stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(a.totals, 0, 2 * sizeof(uint32_t), stream);
    if (e != cudaSuccess || a.nv == 0) return e;
    weld_insert_kernel<<<gv, 256, 0, stream>>>(reinterpret_cast<const int4 *>(a.edge_ids), a.nv, a.set, a.slot_of,
                                               a.first, a.totals + 1);
    weld_keep_kernel<<<gv, 256, 0, stream>>>(a.slot_of, a.first, a.nv, a.keep);
    const dim3 chunks((a.nv + 1023) / 1024, 1);
    scan_reduce_kernel<<<chunks, 1024, 0, stream>>>(a.keep, a.partials, a.nv);
    scan_apply_kernel<<<chunks, 1024, 0, stream>>>(a.keep, a.newidx, a.partials, a.totals, a.nv);
    weld_emit_kernel<<<gv, 256, 0, stream>>>(a.vertices, a.colors, reinterpret_cast<const int4 *>(a.edge_ids), a.keep,
                                             a.newidx, a.nv, a.out_vertices, a.out_colors,
                                             reinterpret_cast<int4 *>(a.out_edge_ids));
    if (a.nt)
        weld_triangles_kernel<<<gt, 256, 0, stream>>>(a.triangles, a.nt, a.vbase, a.tbase, a.n_pieces, a.slot_of,
                                                      a.first, a.newidx, a.out_triangles);
    return cudaGetLastError();
}

}  // namespace b2v
