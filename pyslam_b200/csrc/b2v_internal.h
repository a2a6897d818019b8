// b2v_internal.h — host-side state of a volume and the kernel launchers (one .cu per kernel family).
#pragma once

#include <algorithm>
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/b2v.h"
#include "b2v_device.cuh"

// return B2V_ERR_CUDA from the enclosing function, with the failing call in (v)->err, if `call` fails
#define B2V_CUDA(v, call)                                                                  \
    do {                                                                                   \
        cudaError_t e_ = (call);                                                           \
        if (e_ != cudaSuccess) {                                                           \
            (v)->err = std::string(#call) + ": " + cudaGetErrorString(e_);                 \
            return B2V_ERR_CUDA;                                                           \
        }                                                                                  \
    } while (0)

namespace b2v {

// ---- small host utilities (b2v_api.cu) ----
uint32_t next_pow2(uint64_t v);
bool is_device_pointer(const void *p);   // device or managed memory

// One cudaMalloc allocation of T, freed with its owner.  reserve(n) grows it to at least n elements; the contents are
// not kept across a growth and nothing is synchronised beyond what cudaFree does, so a caller whose kernels may
// still read the old allocation synchronises first.
template <typename T> class DeviceBuffer {
  public:
    DeviceBuffer() = default;
    DeviceBuffer(const DeviceBuffer &) = delete;
    DeviceBuffer &operator=(const DeviceBuffer &) = delete;
    DeviceBuffer(DeviceBuffer &&o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
    DeviceBuffer &operator=(DeviceBuffer &&o) noexcept {
        std::swap(p_, o.p_);
        std::swap(n_, o.n_);
        return *this;
    }
    ~DeviceBuffer() { cudaFree(p_); }
    T *get() const { return p_; }
    size_t size() const { return n_; }   // elements
    // nothing if n <= size(); else a fresh allocation of max(n, 1) elements.  On failure it holds nothing (size 0).
    cudaError_t reserve(size_t n) {
        if (n <= n_) return cudaSuccess;
        cudaFree(p_);
        p_ = nullptr;
        n_ = 0;
        const cudaError_t e = cudaMalloc(&p_, std::max<size_t>(n, 1) * sizeof(T));
        if (e == cudaSuccess) n_ = std::max<size_t>(n, 1);
        else p_ = nullptr;
        return e;
    }

  private:
    T *p_ = nullptr;
    size_t n_ = 0;
};

// ---- device storage that grows in place (b2v_api.cu) ----
// One virtual-address range reserved for the maximum size; physical memory is mapped into it in whole granules with
// the driver's virtual memory management entry points, so the address the kernels see never changes and a growth
// copies nothing.  Fixed-size storage takes the same path with the whole reservation mapped at create.  The range
// is released with its owner.
struct VmmRange {
    CUdeviceptr va = 0;
    size_t reserved = 0, mapped = 0, gran = 0;      // bytes
    int device = 0;
    std::vector<std::pair<size_t, size_t>> chunks;  // (offset, bytes) of each mapping
    VmmRange() = default;
    VmmRange(const VmmRange &) = delete;
    VmmRange &operator=(const VmmRange &) = delete;
    ~VmmRange();
};
// reserve at least `bytes`, rounded up to the granularity; false (and *err) on failure
bool vmm_reserve(VmmRange *r, size_t bytes, int device, std::string *err);
// map at least `bytes` (whole granules, capped at the reservation); the newly mapped bytes are zeroed on `stream`
bool vmm_map(VmmRange *r, size_t bytes, cudaStream_t stream, std::string *err);
void vmm_release(VmmRange *r);

// ---- frame store: the frames a map keeps on the device for a loop-closure rebuild (b2v_api.cu) ----
// Slot s of a store holds one frame of the stored frames' size at s * pitch bytes of one address range, reserved for
// `max` frames at the first stored frame and mapped as the store fills, so a stored frame never moves.  Frames, not
// map state: the owner's reset, uploads and growth leave it as it is.  The owner packs a frame into slot(s) and calls
// filled(s) once that copy is enqueued.
struct FrameStore {
    int32_t max = 0;               // 0: off
    int32_t count = 0;             // filled slots, [0, count): their copies are enqueued
    int H = 0, W = 0;              // size of every stored frame (0: none stored yet)
    size_t pitch = 0;              // bytes per slot
    bool stopped = false;          // the device could not reserve or map more: no frame is stored any more
    size_t map_limit = SIZE_MAX;   // B2V_FRAME_STORE_MAX_BYTES: the most the store maps (tests of that path)
    VmmRange range;
    std::vector<int32_t> last;     // slot of each frame of the owner's most recent call, or -1

    FrameStore();   // reads B2V_FRAME_STORE_MAX_BYTES
    void *slot(int32_t s) const { return reinterpret_cast<char *>(range.va) + static_cast<size_t>(s) * pitch; }
    // last := n times -1 (every call that may store frames starts with it, and so does one that stores none)
    void begin_call(int32_t n) { last.assign(static_cast<size_t>(std::max(n, 0)), -1); }
    // The slots of the first n entries of `last`, before anything is launched: handed out in frame order while the
    // store has room, to frames of the stored frames' size.  The first stored frame sets that size and reserves the
    // address range (pitch bytes per slot); the storage the frames need is mapped here (zeroed on `stream`; at least
    // doubling the mapping, else just what they need).  When the device cannot reserve or map it, the frames that fit
    // in what is mapped get slots and the store stops: later frames are not stored and the owner's call goes on.
    void assign(int32_t n, int H, int W, size_t pitch, int device, cudaStream_t stream);
    void filled(int32_t s) { count = s + 1; }   // slots are handed out and filled in frame order
    // on every return of a call: the slots whose copies were not enqueued go back to -1
    void drop_unfilled() {
        for (int32_t &s : last)
            if (s >= count) s = -1;
    }
    bool holds(int32_t s) const { return s >= 0 && s < count; }
    // empties the store and releases its memory; the caller first waits for every call that may read or write it
    void release();
};

// Texel of the update kernels, one per pixel of a frame, packed by the allocate kernels: {depth, r | g << 8 | b << 16}.
// depth is 0 where the pixel is invalid (0, or beyond depth_trunc).  The depth-to-camera-distance multiplier is not
// in the texel: the update kernels read it from the lambda image at the same pixel (one image per set of intrinsics).
struct alignas(8) Texel {
    float depth;
    uint32_t rgb;
};
__device__ __forceinline__ Texel make_texel(float depth, uint8_t r, uint8_t g, uint8_t b) {
    return Texel{depth, static_cast<uint32_t>(r) | (static_cast<uint32_t>(g) << 8) | (static_cast<uint32_t>(b) << 16)};
}
__device__ __forceinline__ Texel load_texel(const Texel *p) {  // read-only path, one 8-byte load
    const uint2 u = __ldg(reinterpret_cast<const uint2 *>(p));
    return Texel{__uint_as_float(u.x), u.y};
}
// colour channel c (0 = r, 1 = g, 2 = b) as float32, exactly: (2^23 + c) - 2^23.  One byte permute builds the bits
// 0x4B0000cc: byte 0 = byte c of rgb, bytes 1, 2 = 0x00 and byte 3 = 0x4B of the constant.
__device__ __forceinline__ float texel_channel(const Texel &t, int c) {
    return __fsub_rn(__uint_as_float(__byte_perm(t.rgb, 0x4B000000u, 0x7440u + c)), 8388608.0f);
}

// Constants of the projective update (Open3D UniformTSDFVolume::IntegrateWithDepthToCameraDistanceMultiplier), split
// into what the frames of a group share and what each frame has of its own.  The shared part sits in kernel-parameter
// space at fixed offsets, so the kernels read it as constant-bank operands.
struct IntConsts {
    float fxf, fyf, cxf, cyf;
    float safe_w, safe_h;   // W - 0.0001f, H - 0.0001f
    float tau, inv_tau;
    int32_t W;
    int32_t pixels;         // W * H: the index that voxels projecting outside the image gather (see below)
    const Texel *tex;       // texels of frame 0 of the group; frame k's start k * tex_pitch texels later
    const float *lam;       // lambda image of the intrinsics, same pixel index as the texels
    int64_t tex_pitch;
};
// The camera pose of one frame, 64 bytes: a frame step reads it with four 16-byte loads.
struct alignas(16) IntPose {
    float E[12];     // Tcw rows 0..2 as float32 (extrinsic.cast<float>())
    float Es[3];     // E[2], E[6], E[10] times voxel_length_f (extrinsic_scaled_f(:, 2)): the per-z-step increment
    float pad;
};
static_assert(sizeof(IntPose) == 64, "IntPose is four float4");
// Texel and lambda images hold one element past the W * H pixels.  The update kernels gather it, instead of
// predicating the loads, for a voxel outside the image.  Its lambda is NaN (written with the lambda image), so the
// voxel's sdf is NaN and the update skips it whatever the texel there holds; the texel buffers are allocated for the
// largest frame so far and reused for smaller ones, where index W * H is a pixel of an earlier frame.
constexpr float kLambdaSentinel = __builtin_nanf("");

// camera -> world of one frame, float64 (allocation samples)
struct FramePose {
    double Rwc[9];   // rigid inverse of Tcw, row-major
    double twc[3];
};

// Per-frame constants of the allocate kernels (+ the update constants of the frame-by-frame kernels).
struct FrameParams {
    // f64 back-projection of the allocation samples (Open3D CreatePointCloudFromFloatDepthImage)
    double fx, fy, cx, cy;
    FramePose pose;
    double tau_d;    // sdf_trunc as float64 (unit mode: the value Open3D holds; D1: (double)sdf_trunc_f)
    double unit_len; // voxel_length * unit resolution, float64 (volume_unit_length_)
    IntConsts I;     // update constants (tex, lam, tex_pitch: set by the caller)
    IntPose E;       // update pose
    float inv_fx, inv_fy;   // 1.0f / fx, 1.0f / fy (lambda image)
    float inv_vs, depth_trunc;
    int32_t unit_shift;     // log2(blocks per unit side): 0 = 8^3 units (D1 allocation), 1 = Open3D's 16^3 units
    int32_t H, W, stride;
    int32_t shard_rank, shard_count;
    int32_t group_buf;      // group buffer the allocation records into (membership masks, union list, counters)
};

// Volume-wide constants of the update kernels (frame independent).
struct VolumeConsts {
    double unit_len;     // float64 volume-unit length
    float vs, half_vs;   // voxel_length_f, voxel_length_f * 0.5f
    int32_t unit_shift;
};

// Frames are integrated in groups.  Fused groups of up to kMaxGroup consecutive frames are applied to a block while
// it is resident in registers; a single frame is a group of one on the frame-by-frame kernels.
constexpr int kMaxGroup = 32;   // frames per fused group (bits of the membership mask); the default group is 16
// group state (masks, union list, staging, texel images, counters) is kGroupBufs-deep: the allocation of group g+3
// may run while group g is still being integrated
constexpr int kGroupBufs = 4;
struct GroupArgs {
    IntPose f[kMaxGroup];
    IntConsts C;
    VolumeConsts V;
    int32_t count;
};

// Block layout of the TSDF pool, by colour type TC.  Every block holds the tsdf and weight float32 planes, then the
// r, g, b planes of TC (voxel index lx + 8 ly + 64 lz in each plane).  TC = float is the default volume: five float32
// planes, kBlockFloats floats (10 KiB) per block.  TC = double is the float64-colour volume (b2v_config.color_f64):
// Open3D's Vector3d colour, 16 KiB per block.  Every kernel that reads or writes the pool has its body templated on
// TC and two entry points: `name` (float, the default volume's kernel as it always was) and `name_c64` (double).
template <typename TC> struct TsdfBlock {
    static constexpr int kFloats = 2 * kVox + 3 * kVox * static_cast<int>(sizeof(TC) / sizeof(float));
    static constexpr size_t kBytes = static_cast<size_t>(kFloats) * sizeof(float);
    // colour plane c (0 = r) of the block at blk
    __host__ __device__ static TC *color(float *blk, int c) { return reinterpret_cast<TC *>(blk + 2 * kVox) + c * kVox; }
    __host__ __device__ static const TC *color(const float *blk, int c) {
        return reinterpret_cast<const TC *>(blk + 2 * kVox) + c * kVox;
    }
    // colour c of voxel v of the block at blk
    __host__ __device__ static TC color_at(const float *blk, int c, int v) {
        if constexpr (sizeof(TC) == sizeof(float)) return blk[(2 + c) * kVox + v];
        else return color(blk, c)[v];
    }
};
static_assert(TsdfBlock<float>::kFloats == kBlockFloats && TsdfBlock<double>::kBytes == 16384, "block layouts");
inline size_t tsdf_block_bytes(bool color_f64) {
    return color_f64 ? TsdfBlock<double>::kBytes : TsdfBlock<float>::kBytes;
}

// Device-resident bookkeeping of one volume.  Everything indexed by table slot or pool index is sized for the
// maximum capacity; only the pool's storage grows (a growable volume maps it on demand, see b2v_api.cu).
struct PoolMeta {
    float *pool;              // [pool_capacity] blocks of TsdfBlock<TC>::kFloats floats (see TsdfBlock)
    int4 *block_keys;         // [capacity] key of pool block i (w unused)
    uint32_t *counters;       // device counters, see Counter
    uint32_t *group_mask;     // [kGroupBufs][table capacity] bit k: the slot is touched by frame k of the group
    uint32_t *union_slots;    // [kGroupBufs][capacity] slots touched by any frame of the group
    uint32_t *block_flags;    // [capacity] sign summary for the mesh extraction's tile filter: bit 0 = some store left
                              // an observed voxel (w != 0) with tsdf < 0, bit 1 = with tsdf >= 0; bits are only ever
                              // set, so the union over a tile is a superset of the signs present now
    uint32_t capacity;        // maximum capacity: stride of the union lists; allocation hands out pool indices below
                              // it (the others get kNoBlock)
    uint32_t pool_capacity;   // blocks with storage now (<= capacity).  A growable volume skips every group from the
                              // first that was handed an index past it, until the host has mapped storage for them
};

enum Counter : int {
    kCtrPool = 0,            // number of allocated blocks (may exceed pool_capacity on overflow)
    kCtrError = 1,           // sticky error flag (1 = pool overflow, 2 = table full)
    kCtrUpdatesLo = 2,       // 64-bit total of (block, frame) updates since reset (8-byte aligned)
    kCtrUpdatesHi = 3,
    kCtrSkipping = 4,        // growable volumes: sticky, set by the gate of the first group that saw kCtrPool pass
                             // pool_capacity; every later group is skipped too until the host grows the pool and
                             // replays them
    kCtrSavedUnion0 = 5,     // [kGroupBufs] kGcUnion of the skipped group of each buffer (restored for the replay)
    kCtrVisitsLo = 12,       // 64-bit total of block visits (one block read + written) since reset
    kCtrVisitsHi = 13,
    kCtrUnitSetFull = 14,    // (unit, frame) pairs of fused groups that found no entry in the group unit set within
                             // its probe limit and touched their blocks directly, since reset
    kCtrGroup0 = 16,         // [kGroupBufs][kGroupCtrStride] per-group-buffer counters, contiguous so that ONE
                             // memset re-arms a buffer: see GroupCounter
    kNumCounters = 16 + 4 * (4 + 32)
};
// offsets inside one group buffer's counter block (M.counters + kCtrGroup0 + buf * kGroupCtrStride)
enum GroupCounter : int {
    kGcUnion = 0,    // number of slots in the group's union list
    kGcNext = 1,     // work-stealing cursor of the fused kernel
    kGcNew = 2,      // blocks newly allocated by the group
    kGcUnits = 3,    // entries of the group unit set (fused groups)
    kGcTouched0 = 4  // [kMaxGroup] blocks touched by frame k of the group
};
constexpr int kGroupCtrStride = 4 + kMaxGroup;
__host__ __device__ __forceinline__ constexpr int group_ctr(int buf, int which) {
    return kCtrGroup0 + buf * kGroupCtrStride + which;
}
static_assert(kGcTouched0 + kMaxGroup <= kGroupCtrStride && kCtrGroup0 + kGroupBufs * kGroupCtrStride <= kNumCounters,
              "counter layout");
static_assert(kCtrSavedUnion0 + kGroupBufs <= kCtrVisitsLo, "counter layout");

struct VolumeGeometry {   // set once per volume (b2v_create)
    float vs, tau, depth_trunc;
    double voxel_length, tau_d;   // float64 values as Open3D holds them
    int32_t unit_shift, stride;
    int32_t shard_rank, shard_count;
};
void fill_frame_params(FrameParams *p, const double K[4], const double Tcw[16], int H, int W,
                       const VolumeGeometry &g);
VolumeConsts volume_consts(const VolumeGeometry &g);

// ---- kernels (b2v_tsdf.cu) ----
// lambda image (Open3D's depth-to-camera-distance multiplier) for the current intrinsics
cudaError_t launch_lambda(const FrameParams &p, float *lam, cudaStream_t stream);
// TMA descriptors of one frame's images (2-D tiled: depth f32, colour u8 x3 interleaved)
struct FrameMaps {
    alignas(64) CUtensorMap depth;
    alignas(64) CUtensorMap color;
    const void *color_ptr = nullptr;  // host-side cache validation only
};
// TMA tile staging needs 16-byte aligned bases and row pitches (W % 16 == 0) and the 32x32 tile
bool tma_tiles_usable(int W, int stride, const void *depth, const void *color);
// returns false if the driver entry point is unavailable or encoding fails
bool encode_frame_maps(FrameMaps *maps, const float *depth, const uint8_t *color, int H, int W, int tile);
// The allocation units a fused group touches and, per unit, the frames that touch it: one set per group buffer, filled
// by allocate_group_kernel (per frame and tile) and read and cleared by allocate_group_expand_kernel (per group).
// Entry {ux, uy, uz, frame mask}; mask 0 = empty.  Sized for the largest union with slack (b2v_api.cu).
struct UnitSet {
    uint4 *entries;   // [kGroupBufs][mask + 1]
    uint32_t *list;   // [kGroupBufs][mask + 1] entry positions of the group's units, in insertion order
    uint32_t mask;    // entries per buffer - 1 (a power of two)
};
// Frame packing (texels) + allocation + touched set of the frames of a group, recorded in group buffer
// P.group_buf.  use_tma: the image tiles are staged into shared memory with TMA (cp.async.bulk.tensor.2d); else
// plain loads.
struct GroupAllocArgs {
    FrameParams P;                 // constants shared by the frames of the group (P.pose / P.I: frame 0's)
    FramePose pose[kMaxGroup];
    const float *depth[kMaxGroup];
    const uint8_t *color[kMaxGroup];
    Texel *tex[kMaxGroup];
    FrameMaps maps[kMaxGroup];
    UnitSet units;                 // fused groups
    int32_t count, use_tma;
};
static_assert(sizeof(GroupAllocArgs) < 32000, "kernel parameter space");
// a one-frame group (frame 0 of args), with the frame-by-frame allocate_kernel.  from_tex: the frame's texel image is
// already in args.tex[0] (a frame replayed from the frame store): depth, colour and maps are not read, nothing is packed
cudaError_t launch_allocate(const GroupAllocArgs &args, const HashTable &table, const PoolMeta &meta,
                            cudaStream_t stream, bool from_tex);
// all frames of a group in ONE launch (blockIdx.z = frame): the per-frame latency chains overlap.  It collects the
// group's units in args.units; a second kernel then touches each block of those units once for the whole group.
// from_tex: as above, for every frame of the group
cudaError_t launch_allocate_group(const GroupAllocArgs &args, const HashTable &table,
                                  const PoolMeta &meta, int sm_count, cudaStream_t stream, bool from_tex);
// projective TSDF + colour update of every block touched by the one-frame group in group buffer group_buf
// (frame 0 of args)
// color_f64: the volume's colour type (TsdfBlock), here and in every launcher below that takes it
cudaError_t launch_integrate(const GroupArgs &args, const HashTable &table, const PoolMeta &meta, int group_buf,
                             int grid_ctas, cudaStream_t stream, bool color_f64);
int integrate_max_resident_ctas_per_sm(bool color_f64);
// d_bad[0]: reciprocals (3 x 2^23 inputs), d_bad[1]: quotients (`pairs` inputs) whose fast path differs from IEEE
cudaError_t launch_selftest_division(unsigned long long *d_bad, uint64_t pairs, cudaStream_t stream);
// fused update of a group of frames (each block is read and written once per group)
cudaError_t launch_integrate_group(const GroupArgs &args, const HashTable &table, const PoolMeta &meta,
                                   int group_buf, int grid_ctas, int sm_count, cudaStream_t stream, bool color_f64);
// keys of the slots in a touched list
cudaError_t launch_gather_active_keys(const HashTable &table, const uint32_t *slots,
                                      uint32_t n, int4 *out, cudaStream_t stream);

// find-or-create the blocks of `keys` (unique) and copy `vox` (n blocks in the pool's layout) into them
// the largest weight a voxel may hold: w + 1 is exact below it and rounds back to it there (integration saturates)
constexpr float kWeightMax = 16777216.0f;  // 2^24
cudaError_t launch_upload_check(const float *vox, uint32_t n, uint32_t *bad, cudaStream_t stream, bool color_f64);
cudaError_t launch_upload_blocks(const int4 *keys, const float *vox, uint32_t n, uint32_t *scratch_idx,
                                 const HashTable &table, const PoolMeta &meta, cudaStream_t stream, bool color_f64);

// ---- pool growth (growable volumes) ----
// one thread, between a group's allocation and its update: if pool indices past the storage were handed out
// (kCtrPool > pool_capacity), or an earlier group is being skipped, mark the volume as skipping, save the group's union
// count and zero it (the update kernels then do nothing and leave the group's masks and list in place for the replay)
cudaError_t launch_group_gate(const PoolMeta &meta, int group_buf, cudaStream_t stream);
// when the storage could not grow: entries holding an index past it lose it (kNoBlock, "block pool full")
cudaError_t launch_drop_unbacked_blocks(const HashTable &table, const PoolMeta &meta, cudaStream_t stream);
// the same for any block table: entries with a pool index in [storage, capacity) get kNoBlock and set bit 0 of *error
cudaError_t launch_drop_unbacked_slots(const HashTable &table, uint32_t storage, uint32_t capacity, uint32_t *error,
                                       cudaStream_t stream);

// ---- mesh (b2v_mesh.cu) ----
// Scratch and outputs of one extraction.  Per-voxel scratch is indexed [pool block][voxel].
struct MeshBuffers {
    uint32_t n_blocks;
    int32_t *nbr;            // [n_blocks][8] pool index of the block at +(dx,dy,dz) (bit0=x), -1 if missing
    uint8_t *cube;           // [n_blocks][512] marching-cubes case of the cube rooted here (0 = none)
    uint32_t *edge_mask;     // [n_blocks][128] byte per voxel: bit a = a vertex lives on its +a edge
    uint32_t *local;         // [n_blocks][512] position of the voxel's first vertex (low 16 bits) / triangle (high) in its block
    uint32_t *sums;          // [2][n_blocks] per-block vertex / triangle counts
    uint32_t *offs;          // [2][n_blocks] exclusive scans of sums
    uint32_t *partials;      // [2][ceil(n_blocks / 1024)] chunk sums of the two-level scan
    uint32_t *totals;        // [8] total vertices, triangles; blocks with vertices, blocks with triangles; candidate
                             // tiles (sign-summary filter), classified tiles (see MeshTotal)
    uint32_t *work;          // [4][n_blocks] the blocks with vertices / with triangles (what the emit kernels visit);
                             // candidate tiles; tiles with a sign change (what classify / block sums visit)
    double *vertices;        // [nv][3] float64, Open3D's formula
    double *colors;          // [nv][3] in [0,1]
    int32_t *edge_ids;       // [nv][4] canonical weld key (voxel x,y,z, axis)
    int32_t *triangles;      // [nt][3]
};
enum MeshTotal : int { kMtVertices = 0, kMtTriangles = 1, kMtVertexBlocks = 2, kMtTriangleBlocks = 3,
                       kMtCandidates = 4, kMtTiles = 5, kNumMeshTotals = 8 };
// neighbour lookup (7 hash probes per block) + candidate tiles from the blocks' sign summaries, then the
// marching-cubes case per voxel + vertex ownership masks of the candidates (Open3D ExtractTriangleMesh semantics)
cudaError_t launch_mesh_classify(const HashTable &table, const PoolMeta &meta, const MeshBuffers &mb, int grid_ctas,
                                 cudaStream_t stream, bool color_f64);
// the same front end + zero-crossing masks of Open3D ExtractPointCloud (no cube validity requirement)
cudaError_t launch_point_masks(const HashTable &table, const PoolMeta &meta, const MeshBuffers &mb, int grid_ctas,
                               cudaStream_t stream, bool color_f64);
// per-block sums + exclusive scans -> offs, totals
cudaError_t launch_mesh_scan(const MeshBuffers &mb, int grid_ctas, cudaStream_t stream);
cudaError_t launch_mesh_vertices(const PoolMeta &meta, const MeshBuffers &mb, double voxel_length, int unit_shift,
                                 bool points, uint32_t work_blocks, cudaStream_t stream, bool color_f64);
cudaError_t launch_mesh_triangles(const MeshBuffers &mb, uint32_t work_blocks, cudaStream_t stream);

// ---- face-halo exchange of a sharded volume (b2v_shard.cu) ----
// a halo record carries the union of the faces / lines / corner a rank needs of a block: at most the 512 - 7^3 = 169
// voxels with some local coordinate 0
constexpr int kHaloMaxVoxels = 169;
// counts [2][world * nb] (zeroed here), offs the same, partials [2][ceil(world * nb / 1024)], totals [2];
// dest_offs [2][world + 1]: the first record / payload voxel of each destination (index world: the totals)
cudaError_t launch_halo_count(const PoolMeta &meta, uint32_t nb, uint32_t world, uint32_t *counts, uint32_t *offs,
                              uint32_t *partials, uint32_t *totals, uint32_t *dest_offs, cudaStream_t stream);
// headers int32 [records][4] = {key x, y, z, mask}, payload [voxels][HaloVoxel<TC>::kWords], at the positions of
// launch_halo_count.  A float64-colour volume sets kHaloColorF64 in every mask it sends and imports only such records.
constexpr int kHaloColorF64 = B2V_HALO_COLOR_F64;
template <typename TC> struct HaloVoxel {   // {tsdf, weight, r, g, b}: float32 tsdf, weight and colour of type TC
    static constexpr int kWords = 2 + 3 * static_cast<int>(sizeof(TC) / sizeof(float));   // 5 or 8 float32 words
    static constexpr int kMaskFlag = sizeof(TC) == sizeof(double) ? kHaloColorF64 : 0;
};
inline int halo_voxel_words(bool color_f64) { return color_f64 ? HaloVoxel<double>::kWords : HaloVoxel<float>::kWords; }
cudaError_t launch_halo_emit(const PoolMeta &meta, uint32_t nb, uint32_t world, const uint32_t *offs, int32_t *headers,
                             float *payload, cudaStream_t stream, bool color_f64);
// scratch dst := src blocks [0, n_owned) at the same pool indices + the records as zero-filled halo blocks at
// [n_owned, n_owned + n_records); the table must be empty.  sizes / offs [n_records], partials, totals: scan scratch.
// dst.counters[kCtrError]: bit 1 table full, bit 2 a record with a bad mask, bit 3 a key imported twice
cudaError_t launch_halo_import(const PoolMeta &src, uint32_t n_owned, const int32_t *headers, const float *payload,
                               uint32_t n_records, uint32_t *sizes, uint32_t *offs, uint32_t *partials,
                               uint32_t *totals, const HashTable &table, const PoolMeta &dst, cudaStream_t stream,
                               bool color_f64);
// weld of concatenated mesh pieces by edge id: vertices in order of first occurrence, triangles remapped
struct WeldArgs {
    uint32_t nv, nt;
    int32_t n_pieces;
    const double *vertices, *colors;
    const int32_t *edge_ids, *triangles;   // triangles hold piece-local vertex indices
    const uint32_t *vbase, *tbase;         // [n_pieces + 1] first vertex / triangle of each piece
    HashTable set;                         // edge-id set, >= 2 nv slots
    uint32_t *first, *slot_of, *keep, *newidx, *partials;
    uint32_t *totals;                      // [2]: kept vertices, set-full flag
    double *out_vertices, *out_colors;
    int32_t *out_edge_ids, *out_triangles;
};
cudaError_t launch_weld(const WeldArgs &args, cudaStream_t stream);

// ---- sparse block grids: the point-average grid (b2v_grid.cu) and the semantic grids (b2v_semantic.cu) ----
// Both keep their blocks in a 128-bit-CAS table whose entries hold a pool index, and the key of pool block i in
// block_keys[i].  They differ only in what a voxel stores and how it is updated.
enum BlockGridCounter : int {
    kBgPool = 0,            // number of allocated blocks (may exceed pool_capacity on overflow)
    kBgError = 1,           // sticky error flag (1 = pool overflow, 2 = table full)
    kBgLabelOverflow = 2,   // semantic grids: label pairs evicted for want of a slot
    kBgNumCounters = 4
};
struct BlockIndex {
    int4 *block_keys;         // [capacity]
    uint32_t *counters;       // see BlockGridCounter
    uint32_t capacity;        // maximum capacity: allocation hands out pool indices below it (the others get kNoBlock)
    uint32_t pool_capacity;   // blocks with storage now (<= capacity); a growable grid maps more within the call
    // hash sharding (SURVEY.md 8e): the grid holds only the blocks with block_owner(key, shard_count) == shard_rank
    uint32_t shard_rank = 0, shard_count = 1;
};
// Block insert of every point (optional per-point mask `valid`): each block (side 1 << log2_block) a point falls in
// gets a table entry and a pool index (kNoBlock once the index passes index.capacity).  Points are float or double
// [n][3].
cudaError_t launch_point_insert(const void *pts, bool pts_f64, const uint8_t *valid, int64_t n, float inv_vs,
                                int log2_block, const HashTable &table, const BlockIndex &index, cudaStream_t stream);
// sort key of a point without storage in the pass's window: above every voxel id, so it sorts last
constexpr uint32_t kBadVid = 0xFFFFFFFFu;

// The block sides the grids accept: B = 1, 2, 8, 16 (L = 0, 1, 3, 4).  B = 4 keeps the rejection the grids gave every
// size but 8 before block sizes were supported, which their argument checks pin (tests/test_gpu_grid.py,
// tests/test_gpu_semantic.py); the kernels and the key rules are written for any L in [0, kMaxGridLog2B].
__host__ __device__ constexpr bool grid_log2_block_supported(int l) { return l == 0 || l == 1 || l == 3 || l == 4; }
static_assert(kMaxGridLog2B == 4, "grid_log2_block_supported lists L = 0 .. 4");

// The grids' block side B = 1 << L is a template parameter of their kernels: f(std::integral_constant<int, L>{}) for
// a supported log2_block (grid_log2_block_supported), the one place a grid's runtime block size picks its kernels.
template <typename F> decltype(auto) with_grid_block(int log2_block, F &&f) {
    switch (log2_block) {
    case 0: return f(std::integral_constant<int, 0>{});
    case 1: return f(std::integral_constant<int, 1>{});
    case 3: return f(std::integral_constant<int, 3>{});
    default: return f(std::integral_constant<int, 4>{});
    }
}

// Fused RGBD front-end: depth2pointcloud (pyslam/utilities/depth.py:45-85) + world transform
// (pyslam/dense/volumetric_integrator_voxel_grid.py:262-281, volumetric_integrator_voxel_semantic_grid.py:411-436),
// without materialising the point cloud.  float64 arithmetic in the reference's operation order, then float32 like
// the front-end.
struct RgbdParams {
    double fx_inv, fy_inv, cx, cy;   // 1.0 / fx, 1.0 / fy (depth.py:67-68)
    double R[9], t[3];               // Twc (camera -> world)
    float min_depth, max_depth;
    int32_t H, W;
};
RgbdParams rgbd_params(const double K[4], const double Twc[16], float min_depth, float max_depth, int H, int W);

// Spatial read-outs / carving over the existing blocks (voxel_block_grid.hpp:717-1195, 1334-1540;
// voxel_grid_carving.h:47-80; camera_frustrum.cpp:174-196).  A voxel qualifies if it passes its grid's own count
// rule and, in box and frustum mode, its key lies in [min_key, max_key] and its mean position passes the fine test
// (double arithmetic like the reference).
enum QueryMode : int32_t { kQueryAll = 0, kQueryBox = 1, kQueryFrustum = 2 };
struct GridQuery {
    int32_t mode, min_count;      // mode: QueryMode
    int32_t min_key[3], max_key[3];
    double bb[6];                 // min xyz, max xyz
    double R[9], t[3];            // world -> camera
    float fx, fy, cx, cy, depth_min, depth_max;
    int32_t W, H;
};

// The per-voxel arrays of a grid's blocks as a block upload copies them: array k holds a run of block_bytes[k] bytes
// per block at dst[k] + pool index * block_bytes[k], and the uploaded blocks' runs follow one another in src[k].
constexpr int kMaxBlockArrays = 11;
struct BlockArrays {
    void *dst[kMaxBlockArrays];
    const void *src[kMaxBlockArrays];
    uint32_t block_bytes[kMaxBlockArrays];
    int32_t n_arrays;
};

// The host half both grids share: device and stream, table, block index, counters, growth, scan buffers.
struct BlockGridCore {
    int device = 0;
    cudaStream_t stream = nullptr;
    // the reference stores the voxel size as float and inverts it in float (voxel_block_grid.h:225-226, .hpp:6)
    float inv_voxel_size = 0.0f;
    int log2_block = 3;   // block side B = 1 << log2_block (block_size of create)
    HashTable table{};   // views of table_mem, block_keys, counters
    BlockIndex index{};
    // the table and block_keys are sized for index.capacity; a growable grid maps its storage on demand
    DeviceBuffer<uint4> table_mem;
    DeviceBuffer<int4> block_keys;
    DeviceBuffer<uint32_t> counters;
    bool growable = false;
    int64_t growths = 0;
    uint32_t *h_counters = nullptr;   // pinned mirror of index.counters
    DeviceBuffer<uint32_t> d_sums, d_offs, d_total;   // count -> scan of the read-outs
    std::string err;

    // log2 of a supported block size (1, 2, 8, 16), else -1
    static int log2_block_size(int32_t block_size);
    // the most blocks of side 1 << log2_block a grid may hold: 2^31 voxels (the semantic sort key
    // pool index * B^3 + local stays below its kBadVid), 2^22 blocks at B = 8, and at most 2^30 blocks (the table holds
    // twice the blocks in a power of two of 32-bit slots)
    static uint32_t max_blocks(int log2_block) {
        return static_cast<uint32_t>(std::min<uint64_t>(1ull << 30, (1ull << 31) >> (3 * log2_block)));
    }
    // the arguments both grids accept (max_capacity_blocks 0: a fixed grid)
    static bool valid_args(double voxel_size, int32_t block_size, uint32_t capacity_blocks,
                           uint32_t max_capacity_blocks);
    // stream, table, block index and counters for max(capacity_blocks, max_capacity_blocks) blocks; the grid then
    // maps its storage, sets index.pool_capacity and clears the index (clear_index) with its storage
    int create(double voxel_size, int32_t block_size, uint32_t capacity_blocks, uint32_t max_capacity_blocks,
               int32_t device);
    uint32_t block_voxels() const { return 1u << (3 * log2_block); }   // B^3
    // CTAs of a per-voxel pass over n_blocks blocks (cta_voxel): one per 512 voxels
    uint32_t voxel_ctas(uint32_t n_blocks) const {
        return static_cast<uint32_t>((static_cast<uint64_t>(n_blocks) * block_voxels() + 511) / 512);
    }
    template <typename F> decltype(auto) dispatch(F &&f) const { return with_grid_block(log2_block, f); }
    void destroy();         // waits for the stream, destroys it and frees the pinned mirror
    int fetch_counters();   // h_counters := index.counters (synchronises)
    int read_counters();    // fetch_counters + B2V_ERR_CAPACITY ("hash table full" / "block pool full") on an error bit
    uint32_t block_count() const {   // blocks with storage, as of the last fetch_counters
        return std::min(h_counters[kBgPool], index.pool_capacity);
    }
    int capacity(int64_t *capacity_blocks, int64_t *growths_out);
    // keep only the blocks rank `rank` of `count` owns from now on; only on a grid without blocks (synchronises).
    // clear() keeps the setting.
    int set_shard(int32_t rank, int32_t count);
    int clear_index();      // empty table, zero counters (asynchronous)
    // Growable grids, at the end of an integrate call: the call's first pass skipped the points of blocks handed a
    // pool index past the storage.  map_storage(blocks) maps storage for at least that many blocks and updates
    // index.pool_capacity (at least doubling, at most the maximum); replay(lo, hi) then repeats the pass over the
    // blocks that just got storage, from the same inputs, which must still be alive.  All observations of a voxel
    // in one call belong to one block and a block's index never changes, so every voxel is updated by exactly one of
    // the passes.  If the storage cannot grow, the blocks past it are dropped ("block pool full").  Synchronises.
    template <typename MapStorage, typename Replay> int resolve(MapStorage map_storage, Replay replay);
    // Block upload of both grids (b2v_grid_upload_blocks, b2v_sgrid_upload_blocks): the n HOST keys int32 [n][4]
    // {x, y, z, 0} go through the block insert (a sharded grid skips the blocks it does not own; past index.capacity
    // the index is kNoBlock and the error flag says "block pool full"), a growable grid maps storage for the new pool
    // count (resolve with the grid's map_storage, and fill(lo, hi) setting the blocks that got storage to the cleared
    // state), then every block's run of each array replaces its pool block's run.  Synchronises.
    template <typename MapStorage, typename Fill>
    int upload_blocks(int64_t n, const int32_t *keys4, const BlockArrays &arrays, MapStorage map_storage, Fill fill);
    // its steps: the keys into *d_keys and the table (asynchronous); the copy of the runs (synchronises)
    int insert_keys(int64_t n, const int32_t *keys4, DeviceBuffer<int4> *d_keys);
    int scatter_blocks(int64_t n, const int4 *d_keys, const BlockArrays &arrays);
    // Voxel-order sort of the input-order updates (the semantic grids, the point grid's input-order sums): per point
    // the key pool index * B^3 + local index (kBadVid where the point is masked out by `valid` or its block has no
    // pool index in [lo, hi)) and the point index, sorted stably over all 32 key bits into vid[1] / ord[1], so each
    // voxel's points form one run in input order.  vid[0] / ord[0] and tmp are the sort's scratch.
    struct VoxelSort {
        DeviceBuffer<uint32_t> vid[2], ord[2];
        DeviceBuffer<uint8_t> tmp;
    } sort;
    // room for `cap` points in `sort`; a short buffer is reallocated, so the caller synchronises first
    int reserve_sort(size_t cap);
    // keys -> sort of n float or double [n][3] points (asynchronous; needs reserve_sort(>= n))
    cudaError_t sort_voxels(const void *pts, bool pts_f64, const uint8_t *valid, int64_t n, uint32_t lo, uint32_t hi);
    // room for n per-CTA counts in d_sums / offsets in d_offs (the CTAs of a per-voxel pass, voxel_ctas)
    int ensure_scan(uint32_t n);
    // exclusive scan of the per-CTA counts d_sums -> d_offs, and their total (synchronises)
    cudaError_t scan_total(uint32_t n, uint32_t *total);
    GridQuery all_query(int min_count) const;
    // voxel_block_grid.hpp:828-831: keys in double with the float inverse voxel size
    GridQuery box_query(const double bbox[6], int min_count) const;
    // world AABB of the frustum corners (camera_frustrum.cpp:209-260) -> voxel key bounds (voxel_block_grid.hpp:1340-1345)
    GridQuery frustum_query(const float K[4], int W, int H, const double Tcw[16], float depth_max, float depth_min,
                            int min_count) const;
    // Per-call images of integrate_rgbd, carve and the association, in buffers sized for the largest call so far.
    // Kept apart from `frame`, so a staged frame stays valid across calls made with host images.  A call's buffers
    // are next written by a later call on the same stream, so the growth replay of the call may read them.
    struct InputStage {
        DeviceBuffer<float> depth, filtered;
        DeviceBuffer<uint8_t> rgb, shadow_scratch;
        DeviceBuffer<int32_t> cls, obj;   // class and object (or instance) images (semantic grids)
    } input;
    // The [H][W] images of one call on the device: each non-NULL pointer is read in place if it is device memory, else
    // replaced by its upload into `input` on the stream.  filter_shadow_points: *depth is then replaced by its
    // shadow-filtered copy in input.filtered.  Arguments are checked before anything is uploaded; `fn` names the call
    // in err.
    int stage_input(const char *fn, int H, int W, bool filter_shadow_points, const float **depth,
                    const uint8_t **rgb = nullptr, const int32_t **cls = nullptr, const int32_t **obj = nullptr);

    // Per-frame preparation (b2v_grid_set_frame / b2v_sgrid_set_frame): the rectification maps and the staged images
    // of the last frame, in buffers sized for the largest frame so far.
    struct FrameStage {
        DeviceBuffer<float> mapx, mapy;           // empty: no rectification
        int32_t map_h = 0, map_w = 0, swap_rb = 0;
        DeviceBuffer<uint32_t> raw;               // upload of one host image at a time (4 bytes per pixel)
        DeviceBuffer<float> depth, filtered;
        DeviceBuffer<uint8_t> rgb, shadow_scratch;
        DeviceBuffer<int32_t> cls, inst, obj;     // label images (semantic grids)
        b2v_frame staged{};                       // the last staged frame (all NULL: none)
    } frame;
    int set_rectification(const float *map_x, const float *map_y, int H, int W, int swap_rb);   // synchronises
    // upload once -> widen uint16 depth -> rectify -> shadow filter; *out = frame.staged.  Synchronises.  Arguments
    // are checked before anything is touched.
    int set_frame(const void *depth, bool depth_u16, float depth_scale, const uint8_t *color, const int32_t *cls,
                  const int32_t *inst, int H, int W, bool filter_shadow_points, b2v_frame *out);

    // Frame store (b2v_grid_set_frame_store / b2v_sgrid_set_frame_store): with it on, each successful set_frame packs
    // its staged images into the next slot (launch_grid_frame_pack), one record per pixel: 8 bytes, or 16 with the
    // label images of the semantic grids (frame_labels).  stage_stored unpacks a slot back into `frame`.
    FrameStore frame_store;
    bool frame_labels = false;   // semantic grids: records carry the class and instance images
    enum : uint8_t { kStoredClass = 1, kStoredInstance = 2, kStoredFiltered = 4 };
    std::vector<uint8_t> store_flags;   // per filled slot: which images set_frame staged
    int set_frame_store(int32_t max_frames);   // empties the store (synchronises)
    // set_frame / stage_stored: frame.staged := {}, the frame buffers sized for `pixels` (label buffers with labels);
    // then frame.staged := the staged images and *out := frame.staged
    int reserve_frame(size_t pixels, bool labels);
    void finish_frame(int H, int W, bool filtered, bool cls, bool inst, b2v_frame *out);
    // *out := the b2v_frame set_frame returned for the slot's frame, its images unpacked into `frame`.  A slot the
    // store does not hold changes nothing.  Synchronises.
    int stage_stored(int32_t slot, b2v_frame *out);
};

template <typename MapStorage, typename Replay> int BlockGridCore::resolve(MapStorage map_storage, Replay replay) {
    const int rc = fetch_counters();
    if (rc != B2V_OK) return rc;
    const uint32_t used = h_counters[kBgPool], old = index.pool_capacity;
    if (used <= old || old >= index.capacity) return B2V_OK;
    map_storage(std::min<uint64_t>(index.capacity, std::max<uint64_t>(used, 2ull * old)));
    if (index.pool_capacity > old) {
        growths += 1;
        const int rr = replay(old, index.pool_capacity);
        if (rr != B2V_OK) return rr;
    }
    if (used > index.pool_capacity)   // the storage could not grow far enough
        B2V_CUDA(this, launch_drop_unbacked_slots(table, index.pool_capacity, index.capacity,
                                                  index.counters + kBgError, stream));
    B2V_CUDA(this, cudaStreamSynchronize(stream));
    return B2V_OK;
}

template <typename MapStorage, typename Fill>
int BlockGridCore::upload_blocks(int64_t n, const int32_t *keys4, const BlockArrays &arrays, MapStorage map_storage,
                                 Fill fill) {
    DeviceBuffer<int4> d_keys;
    int rc = insert_keys(n, keys4, &d_keys);
    if (rc == B2V_OK && growable) rc = resolve(map_storage, fill);
    return rc == B2V_OK ? scatter_blocks(n, d_keys.get(), arrays) : rc;
}

// raw uint16 depth -> float32 metres (b2v_prep.cu)
cudaError_t launch_depth_u16_to_f32(const uint16_t *src, float *dst, size_t n, float scale, cudaStream_t stream);

// Frame-store records of the grids (b2v_prep.cu): per pixel {depth bits, r, g, b, flags} (8 bytes), followed with
// labels by {class, instance} (16 bytes).  flags bit 0: the shadow filter set the pixel, i.e. filtered != depth
// bitwise; the filter writes only `m ? -1.0f : d`, so unpack rebuilds filtered = flag ? -1.0f : depth exactly.
// filtered / cls / inst NULL: not packed (unpack: not written).  `rec` is 16-byte aligned.
constexpr size_t grid_record_pitch(size_t pixels, bool labels) {   // bytes per slot: whole 4-pixel groups
    return (pixels + 3) / 4 * 4 * (labels ? 16 : 8);
}
cudaError_t launch_grid_frame_pack(const float *depth, const float *filtered, const uint8_t *rgb, const int32_t *cls,
                                   const int32_t *inst, size_t pixels, bool labels, void *rec, cudaStream_t stream);
cudaError_t launch_grid_frame_unpack(const void *rec, size_t pixels, bool labels, float *depth, float *filtered,
                                     uint8_t *rgb, int32_t *cls, int32_t *inst, cudaStream_t stream);

// filter_shadow_points (pyslam/utilities/depth.py:103-146) on the device; scratch: 64 + 16384 bytes
constexpr size_t kShadowScratchBytes = 64 + 4096 * sizeof(uint32_t);
cudaError_t launch_filter_shadow_points(const float *depth, int H, int W, int dx, int dy, float fill, float *out,
                                        void *scratch, cudaStream_t stream);

// cv2.remap equivalents (bit-exact fixed-point bilinear for 8-bit x3, nearest for 32-bit pixels)
cudaError_t launch_remap_u8c3_linear(const uint8_t *src, int H, int W, const float *mapx, const float *mapy,
                                     uint8_t *dst, int swap_rb, cudaStream_t stream);
cudaError_t launch_remap_b32_nearest(const void *src, int H, int W, const float *mapx, const float *mapy, void *dst,
                                     cudaStream_t stream);
// remap_instance_ids (image_utils.h:69-163): dst[i] = map_obj[k] where map_inst[k] == src[i] (map_inst sorted
// ascending), else -1; n_map == 0 gives -1 everywhere
cudaError_t launch_remap_instance_ids(const int32_t *src, size_t n, const int32_t *map_inst, const int32_t *map_obj,
                                      int n_map, int32_t *dst, cudaStream_t stream);

}  // namespace b2v
