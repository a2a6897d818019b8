// b2v_api.cu — the C ABI of the TSDF volume (include/b2v.h): lifetime, frame staging and stream pipelining, mesh
// and point-cloud extraction, parity hooks; the device storage that grows in place (VmmRange) and the small host
// utilities the voxel grids share.  Host code only; kernels live in b2v_tsdf.cu, b2v_mesh.cu, b2v_shard.cu.  The
// point-average and semantic grids keep their host code beside their kernels (b2v_grid.cu, b2v_semantic.cu).
//
// Frames are enqueued in groups (enqueue_frames): b2v_integrate_batch fuses groups of up to kMaxGroup frames, and a
// single frame is a group of one on the frame-by-frame kernels.  Group g uses group buffer buf = g % kGroupBufs:
//   copy stream:    H2D depth, colour of the group's host frames         -> event ready[buf]
//   alloc stream:   wait ready[buf]; allocate kernel                      -> event galloc[buf]
//   compute stream: wait galloc[buf]; update kernel                       -> event group_done[buf]
// so the upload and allocation of the next groups overlap the update of this one.  Nothing synchronises with
// the host until b2v_synchronize / an inspection call.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/b2v.h"
#include "b2v_internal.h"

using namespace b2v;

namespace b2v {

// Host-side pose algebra, same operation order as the oracle (and -ffp-contract=off on the host
// compiler), so allocation keys agree bit for bit.
void fill_frame_params(FrameParams *p, const double K[4], const double Tcw[16], int H, int W,
                       const VolumeGeometry &g) {
    p->fx = K[0];
    p->fy = K[1];
    p->cx = K[2];
    p->cy = K[3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) p->pose.Rwc[3 * i + j] = Tcw[4 * j + i];
    for (int i = 0; i < 3; ++i)
        p->pose.twc[i] = -((p->pose.Rwc[3 * i + 0] * Tcw[3] + p->pose.Rwc[3 * i + 1] * Tcw[7]) +
                           p->pose.Rwc[3 * i + 2] * Tcw[11]);
    p->tau_d = g.unit_shift > 0 ? g.tau_d : static_cast<double>(g.tau);
    p->unit_len = g.voxel_length * static_cast<double>(kB << g.unit_shift);
    IntPose &E = p->E;
    for (int i = 0; i < 12; ++i) E.E[i] = static_cast<float>(Tcw[i]);
    for (int i = 0; i < 3; ++i) E.Es[i] = E.E[4 * i + 2] * g.vs;  // extrinsic_f * voxel_length_f, column 2
    E.pad = 0.0f;
    IntConsts &I = p->I;
    I.fxf = static_cast<float>(K[0]);
    I.fyf = static_cast<float>(K[1]);
    I.cxf = static_cast<float>(K[2]);
    I.cyf = static_cast<float>(K[3]);
    I.safe_w = static_cast<float>(W) - 0.0001f;
    I.safe_h = static_cast<float>(H) - 0.0001f;
    I.tau = g.tau;
    I.inv_tau = 1.0f / g.tau;
    I.W = W;
    I.pixels = W * H;
    I.tex = nullptr;
    I.lam = nullptr;
    I.tex_pitch = 0;
    p->inv_fx = 1.0f / I.fxf;
    p->inv_fy = 1.0f / I.fyf;
    p->inv_vs = 1.0f / g.vs;  // voxel_block_grid.hpp:6
    p->depth_trunc = g.depth_trunc;
    p->unit_shift = g.unit_shift;
    p->H = H;
    p->W = W;
    p->stride = g.stride;
    p->shard_rank = g.shard_rank;
    p->shard_count = g.shard_count;
    p->group_buf = 0;
}

VolumeConsts volume_consts(const VolumeGeometry &g) {
    VolumeConsts c;
    c.unit_len = g.voxel_length * static_cast<double>(kB << g.unit_shift);
    c.vs = g.vs;
    c.half_vs = g.vs * 0.5f;
    c.unit_shift = g.unit_shift;
    return c;
}

}  // namespace b2v

uint32_t b2v::next_pow2(uint64_t v) {
    uint64_t p = 1;
    while (p < v) p <<= 1;
    return static_cast<uint32_t>(p);
}

bool b2v::is_device_pointer(const void *p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

namespace {
// staging and texel slots: slot buf * kMaxGroup + k holds frame k of the group in group buffer buf
constexpr int kStage = kGroupBufs * kMaxGroup;

// Slot s of a staging buffer, `per_frame` elements per slot at the pitch of the current frame; the buffers are
// reserved for kStage slots of the largest frame so far.  A slot's address thus moves with the frame size.  That is
// safe because enqueue_frames drains the device whenever H x W changes (cudaDeviceSynchronize, then resolve_skipped,
// before it rewrites the lambda image), so no kernel in flight and no pending replay holds a slot address at the old
// pitch.
template <typename T> T *stage_slot(const DeviceBuffer<T> &b, size_t per_frame, int s) {
    return b.get() + per_frame * static_cast<size_t>(s);
}
// texels per slot: the image + the out-of-image texel at index H * W, rounded up to 256 bytes
size_t texel_pitch(size_t pixels) { return (pixels + 32) & ~static_cast<size_t>(31); }
}  // namespace

struct b2v_volume {
    b2v_config cfg{};
    VolumeGeometry geo{};
    cudaStream_t compute = nullptr, copy = nullptr, alloc = nullptr;
    cudaStream_t update_stream = nullptr;  // stream of the most recent call's update kernels (see last_group_done)
    bool overlap = true;                 // allocate(g+1) on its own stream, concurrent with the update of group g
    bool use_tma = true;                 // stage image tiles with TMA when the layout allows it
    bool fuse = true;                    // b2v_integrate_batch fuses groups of up to kMaxGroup frames
    int group_frames = 16;               // frames per fused group (1..kMaxGroup), b2v_set_group_size
    cudaEvent_t input_event = nullptr;   // b2v_set_input_event: readiness of the next integrate call's device inputs
    uint32_t group_id = 0;               // groups enqueued since reset; group g uses group buffer g % kGroupBufs
    int last_group_count = 0;            // frames of the most recent group
    cudaEvent_t ev_in = nullptr;         // input fence recorded on the caller's stream
    cudaEvent_t ev_ready[kGroupBufs] = {}, ev_galloc[kGroupBufs] = {}, ev_group_done[kGroupBufs] = {};
    int64_t prof_frames = 0, prof_int_launches = 0;
    // optional rectification stage (b2v_set_rectification)
    DeviceBuffer<float> d_mapx, d_mapy;
    int rect_H = 0, rect_W = 0, rect_swap = 0;
    DeviceBuffer<float> d_rdepth;    // rectified frames (same slots as the raw staging)
    DeviceBuffer<uint8_t> d_rcolor;
    // TMA descriptors are cached per image address (encoding costs ~1 us of host time each)
    std::unordered_map<uintptr_t, FrameMaps> map_cache;
    int map_H = 0, map_W = 0;
    // raw 16-bit depth input (b2v_integrate_batch_u16): uploaded as is, widened on the device
    DeviceBuffer<uint16_t> d_depth16;   // same slots as d_depth; allocated on first use
    DeviceBuffer<float> d_depth;        // staging of host frames (and of widened uint16 depth), see stage_slot
    DeviceBuffer<uint8_t> d_color;
    DeviceBuffer<Texel> d_tex;      // texel images, written by the allocate kernels and read by the update kernels
    DeviceBuffer<float> d_lambda;   // lambda image of the cached intrinsics, read by the update kernels
    double lam_K[4] = {0, 0, 0, 0};
    int lam_H = 0, lam_W = 0;
    HashTable table{};                   // the kernels' views of the buffers below
    PoolMeta meta{};
    UnitSet units{};                     // group unit sets of the fused allocation, one per group buffer
    DeviceBuffer<uint4> table_mem, unit_entries;
    DeviceBuffer<int4> block_keys;
    DeviceBuffer<uint32_t> counters, group_mask, union_slots, block_flags, unit_list;
    // The pool is one virtual-address reservation for meta.capacity blocks; physical chunks are mapped as it grows
    // (fixed volumes map it whole at create), so the pool address the kernels see never changes.
    bool growable = false;               // max_capacity_blocks > capacity_blocks
    VmmRange pool;
    int64_t growths = 0;
    // update launch of the group in each buffer, kept for the replay of a skipped group
    GroupArgs gargs[kGroupBufs];
    bool gfused[kGroupBufs] = {};
    uint32_t *h_skip = nullptr;          // pinned [kGroupBufs]: counters[kCtrSkipping] after the gate of the buffer's group
    int grid_ctas = 0;
    int sm_count = 0;
    int64_t launches = 0;
    uint32_t *h_counters = nullptr;  // pinned mirror
    std::string err;
    // mesh / point-cloud extraction: mb is the kernels' view of the buffers in `mesh`
    MeshBuffers mb{};
    struct {
        DeviceBuffer<int32_t> nbr, edge_ids, triangles;
        DeviceBuffer<uint8_t> cube;
        DeviceBuffer<uint32_t> edge_mask, local, sums, offs, partials, totals, work;
        DeviceBuffer<double> vertices, colors;
    } mesh;
    int64_t last_nv = 0, last_nt = 0;
    uint32_t *h_totals = nullptr;
    // sharded extraction (b2v_extract_*_with_halo): an unsharded scratch volume holding this volume's blocks at the
    // same pool indices plus the received halo blocks after them, kept between extractions.  The most recent
    // extraction's output lives in it when last_from_halo is set.
    b2v_volume *halo = nullptr;
    bool last_from_halo = false;
    // optional per-kernel timing (b2v_profile_*)
    bool prof_enabled = false;
    std::vector<cudaEvent_t> prof_events;  // quadruples: allocate begin/end, integrate begin/end
    size_t prof_used = 0;
    // frame store (b2v_set_frame_store): the packed texel image of each stored frame, H * W texels per slot
    FrameStore store;
};

// ---- the block pool: virtual memory management entry points of the driver ----

namespace {
struct VmmApi {
    decltype(&cuMemGetAllocationGranularity) granularity;
    decltype(&cuMemAddressReserve) reserve;
    decltype(&cuMemAddressFree) address_free;
    decltype(&cuMemCreate) create;
    decltype(&cuMemRelease) release;
    decltype(&cuMemMap) map;
    decltype(&cuMemUnmap) unmap;
    decltype(&cuMemSetAccess) set_access;
};

const VmmApi *vmm_api() {
    static VmmApi api{};
    static const bool ok = [] {
        auto get = [](const char *name, auto *fn) {
            void *sym = nullptr;
            cudaDriverEntryPointQueryResult st;
            if (cudaGetDriverEntryPoint(name, &sym, cudaEnableDefault, &st) != cudaSuccess ||
                st != cudaDriverEntryPointSuccess || !sym)
                return false;
            *fn = reinterpret_cast<std::remove_pointer_t<decltype(fn)>>(sym);
            return true;
        };
        return get("cuMemGetAllocationGranularity", &api.granularity) && get("cuMemAddressReserve", &api.reserve) &&
               get("cuMemAddressFree", &api.address_free) && get("cuMemCreate", &api.create) &&
               get("cuMemRelease", &api.release) && get("cuMemMap", &api.map) && get("cuMemUnmap", &api.unmap) &&
               get("cuMemSetAccess", &api.set_access);
    }();
    return ok ? &api : nullptr;
}

CUmemAllocationProp pool_prop(int device) {
    CUmemAllocationProp p{};
    p.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    p.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    p.location.id = device;
    return p;
}

bool cu_failed(CUresult r, const char *what, std::string *err) {
    if (r == CUDA_SUCCESS) return false;
    *err = std::string(what) + ": CUresult " + std::to_string(r);
    return true;
}
}  // namespace

bool b2v::vmm_reserve(VmmRange *r, size_t bytes, int device, std::string *err) {
    const VmmApi *api = vmm_api();
    if (!api) {
        *err = "the driver's virtual memory management entry points are unavailable";
        return false;
    }
    r->device = device;
    const CUmemAllocationProp prop = pool_prop(device);
    if (cu_failed(api->granularity(&r->gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM), "cuMemGetAllocationGranularity",
                  err))
        return false;
    const size_t g = r->gran;
    const size_t reserved = (std::max<size_t>(bytes, 1) + g - 1) / g * g;
    if (cu_failed(api->reserve(&r->va, reserved, 0, 0, 0), "cuMemAddressReserve", err)) return false;
    r->reserved = reserved;
    return true;
}

bool b2v::vmm_map(VmmRange *r, size_t bytes, cudaStream_t stream, std::string *err) {
    const size_t g = r->gran;
    const size_t want = std::min(r->reserved, (bytes + g - 1) / g * g);
    if (want <= r->mapped) return true;
    const VmmApi *api = vmm_api();
    const size_t off = r->mapped, len = want - off;
    const CUmemAllocationProp prop = pool_prop(r->device);
    CUmemGenericAllocationHandle h;
    if (cu_failed(api->create(&h, len, &prop, 0), "cuMemCreate", err)) return false;
    const CUresult m = api->map(r->va + off, len, 0, h, 0);
    api->release(h);  // the mapping keeps the memory until it is unmapped
    if (cu_failed(m, "cuMemMap", err)) return false;
    r->chunks.emplace_back(off, len);
    CUmemAccessDesc acc{};
    acc.location = prop.location;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    if (cu_failed(api->set_access(r->va + off, len, &acc, 1), "cuMemSetAccess", err)) return false;
    r->mapped = want;
    const cudaError_t e = cudaMemsetAsync(reinterpret_cast<void *>(r->va + off), 0, len, stream);
    if (e != cudaSuccess) {
        *err = std::string("cudaMemsetAsync: ") + cudaGetErrorString(e);
        return false;
    }
    return true;
}

b2v::VmmRange::~VmmRange() { vmm_release(this); }

void b2v::vmm_release(VmmRange *r) {
    const VmmApi *api = vmm_api();
    if (!api || !r->va) return;
    for (const auto &c : r->chunks) api->unmap(r->va + c.first, c.second);
    api->address_free(r->va, r->reserved);
    r->chunks.clear();
    r->va = 0;
    r->reserved = r->mapped = 0;
}

// ---- frame store ----

b2v::FrameStore::FrameStore() {
    if (const char *e = std::getenv("B2V_FRAME_STORE_MAX_BYTES")) map_limit = std::strtoull(e, nullptr, 10);
}

void b2v::FrameStore::assign(int32_t n_frames, int fH, int fW, size_t fpitch, int device, cudaStream_t stream) {
    if (max == 0 || stopped) return;
    std::string err;   // not the owner's error: a store that cannot grow stops storing, the call goes on
    if (H == 0) {
        if (!vmm_reserve(&range, static_cast<size_t>(max) * fpitch, device, &err)) {
            stopped = true;
            return;
        }
        H = fH;
        W = fW;
        pitch = fpitch;
    }
    if (fH != H || fW != W) return;
    // map the store's first `bytes` bytes; false, with nothing mapped past what was, past map_limit or on failure
    auto map = [&](size_t bytes) {
        const size_t g = range.gran;
        return (bytes + g - 1) / g * g <= map_limit && vmm_map(&range, bytes, stream, &err);
    };
    int32_t n = std::min(n_frames, max - count);
    const size_t need = static_cast<size_t>(count + n) * pitch;
    if (n > 0 && need > range.mapped) {
        const size_t doubled = std::min(range.reserved, 2 * range.mapped);
        if (!(doubled > need && map(doubled)) && !map(need)) {
            stopped = true;
            n = static_cast<int32_t>(std::min<size_t>(n, range.mapped / pitch - count));
        }
    }
    for (int32_t f = 0; f < n; ++f) last[f] = count + f;
}

void b2v::FrameStore::release() {
    vmm_release(&range);
    count = 0;
    H = W = 0;
    pitch = 0;
    stopped = false;
    std::fill(last.begin(), last.end(), -1);
}

// reserve the address range of meta.capacity blocks
static size_t block_bytes(const b2v_volume *v) { return tsdf_block_bytes(v->cfg.color_f64 != 0); }

static int pool_reserve(b2v_volume *v) {
    if (!vmm_reserve(&v->pool, static_cast<size_t>(v->meta.capacity) * block_bytes(v), v->cfg.device, &v->err))
        return B2V_ERR_CUDA;
    v->meta.pool = reinterpret_cast<float *>(v->pool.va);
    return B2V_OK;
}

// map (and zero: allocation relies on a zeroed pool) storage for at least `blocks` blocks, in whole granules, up to
// the reservation; pool_capacity follows
static int pool_map(b2v_volume *v, uint64_t blocks) {
    if (!vmm_map(&v->pool, static_cast<size_t>(blocks) * block_bytes(v), v->compute, &v->err)) return B2V_ERR_CUDA;
    v->meta.pool_capacity = static_cast<uint32_t>(std::min<size_t>(v->meta.capacity, v->pool.mapped / block_bytes(v)));
    return B2V_OK;
}

// growth policy: at least double, at least `need` blocks, at most the maximum
static int pool_grow(b2v_volume *v, uint64_t need) {
    const uint32_t old = v->meta.pool_capacity;
    if (need <= old || old >= v->meta.capacity) return B2V_OK;
    const int rc = pool_map(v, std::min<uint64_t>(v->meta.capacity, std::max<uint64_t>(need, 2ull * old)));
    if (v->meta.pool_capacity > old) v->growths += 1;
    return rc;
}

static int volume_clear_device(b2v_volume *v) {
    const size_t tcap = static_cast<size_t>(v->table.mask) + 1;
    B2V_CUDA(v, cudaMemsetAsync(v->table.entries, 0xFF, tcap * sizeof(uint4), v->compute));
    B2V_CUDA(v, cudaMemsetAsync(v->meta.group_mask, 0, tcap * kGroupBufs * sizeof(uint32_t), v->compute));
    B2V_CUDA(v, cudaMemsetAsync(v->meta.counters, 0, kNumCounters * sizeof(uint32_t), v->compute));
    B2V_CUDA(v, cudaMemsetAsync(v->units.entries, 0, (static_cast<size_t>(v->units.mask) + 1) * kGroupBufs * sizeof(uint4),
                                v->compute));
    return B2V_OK;
}

extern "C" int b2v_version(void) { return 113; }

extern "C" int b2v_selftest_division(int32_t device, uint64_t pairs, uint64_t *bad_reciprocals, uint64_t *bad_quotients) {
    if (cudaSetDevice(device) != cudaSuccess) return B2V_ERR_CUDA;
    DeviceBuffer<unsigned long long> d;
    unsigned long long h[2] = {0, 0};
    cudaError_t e = d.reserve(2);
    if (e == cudaSuccess) e = cudaMemset(d.get(), 0, sizeof(h));
    if (e == cudaSuccess) e = launch_selftest_division(d.get(), pairs, nullptr);
    if (e == cudaSuccess) e = cudaMemcpy(h, d.get(), sizeof(h), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return B2V_ERR_CUDA;
    if (bad_reciprocals) *bad_reciprocals = h[0];
    if (bad_quotients) *bad_quotients = h[1];
    return B2V_OK;
}

extern "C" int b2v_device_sm_count(int32_t device) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) return -1;
    return n;
}

extern "C" const char *b2v_last_error(const b2v_volume *v) { return v ? v->err.c_str() : "null volume"; }

extern "C" int b2v_create(const b2v_config *cfg, b2v_volume **out) {
    if (!cfg || !out) return B2V_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    if (cfg->block_size != B2V_BLOCK_SIZE || !(cfg->voxel_size > 0.0f) || !(cfg->sdf_trunc > 0.0f) ||
        !(cfg->depth_trunc > 0.0f) || cfg->capacity_blocks == 0 || cfg->shard_count < 1 ||
        cfg->shard_rank < 0 || cfg->shard_rank >= cfg->shard_count ||
        (cfg->unit_resolution != 0 && cfg->unit_resolution != 8 && cfg->unit_resolution != 16) ||
        (cfg->color_f64 != 0 && cfg->color_f64 != 1) ||
        (cfg->max_capacity_blocks != 0 &&
         (cfg->max_capacity_blocks < cfg->capacity_blocks || cfg->max_capacity_blocks > (1u << 30))) ||
        static_cast<float>(cfg->voxel_length > 0.0 ? cfg->voxel_length : cfg->voxel_size) != cfg->voxel_size ||
        static_cast<float>(cfg->sdf_trunc_d > 0.0 ? cfg->sdf_trunc_d : cfg->sdf_trunc) != cfg->sdf_trunc)
        return B2V_ERR_INVALID_ARGUMENT;
    // allocate_kernel packs 21 bits per axis inside one frustum
    if (static_cast<double>(cfg->depth_trunc) / (static_cast<double>(cfg->voxel_size) * kB) > 5.0e5)
        return B2V_ERR_UNSUPPORTED;
    b2v_volume *v = new (std::nothrow) b2v_volume();
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    v->cfg = *cfg;
    if (v->cfg.depth_stride < 1) v->cfg.depth_stride = 4;
    if (v->cfg.unit_resolution == 0) v->cfg.unit_resolution = 16;
    if (!(v->cfg.voxel_length > 0.0)) v->cfg.voxel_length = static_cast<double>(cfg->voxel_size);
    if (!(v->cfg.sdf_trunc_d > 0.0)) v->cfg.sdf_trunc_d = static_cast<double>(cfg->sdf_trunc);
    v->geo.vs = cfg->voxel_size;
    v->geo.tau = cfg->sdf_trunc;
    v->geo.depth_trunc = cfg->depth_trunc;
    v->geo.voxel_length = v->cfg.voxel_length;
    v->geo.tau_d = v->cfg.sdf_trunc_d;
    v->geo.unit_shift = v->cfg.unit_resolution == 16 ? 1 : 0;
    v->geo.stride = v->cfg.depth_stride;
    v->geo.shard_rank = cfg->shard_rank;
    v->geo.shard_count = cfg->shard_count;
    *out = v;  // returned even on CUDA failure so the caller can read b2v_last_error and destroy
    B2V_CUDA(v, cudaSetDevice(cfg->device));
    B2V_CUDA(v, cudaStreamCreateWithFlags(&v->compute, cudaStreamNonBlocking));
    B2V_CUDA(v, cudaStreamCreateWithFlags(&v->copy, cudaStreamNonBlocking));
    B2V_CUDA(v, cudaStreamCreateWithFlags(&v->alloc, cudaStreamNonBlocking));
    B2V_CUDA(v, cudaEventCreateWithFlags(&v->ev_in, cudaEventDisableTiming));
    if (const char *e = std::getenv("B2V_OVERLAP")) v->overlap = std::atoi(e) != 0;
    if (const char *e = std::getenv("B2V_TMA")) v->use_tma = std::atoi(e) != 0;
    if (const char *e = std::getenv("B2V_FUSE")) v->fuse = std::atoi(e) != 0;
    if (const char *e = std::getenv("B2V_GROUP")) {
        const int n = std::atoi(e);
        if (n >= 1 && n <= kMaxGroup) v->group_frames = n;
    }
    for (int b = 0; b < kGroupBufs; ++b) {
        B2V_CUDA(v, cudaEventCreateWithFlags(&v->ev_ready[b], cudaEventDisableTiming));
        B2V_CUDA(v, cudaEventCreateWithFlags(&v->ev_galloc[b], cudaEventDisableTiming));
        B2V_CUDA(v, cudaEventCreateWithFlags(&v->ev_group_done[b], cudaEventDisableTiming));
    }
    // the table and everything indexed by slot or pool index are sized for the maximum; only the pool's storage grows
    const uint32_t cap = std::max(cfg->capacity_blocks, cfg->max_capacity_blocks);
    v->growable = cap > cfg->capacity_blocks;
    const uint32_t tcap = next_pow2(static_cast<uint64_t>(cap) * 2);
    v->table.mask = tcap - 1;
    v->meta.capacity = cap;
    B2V_CUDA(v, v->table_mem.reserve(tcap));
    v->table.entries = v->table_mem.get();
    {
        int rc = pool_reserve(v);
        if (rc == B2V_OK) rc = pool_map(v, cfg->capacity_blocks);
        if (rc != B2V_OK) return rc;
        v->meta.pool_capacity = cfg->capacity_blocks;   // the rest of the last granule is used only after a growth
    }
    B2V_CUDA(v, cudaMallocHost(&v->h_skip, kGroupBufs * sizeof(uint32_t)));
    std::memset(v->h_skip, 0, kGroupBufs * sizeof(uint32_t));
    B2V_CUDA(v, v->block_keys.reserve(cap));
    B2V_CUDA(v, v->counters.reserve(kNumCounters));
    B2V_CUDA(v, v->group_mask.reserve(static_cast<size_t>(tcap) * kGroupBufs));
    B2V_CUDA(v, v->union_slots.reserve(static_cast<size_t>(cap) * kGroupBufs));
    B2V_CUDA(v, v->block_flags.reserve(cap));
    v->meta.block_keys = v->block_keys.get();
    v->meta.counters = v->counters.get();
    v->meta.group_mask = v->group_mask.get();
    v->meta.union_slots = v->union_slots.get();
    v->meta.block_flags = v->block_flags.get();
    {
        // Group unit sets: 2^16 entries (1 MB) per group buffer, L2-resident.  The largest union of 32-frame groups
        // on the bench configs is ~2.6 k 16^3 units on C2 (~21 k under decision D1's 8^3 units); units that find no
        // entry take the direct path, exactly.  B2V_GROUP_UNIT_SET (a power of two) overrides the size, for tuning
        // and for tests of that path.
        uint32_t entries = 1u << 16;
        if (const char *e = std::getenv("B2V_GROUP_UNIT_SET")) {
            const long n = std::atol(e);
            if (n >= 1 && n <= (1l << 24) && (n & (n - 1)) == 0) entries = static_cast<uint32_t>(n);
        }
        v->units.mask = entries - 1;
        B2V_CUDA(v, v->unit_entries.reserve(static_cast<size_t>(entries) * kGroupBufs));
        B2V_CUDA(v, v->unit_list.reserve(static_cast<size_t>(entries) * kGroupBufs));
        v->units.entries = v->unit_entries.get();
        v->units.list = v->unit_list.get();
    }
    B2V_CUDA(v, cudaMemsetAsync(v->meta.block_flags, 0, static_cast<size_t>(cap) * sizeof(uint32_t), v->compute));
    B2V_CUDA(v, cudaMallocHost(&v->h_counters, kNumCounters * sizeof(uint32_t)));
    B2V_CUDA(v, cudaMallocHost(&v->h_totals, kNumMeshTotals * sizeof(uint32_t)));
    std::memset(v->h_totals, 0, kNumMeshTotals * sizeof(uint32_t));
    int rc = volume_clear_device(v);
    if (rc != B2V_OK) return rc;
    int sms = 0;
    B2V_CUDA(v, cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cfg->device));
    // persistent grid: exactly one wave of resident CTAs (B2V_INT_CTAS_PER_SM overrides, for tuning)
    int per_sm = integrate_max_resident_ctas_per_sm(cfg->color_f64 != 0);
    if (const char *e = std::getenv("B2V_INT_CTAS_PER_SM")) {
        const int n = std::atoi(e);
        if (n >= 1 && n <= 32) per_sm = n;
    }
    v->grid_ctas = sms * per_sm;
    v->sm_count = sms;
    B2V_CUDA(v, cudaStreamSynchronize(v->compute));
    return B2V_OK;
}

extern "C" int b2v_destroy(b2v_volume *v) {
    if (!v) return B2V_OK;
    b2v_destroy(v->halo);
    cudaSetDevice(v->cfg.device);
    cudaDeviceSynchronize();
    if (v->ev_in) cudaEventDestroy(v->ev_in);
    for (int b = 0; b < kGroupBufs; ++b) {
        if (v->ev_ready[b]) cudaEventDestroy(v->ev_ready[b]);
        if (v->ev_galloc[b]) cudaEventDestroy(v->ev_galloc[b]);
        if (v->ev_group_done[b]) cudaEventDestroy(v->ev_group_done[b]);
    }
    cudaFreeHost(v->h_skip);
    cudaFreeHost(v->h_counters);
    cudaFreeHost(v->h_totals);
    for (cudaEvent_t e : v->prof_events)
        if (e) cudaEventDestroy(e);
    if (v->compute) cudaStreamDestroy(v->compute);
    if (v->copy) cudaStreamDestroy(v->copy);
    if (v->alloc) cudaStreamDestroy(v->alloc);
    delete v;
    return B2V_OK;
}

// Completion of the update of the most recent group, or nullptr when no group was enqueued since create or reset.
// It marks the end of every call's updates so far, whatever their streams: the first group of a call on another
// update stream than the previous call's waits for it (enqueue_frames), and the groups of one call share a stream.
static cudaEvent_t last_group_done(const b2v_volume *v) {
    return v->group_id ? v->ev_group_done[(v->group_id - 1) % kGroupBufs] : nullptr;
}

// waits for the volume's streams and the updates of every call so far, then mirrors the counters
static int drain_and_copy_counters(b2v_volume *v) {
    B2V_CUDA(v, cudaSetDevice(v->cfg.device));
    B2V_CUDA(v, cudaStreamSynchronize(v->copy));
    B2V_CUDA(v, cudaStreamSynchronize(v->alloc));
    if (cudaEvent_t e = last_group_done(v)) B2V_CUDA(v, cudaEventSynchronize(e));
    B2V_CUDA(v, cudaMemcpyAsync(v->h_counters, v->meta.counters, kNumCounters * sizeof(uint32_t),
                                cudaMemcpyDeviceToHost, v->compute));
    B2V_CUDA(v, cudaStreamSynchronize(v->compute));
    return B2V_OK;
}

static int launch_group_update(b2v_volume *v, int buf, cudaStream_t cs) {
    const GroupArgs &a = v->gargs[buf];
    const bool f64 = v->cfg.color_f64 != 0;
    B2V_CUDA(v, v->gfused[buf] ? launch_integrate_group(a, v->table, v->meta, buf, v->grid_ctas, v->sm_count, cs, f64)
                               : launch_integrate(a, v->table, v->meta, buf, v->grid_ctas, cs, f64));
    v->launches += v->gfused[buf] ? 2 : 1;  // update (+ the mask clear of a fused group)
    return B2V_OK;
}

// Growable volumes: if groups were skipped because they were handed pool indices past the storage, map storage for
// every handed-out index and apply the skipped groups in order.  Called at quiescent points (it drains every stream first) and before
// anything the skipped groups still read is overwritten: their texel images, the lambda image.
static int resolve_skipped(b2v_volume *v) {
    int rc = drain_and_copy_counters(v);
    if (rc != B2V_OK || !v->h_counters[kCtrSkipping]) return rc;
    // the allocate kernels handed out the dense indices [0, kCtrPool) below the maximum; map storage for them
    const int grow_rc = pool_grow(v, v->h_counters[kCtrPool]);
    if (v->h_counters[kCtrPool] > v->meta.pool_capacity && v->meta.pool_capacity < v->meta.capacity) {
        B2V_CUDA(v, launch_drop_unbacked_blocks(v->table, v->meta, v->compute));  // the storage could not grow
        v->launches += 1;
    }
    B2V_CUDA(v, cudaMemsetAsync(v->meta.counters + kCtrSkipping, 0, sizeof(uint32_t), v->compute));
    // the skipped groups are a suffix of the enqueued ones, and the enqueue throttle keeps the first of them among the
    // last kGroupBufs groups
    bool skipping = false;
    for (uint32_t g = v->group_id > kGroupBufs ? v->group_id - kGroupBufs : 0; g < v->group_id; ++g) {
        const int buf = static_cast<int>(g % kGroupBufs);
        skipping = skipping || v->h_skip[buf] != 0;
        if (!skipping) continue;
        B2V_CUDA(v, cudaMemcpyAsync(v->meta.counters + group_ctr(buf, kGcUnion), v->meta.counters + kCtrSavedUnion0 + buf,
                                    sizeof(uint32_t), cudaMemcpyDeviceToDevice, v->compute));
        B2V_CUDA(v, cudaMemsetAsync(v->meta.counters + group_ctr(buf, kGcNext), 0, sizeof(uint32_t), v->compute));
        rc = launch_group_update(v, buf, v->compute);
        if (rc != B2V_OK) return rc;
    }
    std::memset(v->h_skip, 0, kGroupBufs * sizeof(uint32_t));
    rc = drain_and_copy_counters(v);
    return rc != B2V_OK ? rc : grow_rc;
}

static int read_counters(b2v_volume *v) {
    const int rc = v->growable ? resolve_skipped(v) : drain_and_copy_counters(v);
    if (rc != B2V_OK) return rc;
    if (v->h_counters[kCtrError]) {
        v->err = (v->h_counters[kCtrError] & 2u) ? "hash table full: raise capacity_blocks"
                                                 : "block pool full: raise capacity_blocks";
        return B2V_ERR_CAPACITY;
    }
    return B2V_OK;
}

static uint32_t block_count(const b2v_volume *v) {
    const uint32_t n = v->h_counters[kCtrPool];
    return n < v->meta.pool_capacity ? n : v->meta.pool_capacity;
}

extern "C" int b2v_reset(b2v_volume *v) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    // pending skipped groups are discarded, not replayed; the grown pool is kept
    int rc = drain_and_copy_counters(v);
    if (rc != B2V_OK) return rc;
    std::memset(v->h_skip, 0, kGroupBufs * sizeof(uint32_t));
    const uint32_t nb = block_count(v);
    B2V_CUDA(v, cudaMemsetAsync(v->meta.pool, 0, static_cast<size_t>(nb) * block_bytes(v),
                                v->compute));
    B2V_CUDA(v, cudaMemsetAsync(v->meta.block_flags, 0, static_cast<size_t>(nb) * sizeof(uint32_t), v->compute));
    rc = volume_clear_device(v);
    if (rc != B2V_OK) return rc;
    v->group_id = 0;
    v->last_group_count = 0;
    v->err.clear();
    B2V_CUDA(v, cudaStreamSynchronize(v->compute));
    return B2V_OK;
}

// Raw staging, texel images and the lambda image for frames of up to `pixels` pixels.
static int ensure_staging(b2v_volume *v, size_t pixels) {
    // the lambda image is reserved last, so it is short whenever a buffer below that holds memory is reallocated
    if (v->d_lambda.size() <= pixels) {
        // the texel and lambda images are read by update kernels on the library's streams and on callers'
        B2V_CUDA(v, cudaDeviceSynchronize());
        if (v->growable) {  // and by the replay of skipped groups
            const int rc = resolve_skipped(v);
            if (rc == B2V_ERR_CUDA) return rc;
        }
        v->lam_H = v->lam_W = 0;
    }
    // the slots of a buffer are contiguous, so the frames of a group (which are contiguous in the caller's arrays)
    // upload with ONE copy per image type
    B2V_CUDA(v, v->d_depth.reserve(pixels * kStage));
    B2V_CUDA(v, v->d_color.reserve(pixels * 3 * kStage));
    const size_t texels = texel_pitch(pixels) * kStage;
    if (texels > v->d_tex.size()) {   // zeroed once, here
        B2V_CUDA(v, v->d_tex.reserve(texels));
        B2V_CUDA(v, cudaMemsetAsync(v->d_tex.get(), 0, texels * sizeof(Texel), v->compute));
        B2V_CUDA(v, cudaStreamSynchronize(v->compute));
    }
    // + the out-of-image element, which launch_lambda sets to kLambdaSentinel at index W * H of each image it writes
    B2V_CUDA(v, v->d_lambda.reserve(pixels + 1));
    return B2V_OK;
}

static int grow_profile_events(b2v_volume *v, size_t need) {
    if (v->prof_used + need > v->prof_events.size()) {
        const size_t old = v->prof_events.size();
        v->prof_events.resize(old + 4 * 256, nullptr);
        for (size_t k = old; k < v->prof_events.size(); ++k) B2V_CUDA(v, cudaEventCreate(&v->prof_events[k]));
    }
    return B2V_OK;
}

// cached TMA descriptors of a frame (keyed by the depth image address; colour address is checked)
static const FrameMaps *frame_maps(b2v_volume *v, const float *d_depth, const uint8_t *d_color, int H, int W) {
    if (!v->use_tma || !tma_tiles_usable(W, v->cfg.depth_stride, d_depth, d_color)) return nullptr;
    if (v->map_H != H || v->map_W != W || v->map_cache.size() > 4096) {
        v->map_cache.clear();
        v->map_H = H;
        v->map_W = W;
    }
    auto it = v->map_cache.find(reinterpret_cast<uintptr_t>(d_depth));
    if (it != v->map_cache.end() && it->second.color_ptr == d_color) return &it->second;
    FrameMaps m;
    if (!encode_frame_maps(&m, d_depth, d_color, H, W, 32)) return nullptr;
    m.color_ptr = d_color;
    auto res = v->map_cache.insert_or_assign(reinterpret_cast<uintptr_t>(d_depth), m);
    return &res.first->second;
}

// raw uint16 staging, one contiguous allocation carved into the same slots as the float staging
static int ensure_staging16(b2v_volume *v, size_t pixels) {
    if (pixels * kStage <= v->d_depth16.size()) return B2V_OK;
    B2V_CUDA(v, cudaStreamSynchronize(v->compute));
    B2V_CUDA(v, cudaStreamSynchronize(v->copy));
    B2V_CUDA(v, cudaStreamSynchronize(v->alloc));
    if (cudaEvent_t e = last_group_done(v)) B2V_CUDA(v, cudaEventSynchronize(e));
    B2V_CUDA(v, v->d_depth16.reserve(pixels * kStage));
    return B2V_OK;
}

extern "C" int b2v_set_rectification(b2v_volume *v, const float *map_x, const float *map_y, int32_t height,
                                     int32_t width, int32_t swap_rb) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    const int rc = read_counters(v);  // drains every stream
    if (rc == B2V_ERR_CUDA) return rc;
    v->d_mapx = {};
    v->d_mapy = {};
    v->d_rdepth = {};
    v->d_rcolor = {};
    v->rect_H = v->rect_W = 0;
    v->rect_swap = swap_rb;
    v->map_cache.clear();
    if (!map_x || !map_y) return B2V_OK;
    if (height <= 0 || width <= 0) {
        v->err = "b2v_set_rectification: bad image size";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    const size_t pixels = static_cast<size_t>(height) * width;
    B2V_CUDA(v, v->d_mapx.reserve(pixels));
    B2V_CUDA(v, v->d_mapy.reserve(pixels));
    B2V_CUDA(v, cudaMemcpy(v->d_mapx.get(), map_x, pixels * sizeof(float), cudaMemcpyHostToDevice));
    B2V_CUDA(v, cudaMemcpy(v->d_mapy.get(), map_y, pixels * sizeof(float), cudaMemcpyHostToDevice));
    B2V_CUDA(v, v->d_rdepth.reserve(pixels * kStage));
    B2V_CUDA(v, v->d_rcolor.reserve(pixels * 3 * kStage));
    v->rect_H = height;
    v->rect_W = width;
    return B2V_OK;
}

extern "C" int b2v_remap(const void *src, int32_t kind, int32_t height, int32_t width, const float *map_x,
                         const float *map_y, void *dst, int32_t swap_rb, int32_t device) {
    if (!src || !dst || !map_x || !map_y || height <= 0 || width <= 0 || (kind != 0 && kind != 1))
        return B2V_ERR_INVALID_ARGUMENT;
    if (cudaSetDevice(device) != cudaSuccess) return B2V_ERR_CUDA;
    const size_t pixels = static_cast<size_t>(height) * width;
    const size_t bytes = pixels * (kind == 0 ? 3 : 4);
    DeviceBuffer<uint8_t> d_src, d_dst;
    DeviceBuffer<float> d_mx, d_my;
    cudaError_t e = d_src.reserve(bytes);
    if (e == cudaSuccess) e = d_dst.reserve(bytes);
    if (e == cudaSuccess) e = d_mx.reserve(pixels);
    if (e == cudaSuccess) e = d_my.reserve(pixels);
    if (e == cudaSuccess) e = cudaMemcpy(d_src.get(), src, bytes, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_mx.get(), map_x, pixels * sizeof(float), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_my.get(), map_y, pixels * sizeof(float), cudaMemcpyHostToDevice);
    if (e == cudaSuccess)
        e = kind == 0 ? launch_remap_u8c3_linear(d_src.get(), height, width, d_mx.get(), d_my.get(), d_dst.get(),
                                                 swap_rb, nullptr)
                      : launch_remap_b32_nearest(d_src.get(), height, width, d_mx.get(), d_my.get(), d_dst.get(),
                                                 nullptr);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(dst, d_dst.get(), bytes, cudaMemcpyDeviceToHost);
    return e == cudaSuccess ? B2V_OK : B2V_ERR_CUDA;
}

// rectify one frame (raw staging or caller device buffers -> rectified slot), on the allocate stream
static int rectify_frame(b2v_volume *v, const float **d_depth, const uint8_t **d_color, int H, int W, int slot,
                         cudaStream_t as) {
    if (!v->d_mapx.get()) return B2V_OK;
    if (H != v->rect_H || W != v->rect_W) {
        v->err = "rectification maps were installed for a different image size";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    const size_t pixels = static_cast<size_t>(H) * W;
    float *depth = stage_slot(v->d_rdepth, pixels, slot);
    uint8_t *color = stage_slot(v->d_rcolor, pixels * 3, slot);
    B2V_CUDA(v, launch_remap_b32_nearest(*d_depth, H, W, v->d_mapx.get(), v->d_mapy.get(), depth, as));
    B2V_CUDA(v, launch_remap_u8c3_linear(*d_color, H, W, v->d_mapx.get(), v->d_mapy.get(), color, v->rect_swap, as));
    *d_depth = depth;
    *d_color = color;
    v->launches += 2;
    return B2V_OK;
}

// Enqueues n_frames frames, contiguous in the caller's arrays, as groups in the group buffers: groups of up to
// group_frames frames on the fused kernels when fusion is on and there are two frames or more, else groups of one
// frame on the frame-by-frame kernels.  depth is float32 metres (u16_scale = 0) or raw uint16 widened on the device
// to float32(depth) * u16_scale (u16_scale > 0).  Consumes the input event of b2v_set_input_event.
// stored != nullptr: the frames are the frame store's slots stored[0..n_frames) (b2v_integrate_stored), at the stored
// frames' size; depth and color are not read.  Each group's texel images are copied from the store into its staging
// slots and the allocate kernels read depth from them (launch_allocate*, from_tex); the update is the same.
static int enqueue_frames(b2v_volume *v, const char *what, int32_t n_frames, const void *depth, float u16_scale,
                          const uint8_t *color, int32_t height, int32_t width, const double K[4], const double *Tcw,
                          void *stream, const int32_t *stored = nullptr) {
    const cudaEvent_t inputs_ready = v->input_event;  // one-shot: consumed by bad arguments too
    v->input_event = nullptr;
    v->store.begin_call(n_frames);  // (also when the call fails)
    // on every return: the slots of frames whose copies were not enqueued are not stored
    struct UnfilledSlots {
        FrameStore &s;
        ~UnfilledSlots() { s.drop_unfilled(); }
    } unfilled{v->store};
    const bool replay = stored != nullptr;
    if (n_frames < 0 || (n_frames > 0 && ((!replay && (!depth || !color)) || !Tcw || !K)) || height <= 0 ||
        width <= 0) {
        v->err = std::string(what) + ": bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    if (n_frames == 0) return B2V_OK;
    if (!(K[0] > 0.0) || !(K[1] > 0.0)) {
        v->err = std::string(what) + ": focal lengths must be positive";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    B2V_CUDA(v, cudaSetDevice(v->cfg.device));
    const size_t pixels = static_cast<size_t>(height) * width;
    // (a replay reads no caller images)
    const bool dev_depth = replay || is_device_pointer(depth), dev_color = replay || is_device_pointer(color);
    if (stream != nullptr && !(dev_depth && dev_color)) {
        v->err = std::string(what) + ": a caller stream requires device image pointers";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    cudaStream_t cs = stream ? static_cast<cudaStream_t>(stream) : v->compute;
    cudaStream_t as = v->overlap ? v->alloc : cs;  // stream of the allocate kernels
    const bool u16 = !replay && u16_scale > 0.0f;
    const float *depth32 = static_cast<const float *>(depth);
    const uint16_t *depth16 = static_cast<const uint16_t *>(depth);
    {
        int rc = ensure_staging(v, pixels);
        if (rc == B2V_OK && u16) rc = ensure_staging16(v, pixels);
        if (rc != B2V_OK) return rc;
        if (!replay) v->store.assign(n_frames, height, width, pixels * sizeof(Texel), v->cfg.device, as);
    }
    // This call's updates touch the blocks the previous call's did, and a block's running average depends on frame
    // order: on another stream they wait for the previous call's last update (on the same stream, stream order does
    // it).  Overlapped allocate kernels run on their own stream and are not held by this wait.
    if (cs != v->update_stream) {
        if (cudaEvent_t e = last_group_done(v)) B2V_CUDA(v, cudaStreamWaitEvent(cs, e, 0));
        v->update_stream = cs;
    }
    if (v->lam_H != height || v->lam_W != width || std::memcmp(v->lam_K, K, sizeof(v->lam_K)) != 0) {
        // the lambda image is read by update kernels of earlier frames that may still run, on the library's streams
        // or on a caller's; new intrinsics are rare, so the whole device is drained before the image is rewritten
        FrameParams P;
        fill_frame_params(&P, K, Tcw, height, width, v->geo);
        B2V_CUDA(v, cudaDeviceSynchronize());
        if (v->growable) {  // a skipped group is replayed with the lambda image it was enqueued with
            const int rc = resolve_skipped(v);
            if (rc == B2V_ERR_CUDA) return rc;
        }
        B2V_CUDA(v, launch_lambda(P, v->d_lambda.get(), as));
        std::memcpy(v->lam_K, K, sizeof(v->lam_K));
        v->lam_H = height;
        v->lam_W = width;
        v->launches += 1;
    }
    const bool fused = v->fuse && n_frames >= 2;
    const int gsz = fused ? std::max(1, std::min(v->group_frames, kMaxGroup)) : 1;
    for (int32_t g0 = 0; g0 < n_frames; g0 += gsz) {
        const int count = std::min<int32_t>(gsz, n_frames - g0);
        const int buf = static_cast<int>(v->group_id % kGroupBufs);
        const int s0 = buf * kMaxGroup;  // the buffer's staging and texel slots
        // growable volumes: the group that last used this buffer may have been skipped, and its replay needs the
        // buffer's state; the host waits for that group (so it runs at most kGroupBufs groups ahead) and resolves first
        if (v->growable) {
            B2V_CUDA(v, cudaEventSynchronize(v->ev_group_done[buf]));
            if (v->h_skip[buf]) {
                const int rc = resolve_skipped(v);
                if (rc == B2V_ERR_CUDA) return rc;
            }
            v->h_skip[buf] = 0;
        }
        // the group buffer (masks, union list, counters, texel images) was last used by group id - kGroupBufs
        B2V_CUDA(v, cudaStreamWaitEvent(as, v->ev_group_done[buf], 0));
        B2V_CUDA(v, cudaMemsetAsync(v->meta.counters + group_ctr(buf, 0), 0, kGroupCtrStride * sizeof(uint32_t), as));
        if (g0 == 0 && !replay && (dev_depth || dev_color)) {
            // one input fence per call: by default everything enqueued on the caller's stream so far (the inputs'
            // producers, earlier frames) happens before the allocate kernels.  A caller that knows better
            // (b2v_set_input_event: "the inputs are ready when this event fires") keeps the allocate kernels of this
            // call from also waiting for the update kernels of the previous one.  The counter memset above does not
            // read the inputs, so it stays off that path.  Host frames are ordered by their uploads.
            if (inputs_ready) {
                B2V_CUDA(v, cudaStreamWaitEvent(as, inputs_ready, 0));
            } else if (v->overlap) {
                B2V_CUDA(v, cudaEventRecord(v->ev_in, cs));
                B2V_CUDA(v, cudaStreamWaitEvent(as, v->ev_in, 0));
            }
        }
        if (!dev_depth || !dev_color) {
            // the raw staging slots of this buffer were consumed by the allocate launch of group id - kGroupBufs;
            // the group's frames are contiguous on both sides: one H2D copy per image type
            B2V_CUDA(v, cudaStreamWaitEvent(v->copy, v->ev_galloc[buf], 0));
            if (!dev_depth && u16)
                B2V_CUDA(v, cudaMemcpyAsync(stage_slot(v->d_depth16, pixels, s0), depth16 + pixels * g0,
                                            pixels * sizeof(uint16_t) * count, cudaMemcpyHostToDevice, v->copy));
            else if (!dev_depth)
                B2V_CUDA(v, cudaMemcpyAsync(stage_slot(v->d_depth, pixels, s0), depth32 + pixels * g0,
                                            pixels * sizeof(float) * count, cudaMemcpyHostToDevice, v->copy));
            if (!dev_color)
                B2V_CUDA(v, cudaMemcpyAsync(stage_slot(v->d_color, pixels * 3, s0), color + pixels * 3 * g0,
                                            pixels * 3 * count, cudaMemcpyHostToDevice, v->copy));
            B2V_CUDA(v, cudaEventRecord(v->ev_ready[buf], v->copy));
            B2V_CUDA(v, cudaStreamWaitEvent(as, v->ev_ready[buf], 0));
        }
        if (u16) {  // widen the group's raw depth into its (contiguous) float staging slots in one launch
            const uint16_t *src = dev_depth ? depth16 + pixels * g0 : stage_slot(v->d_depth16, pixels, s0);
            B2V_CUDA(v, launch_depth_u16_to_f32(src, stage_slot(v->d_depth, pixels, s0), pixels * count,
                                                u16_scale, as));
            v->launches += 1;
        }
        static thread_local GroupAllocArgs aargs;  // ~15 KB: keep it off the stack
        GroupArgs &args = v->gargs[buf];
        std::memset(&args, 0, sizeof(args));
        v->gfused[buf] = fused;
        args.V = volume_consts(v->geo);
        args.count = aargs.count = count;
        aargs.use_tma = 1;
        for (int k = 0; k < count; ++k) {
            const size_t f = static_cast<size_t>(g0 + k);
            // (widened) staging
            const float *d_depth = nullptr;
            const uint8_t *d_color = nullptr;
            Texel *tex = stage_slot(v->d_tex, texel_pitch(pixels), s0 + k);
            if (replay) {  // the gather: the stored texel image into the frame's staging slot
                B2V_CUDA(v, cudaMemcpyAsync(tex, v->store.slot(stored[f]), pixels * sizeof(Texel),
                                            cudaMemcpyDeviceToDevice, as));
            } else {
                d_depth = dev_depth && !u16 ? depth32 + pixels * f : stage_slot(v->d_depth, pixels, s0 + k);
                d_color = dev_color ? color + pixels * 3 * f : stage_slot(v->d_color, pixels * 3, s0 + k);
                const int rc = rectify_frame(v, &d_depth, &d_color, height, width, s0 + k, as);
                if (rc != B2V_OK) return rc;
            }
            FrameParams P;
            fill_frame_params(&P, K, Tcw + 16 * f, height, width, v->geo);
            P.group_buf = buf;
            if (k == 0) {  // the update constants of frame 0 serve the group: one set of intrinsics per call
                P.I.tex = tex;
                P.I.lam = v->d_lambda.get();
                P.I.tex_pitch = static_cast<int64_t>(texel_pitch(pixels));
                args.C = P.I;
                aargs.P = P;
            }
            aargs.pose[k] = P.pose;
            aargs.depth[k] = d_depth;
            aargs.color[k] = d_color;
            aargs.tex[k] = tex;
            const FrameMaps *fm = replay ? nullptr : frame_maps(v, d_depth, d_color, height, width);
            if (fm) aargs.maps[k] = *fm; else aargs.use_tma = 0;
            args.f[k] = P.E;
        }
        cudaEvent_t *pe = nullptr;
        if (v->prof_enabled) {
            const int rc = grow_profile_events(v, 4);
            if (rc != B2V_OK) return rc;
            pe = &v->prof_events[v->prof_used];
            v->prof_used += 4;
            v->prof_frames += count;
            v->prof_int_launches += 1;
            B2V_CUDA(v, cudaEventRecord(pe[0], as));
        }
        aargs.units = v->units;
        B2V_CUDA(v, fused ? launch_allocate_group(aargs, v->table, v->meta, v->sm_count, as, replay)
                          : launch_allocate(aargs, v->table, v->meta, as, replay));
        if (pe) B2V_CUDA(v, cudaEventRecord(pe[1], as));
        B2V_CUDA(v, cudaEventRecord(v->ev_galloc[buf], as));
        v->launches += fused ? 2 : 1;  // (+ the expand kernel of a fused group)
        if (!replay) {
            // the frame store: copy the packed texel images of the group's stored frames (mapped by
            // FrameStore::assign) on the allocate stream, after the pack and before the next group in this buffer
            // overwrites the staging slots (its allocate kernels wait on this stream).  Enqueued after ev_galloc: with
            // overlap on, the update does not wait for the copies; with it off they share its stream.
            for (int k = 0; k < count; ++k) {
                const int32_t slot = v->store.last[g0 + k];
                if (slot < 0) continue;
                B2V_CUDA(v, cudaMemcpyAsync(v->store.slot(slot), aargs.tex[k], pixels * sizeof(Texel),
                                            cudaMemcpyDeviceToDevice, as));
                v->store.filled(slot);
            }
        }
        if (v->overlap) B2V_CUDA(v, cudaStreamWaitEvent(cs, v->ev_galloc[buf], 0));
        if (v->growable && v->meta.pool_capacity < v->meta.capacity) {
            // in group order on one stream, each after its own allocation: the first group skipped is the first that
            // overflowed, and every later one is skipped too, which keeps each block's frame order for the replay
            B2V_CUDA(v, launch_group_gate(v->meta, buf, cs));
            B2V_CUDA(v, cudaMemcpyAsync(v->h_skip + buf, v->meta.counters + kCtrSkipping, sizeof(uint32_t),
                                        cudaMemcpyDeviceToHost, cs));
            v->launches += 1;
        }
        if (pe) B2V_CUDA(v, cudaEventRecord(pe[2], cs));
        {
            const int rc = launch_group_update(v, buf, cs);
            if (rc != B2V_OK) return rc;
        }
        if (pe) B2V_CUDA(v, cudaEventRecord(pe[3], cs));
        B2V_CUDA(v, cudaEventRecord(v->ev_group_done[buf], cs));
        v->last_group_count = count;
        v->group_id += 1;
    }
    return B2V_OK;
}

extern "C" int b2v_integrate_batch(b2v_volume *v, int32_t n_frames, const float *depth,
                                   const uint8_t *color, int32_t height, int32_t width,
                                   const double K[4], const double *Tcw, void *stream) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    return enqueue_frames(v, "b2v_integrate_batch", n_frames, depth, 0.0f, color, height, width, K, Tcw, stream);
}

// Raw 16-bit depth (e.g. TUM / ScanNet PNGs): uploaded as uint16 (2 instead of 4 bytes per pixel over PCIe) and
// widened on the device to float(u16) * depth_scale in float32 - the value numpy's
// `depth.astype(np.float32) * depth_factor` produces (volumetric_integrator_base.py:1008-1015).
extern "C" int b2v_integrate_batch_u16(b2v_volume *v, int32_t n_frames, const uint16_t *depth, float depth_scale,
                                       const uint8_t *color, int32_t height, int32_t width, const double K[4],
                                       const double *Tcw, void *stream) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    if (!(depth_scale > 0.0f)) {
        v->err = "b2v_integrate_batch_u16: depth_scale must be positive";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    return enqueue_frames(v, "b2v_integrate_batch_u16", n_frames, depth, depth_scale, color, height, width, K, Tcw,
                          stream);
}

// ---- frame store ----

// empties the store and releases its memory, after every call that may still read or write it
static int frame_store_release(b2v_volume *v) {
    B2V_CUDA(v, cudaSetDevice(v->cfg.device));
    B2V_CUDA(v, cudaDeviceSynchronize());   // replays gather on the caller's stream when overlap is off
    v->store.release();
    return B2V_OK;
}

extern "C" int b2v_set_frame_store(b2v_volume *v, int32_t max_frames) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    if (max_frames < 0) {
        v->err = "b2v_set_frame_store: max_frames must be >= 0";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    const int rc = frame_store_release(v);
    if (rc != B2V_OK) return rc;
    v->store.max = max_frames;
    return B2V_OK;
}

extern "C" int b2v_frame_store_clear(b2v_volume *v) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    return frame_store_release(v);
}

extern "C" int b2v_frame_store_last(b2v_volume *v, int32_t *slots, int32_t n) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    if (n != static_cast<int32_t>(v->store.last.size()) || (n > 0 && !slots)) {
        v->err = "b2v_frame_store_last: n must be the frame count of the most recent integrate call";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    std::copy(v->store.last.begin(), v->store.last.end(), slots);
    return B2V_OK;
}

extern "C" int b2v_frame_store_stats(b2v_volume *v, int64_t *frames, int64_t *bytes) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    if (frames) *frames = v->store.count;
    if (bytes) *bytes = static_cast<int64_t>(v->store.range.mapped);
    return B2V_OK;
}

extern "C" int b2v_integrate_stored(b2v_volume *v, int32_t n_frames, const int32_t *slots, const double K[4],
                                    const double *Tcw, void *stream) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    v->store.begin_call(n_frames);
    if (n_frames > 0 && !slots) {
        v->err = "b2v_integrate_stored: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    for (int32_t f = 0; f < n_frames; ++f)
        if (!v->store.holds(slots[f])) {
            v->err = "b2v_integrate_stored: slot " + std::to_string(slots[f]) + " holds no frame (the store holds " +
                     std::to_string(v->store.count) + ")";
            return B2V_ERR_INVALID_ARGUMENT;
        }
    return enqueue_frames(v, "b2v_integrate_stored", n_frames, nullptr, 0.0f, nullptr, std::max(v->store.H, 1),
                          std::max(v->store.W, 1), K, Tcw, stream, slots);
}

extern "C" int b2v_set_input_event(b2v_volume *v, void *event) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    v->input_event = static_cast<cudaEvent_t>(event);
    return B2V_OK;
}

extern "C" int b2v_set_group_size(b2v_volume *v, int32_t frames) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    if (frames < 1 || frames > kMaxGroup) {
        v->err = "b2v_set_group_size: 1..32 frames";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    const int rc = read_counters(v);
    if (rc == B2V_ERR_CUDA) return rc;
    v->group_frames = frames;
    return B2V_OK;
}

extern "C" int b2v_set_fusion(b2v_volume *v, int32_t enable) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    const int rc = read_counters(v);
    if (rc == B2V_ERR_CUDA) return rc;
    v->fuse = enable != 0;
    return B2V_OK;
}

extern "C" int b2v_synchronize(b2v_volume *v) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    return read_counters(v);
}

extern "C" int b2v_capacity(b2v_volume *v, int64_t *capacity_blocks, int64_t *growths) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    const int rc = read_counters(v);
    if (rc == B2V_ERR_CUDA) return rc;
    if (capacity_blocks) *capacity_blocks = v->meta.pool_capacity;
    if (growths) *growths = v->growths;
    return rc;
}

extern "C" int64_t b2v_num_blocks(b2v_volume *v) {
    if (!v) return -1;
    const int rc = read_counters(v);
    if (rc == B2V_ERR_CUDA) return -1;
    return block_count(v);
}

extern "C" int b2v_last_frame_stats(b2v_volume *v, int64_t *touched_blocks, int64_t *new_blocks) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    const int rc = read_counters(v);
    if (rc == B2V_ERR_CUDA) return rc;
    const int buf = static_cast<int>((v->group_id - 1) % kGroupBufs);  // the most recent group
    // touched: by the group's last frame; new: allocated by the whole group
    if (touched_blocks)
        *touched_blocks = v->group_id ? v->h_counters[group_ctr(buf, kGcTouched0) + v->last_group_count - 1] : 0;
    if (new_blocks) *new_blocks = v->group_id ? v->h_counters[group_ctr(buf, kGcNew)] : 0;
    return rc;
}

extern "C" int b2v_set_overlap(b2v_volume *v, int32_t enable) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    const int rc = read_counters(v);  // drains every stream first
    if (rc == B2V_ERR_CUDA) return rc;
    v->overlap = enable != 0;
    return B2V_OK;
}

extern "C" int b2v_profile_enable(b2v_volume *v, int32_t enable) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    v->prof_enabled = enable != 0;
    v->prof_used = 0;
    v->prof_frames = 0;
    v->prof_int_launches = 0;
    return B2V_OK;
}

extern "C" int b2v_profile_read(b2v_volume *v, double *allocate_ms, double *integrate_ms, int64_t *frames,
                                int64_t *integrate_launches) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    B2V_CUDA(v, cudaSetDevice(v->cfg.device));
    double a = 0.0, b = 0.0;
    if (std::getenv("B2V_DEBUG_TIMELINE") && v->prof_used >= 4) {  // debug: event times relative to the first
        for (size_t k = 0; k + 3 < v->prof_used && k < 4 * 12; k += 4) {
            float t[4];
            for (int j = 0; j < 4; ++j) {
                cudaEventSynchronize(v->prof_events[k + j]);
                cudaEventElapsedTime(&t[j], v->prof_events[0], v->prof_events[k + j]);
            }
            std::fprintf(stderr, "[b2v timeline] launch %zu: alloc %.1f..%.1f us  integrate %.1f..%.1f us\n", k / 4,
                         1e3 * t[0], 1e3 * t[1], 1e3 * t[2], 1e3 * t[3]);
        }
    }
    for (size_t k = 0; k + 3 < v->prof_used; k += 4) {
        B2V_CUDA(v, cudaEventSynchronize(v->prof_events[k + 1]));
        B2V_CUDA(v, cudaEventSynchronize(v->prof_events[k + 3]));
        float ms = 0.0f;
        B2V_CUDA(v, cudaEventElapsedTime(&ms, v->prof_events[k], v->prof_events[k + 1]));
        a += ms;
        B2V_CUDA(v, cudaEventElapsedTime(&ms, v->prof_events[k + 2], v->prof_events[k + 3]));
        b += ms;
    }
    if (allocate_ms) *allocate_ms = a;
    if (integrate_ms) *integrate_ms = b;
    if (frames) *frames = v->prof_frames;
    if (integrate_launches) *integrate_launches = v->prof_int_launches;
    v->prof_used = 0;
    v->prof_frames = 0;
    v->prof_int_launches = 0;
    return B2V_OK;
}

extern "C" int b2v_counters(b2v_volume *v, int64_t *block_updates, int64_t *kernel_launches,
                            int64_t *block_visits) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    const int rc = read_counters(v);
    if (rc == B2V_ERR_CUDA) return rc;
    if (block_updates)
        *block_updates = static_cast<int64_t>(static_cast<uint64_t>(v->h_counters[kCtrUpdatesLo]) |
                                              (static_cast<uint64_t>(v->h_counters[kCtrUpdatesHi]) << 32));
    if (kernel_launches) *kernel_launches = v->launches;
    if (block_visits)
        *block_visits = static_cast<int64_t>(static_cast<uint64_t>(v->h_counters[kCtrVisitsLo]) |
                                             (static_cast<uint64_t>(v->h_counters[kCtrVisitsHi]) << 32));
    return rc;
}

// The blocks cross the ABI in the pool's own layout: keys int4 {x, y, z, 0}, voxels nb blocks of TsdfBlock<TC>.
extern "C" int64_t b2v_export_blocks(b2v_volume *v, int32_t *keys4, float *voxels, int64_t max_blocks) {
    if (!v) return -1;
    if (read_counters(v) == B2V_ERR_CUDA) return -1;
    const uint32_t nb = block_count(v);
    if (!keys4 && !voxels) return nb;
    if (static_cast<int64_t>(nb) > max_blocks) {
        v->err = "b2v_export_blocks: destination too small";
        return -1;
    }
    if (nb == 0) return 0;
    cudaError_t e = cudaSuccess;
    if (keys4) e = cudaMemcpyAsync(keys4, v->meta.block_keys, nb * sizeof(int4), cudaMemcpyDefault, v->compute);
    if (e == cudaSuccess && voxels)
        e = cudaMemcpyAsync(voxels, v->meta.pool, static_cast<size_t>(nb) * block_bytes(v),
                            cudaMemcpyDefault, v->compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(v->compute);
    if (e != cudaSuccess) {
        v->err = std::string("b2v_export_blocks: ") + cudaGetErrorString(e);
        return -1;
    }
    return nb;
}

// growable volumes: before n blocks are uploaded (new or not), storage for all of them after the current ones
static int grow_for_blocks(b2v_volume *v, int64_t n_blocks) {
    if (!v->growable) return B2V_OK;
    const int rc = read_counters(v);
    if (rc == B2V_ERR_CUDA) return rc;
    return pool_grow(v, static_cast<uint64_t>(v->h_counters[kCtrPool]) + static_cast<uint64_t>(n_blocks));
}

extern "C" int b2v_upload_blocks(b2v_volume *v, int64_t n_blocks, const int32_t *keys4, const float *voxels) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    if (n_blocks < 0 || (n_blocks > 0 && (!keys4 || !voxels))) {
        v->err = "b2v_upload_blocks: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    if (n_blocks == 0) return B2V_OK;
    B2V_CUDA(v, cudaSetDevice(v->cfg.device));
    const size_t n = static_cast<size_t>(n_blocks);
    // device arrays are read in place; host ones are staged on the compute stream
    const int4 *d_keys = reinterpret_cast<const int4 *>(keys4);
    const float *d_vox = voxels;
    DeviceBuffer<int4> k_stage;
    DeviceBuffer<float> v_stage;
    DeviceBuffer<uint32_t> d_i;
    cudaError_t e = d_i.reserve(n);
    if (e == cudaSuccess && !is_device_pointer(keys4)) {
        e = k_stage.reserve(n);
        if (e == cudaSuccess) e = cudaMemcpyAsync(k_stage.get(), keys4, n * sizeof(int4), cudaMemcpyHostToDevice, v->compute);
        d_keys = k_stage.get();
    }
    if (e == cudaSuccess && !is_device_pointer(voxels)) {
        e = v_stage.reserve(n * (block_bytes(v) / sizeof(float)));
        if (e == cudaSuccess)
            e = cudaMemcpyAsync(v_stage.get(), voxels, n * block_bytes(v), cudaMemcpyHostToDevice,
                                v->compute);
        d_vox = v_stage.get();
    }
    // the weights are checked before the pool grows or any block is written: a rejected upload leaves the volume as
    // it was (d_i's first element counts the bad weights)
    uint32_t bad = 0;
    if (e == cudaSuccess) e = cudaMemsetAsync(d_i.get(), 0, sizeof(uint32_t), v->compute);
    if (e == cudaSuccess) e = launch_upload_check(d_vox, static_cast<uint32_t>(n), d_i.get(), v->compute, v->cfg.color_f64 != 0);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&bad, d_i.get(), sizeof(uint32_t), cudaMemcpyDeviceToHost, v->compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(v->compute);
    if (e != cudaSuccess) {
        v->err = std::string("b2v_upload_blocks: ") + cudaGetErrorString(e);
        return B2V_ERR_CUDA;
    }
    if (bad) {
        v->err = "b2v_upload_blocks: " + std::to_string(bad) + " voxel weights outside [0, 2^24]; nothing was uploaded";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    {
        const int rc = grow_for_blocks(v, n_blocks);
        if (rc == B2V_ERR_CUDA) return rc;
    }
    if (e == cudaSuccess)
        e = launch_upload_blocks(d_keys, d_vox, static_cast<uint32_t>(n), d_i.get(), v->table, v->meta, v->compute,
                                 v->cfg.color_f64 != 0);
    if (e == cudaSuccess) e = cudaStreamSynchronize(v->compute);
    v->launches += 2;
    if (e != cudaSuccess) {
        v->err = std::string("b2v_upload_blocks: ") + cudaGetErrorString(e);
        return B2V_ERR_CUDA;
    }
    return read_counters(v);
}

extern "C" int64_t b2v_last_touched_keys(b2v_volume *v, int32_t *keys4, int64_t max_keys) {
    if (!v) return -1;
    if (read_counters(v) == B2V_ERR_CUDA) return -1;
    if (v->group_id == 0) return 0;
    const int buf = static_cast<int>((v->group_id - 1) % kGroupBufs);  // the most recent group's touched blocks
    uint32_t n = v->h_counters[group_ctr(buf, kGcUnion)];
    if (n > v->meta.capacity) n = v->meta.capacity;
    if (!keys4) return n;
    if (static_cast<int64_t>(n) > max_keys) n = static_cast<uint32_t>(max_keys);
    if (n == 0) return 0;
    DeviceBuffer<int4> d_k;
    if (d_k.reserve(n) != cudaSuccess) return -1;
    const uint32_t *list = v->meta.union_slots + static_cast<size_t>(buf) * v->meta.capacity;
    cudaError_t e = launch_gather_active_keys(v->table, list, n, d_k.get(), v->compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(v->compute);
    if (e == cudaSuccess) e = cudaMemcpy(keys4, d_k.get(), n * sizeof(int4), cudaMemcpyDeviceToHost);
    v->launches += 1;
    if (e != cudaSuccess) return -1;
    return n;
}

extern "C" int b2v_block_key_hashes(const int32_t *keys4, int64_t n, uint64_t *hashes) {
    if (n < 0 || (n > 0 && (!keys4 || !hashes))) return B2V_ERR_INVALID_ARGUMENT;
    for (int64_t i = 0; i < n; ++i) hashes[i] = block_key_hash(keys4[4 * i], keys4[4 * i + 1], keys4[4 * i + 2]);
    return B2V_OK;
}

// ---- mesh / point cloud ---------------------------------------------------------------------

// per-block scratch of the extraction for nb blocks
static int ensure_mesh_scratch(b2v_volume *v, uint32_t nb) {
    const size_t n = nb;
    auto &m = v->mesh;
    B2V_CUDA(v, m.totals.reserve(kNumMeshTotals));
    B2V_CUDA(v, m.nbr.reserve(n * 8));
    B2V_CUDA(v, m.cube.reserve(n * kVox));
    B2V_CUDA(v, m.edge_mask.reserve(n * (kVox / 4)));
    B2V_CUDA(v, m.local.reserve(n * kVox));
    B2V_CUDA(v, m.sums.reserve(n * 2));
    B2V_CUDA(v, m.offs.reserve(n * 2));
    B2V_CUDA(v, m.partials.reserve(2 * ((n + 1023) / 1024)));
    B2V_CUDA(v, m.work.reserve(n * 4));
    return B2V_OK;
}

// the kernels' view of v->mesh for nb blocks
static MeshBuffers mesh_view(const b2v_volume *v, uint32_t nb) {
    const auto &m = v->mesh;
    return MeshBuffers{nb, m.nbr.get(), m.cube.get(), m.edge_mask.get(), m.local.get(), m.sums.get(),
                       m.offs.get(), m.partials.get(), m.totals.get(), m.work.get(), m.vertices.get(),
                       m.colors.get(), m.edge_ids.get(), m.triangles.get()};
}

static int extract_common(b2v_volume *v, bool mesh, int64_t *n_vertices, int64_t *n_triangles) {
    int rc = read_counters(v);
    if (rc == B2V_ERR_CUDA) return rc;
    const uint32_t nb = block_count(v);
    rc = ensure_mesh_scratch(v, nb);
    if (rc != B2V_OK) return rc;
    v->mb = mesh_view(v, nb);
    v->last_from_halo = false;
    cudaStream_t cs = v->compute;
    const int sms = v->sm_count;
    if (mesh) {
        B2V_CUDA(v, launch_mesh_classify(v->table, v->meta, v->mb, sms, cs, v->cfg.color_f64 != 0));
    } else {
        B2V_CUDA(v, launch_point_masks(v->table, v->meta, v->mb, sms, cs, v->cfg.color_f64 != 0));
    }
    B2V_CUDA(v, launch_mesh_scan(v->mb, sms, cs));
    B2V_CUDA(v, cudaMemcpyAsync(v->h_totals, v->mb.totals, kNumMeshTotals * sizeof(uint32_t), cudaMemcpyDeviceToHost, cs));
    B2V_CUDA(v, cudaStreamSynchronize(cs));
    const size_t nv = v->h_totals[kMtVertices], nt = v->h_totals[kMtTriangles];
    B2V_CUDA(v, v->mesh.vertices.reserve(nv * 3));
    B2V_CUDA(v, v->mesh.colors.reserve(nv * 3));
    B2V_CUDA(v, v->mesh.edge_ids.reserve(nv * 4));
    B2V_CUDA(v, v->mesh.triangles.reserve(nt * 3));
    v->mb = mesh_view(v, nb);
    B2V_CUDA(v, launch_mesh_vertices(v->meta, v->mb, v->geo.voxel_length, v->geo.unit_shift, !mesh, v->h_totals[kMtVertexBlocks], cs,
                                     v->cfg.color_f64 != 0));
    if (mesh) B2V_CUDA(v, launch_mesh_triangles(v->mb, v->h_totals[kMtTriangleBlocks], cs));
    B2V_CUDA(v, cudaStreamSynchronize(cs));
    v->launches += mesh ? 6 : 5;
    v->last_nv = static_cast<int64_t>(nv);
    v->last_nt = mesh ? static_cast<int64_t>(nt) : 0;
    if (n_vertices) *n_vertices = v->last_nv;
    if (n_triangles) *n_triangles = v->last_nt;
    return rc;
}

extern "C" int b2v_last_mesh_stats(b2v_volume *v, int64_t stats[5]) {
    if (!v || !stats) return B2V_ERR_INVALID_ARGUMENT;
    if (v->last_from_halo && v->halo) return b2v_last_mesh_stats(v->halo, stats);
    stats[0] = v->mb.n_blocks;
    stats[1] = v->h_totals[kMtCandidates];
    stats[2] = v->h_totals[kMtTiles];
    stats[3] = v->h_totals[kMtVertexBlocks];
    stats[4] = v->h_totals[kMtTriangleBlocks];
    return B2V_OK;
}

extern "C" int b2v_extract_mesh(b2v_volume *v, int64_t *n_vertices, int64_t *n_triangles) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    return extract_common(v, true, n_vertices, n_triangles);
}

extern "C" int b2v_copy_mesh(b2v_volume *v, double *vertices, double *colors, int32_t *edge_ids,
                             int32_t *triangles) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    if (v->last_from_halo && v->halo) {
        const int rc = b2v_copy_mesh(v->halo, vertices, colors, edge_ids, triangles);
        if (rc != B2V_OK) v->err = v->halo->err;
        return rc;
    }
    const size_t nv = static_cast<size_t>(v->last_nv), nt = static_cast<size_t>(v->last_nt);
    if (vertices && nv) B2V_CUDA(v, cudaMemcpy(vertices, v->mb.vertices, nv * 3 * sizeof(double), cudaMemcpyDeviceToHost));
    if (colors && nv) B2V_CUDA(v, cudaMemcpy(colors, v->mb.colors, nv * 3 * sizeof(double), cudaMemcpyDeviceToHost));
    if (edge_ids && nv) B2V_CUDA(v, cudaMemcpy(edge_ids, v->mb.edge_ids, nv * 4 * sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (triangles && nt) B2V_CUDA(v, cudaMemcpy(triangles, v->mb.triangles, nt * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return B2V_OK;
}

extern "C" int b2v_extract_points(b2v_volume *v, int64_t *n_points) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    return extract_common(v, false, n_points, nullptr);
}

// ---- sharded extraction: face-halo exchange (b2v_shard.cu) --------------------------------------------------------

extern "C" int b2v_export_halo_device(b2v_volume *v, int32_t world, int64_t *records, int64_t *payload_voxels,
                                      int32_t *d_headers, float *d_payload, int64_t max_records,
                                      int64_t max_payload_voxels) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    if (world < 1 || !records || !payload_voxels || ((d_headers == nullptr) != (d_payload == nullptr))) {
        v->err = "b2v_export_halo_device: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    const int rc = read_counters(v);
    if (rc == B2V_ERR_CUDA) return rc;
    B2V_CUDA(v, cudaSetDevice(v->cfg.device));
    const uint32_t nb = block_count(v);
    for (int r = 0; r < world; ++r) records[r] = payload_voxels[r] = 0;
    if (nb == 0 || world == 1) return B2V_OK;
    const uint64_t n = static_cast<uint64_t>(world) * nb;
    if (n >= (1ull << 31)) {
        v->err = "b2v_export_halo_device: world size x blocks must stay below 2^31";
        return B2V_ERR_UNSUPPORTED;
    }
    const uint64_t chunks = (n + 1023) / 1024;
    DeviceBuffer<uint32_t> d_counts, d_offs, d_part, d_tot, d_dest;
    std::vector<uint32_t> dest(2 * (static_cast<size_t>(world) + 1));
    cudaStream_t cs = v->compute;
    cudaError_t e = d_counts.reserve(2 * n);
    if (e == cudaSuccess) e = d_offs.reserve(2 * n);
    if (e == cudaSuccess) e = d_part.reserve(2 * chunks);
    if (e == cudaSuccess) e = d_tot.reserve(2);
    if (e == cudaSuccess) e = d_dest.reserve(dest.size());
    if (e == cudaSuccess)
        e = launch_halo_count(v->meta, nb, world, d_counts.get(), d_offs.get(), d_part.get(), d_tot.get(),
                              d_dest.get(), cs);
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(dest.data(), d_dest.get(), dest.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, cs);
    if (e == cudaSuccess) e = cudaStreamSynchronize(cs);
    int out = B2V_OK;
    if (e == cudaSuccess) {
        const uint32_t *dr = dest.data(), *dp = dest.data() + world + 1;
        for (int r = 0; r < world; ++r) {
            records[r] = dr[r + 1] - dr[r];
            payload_voxels[r] = dp[r + 1] - dp[r];
        }
        if (d_headers) {
            if (static_cast<int64_t>(dr[world]) > max_records || static_cast<int64_t>(dp[world]) > max_payload_voxels) {
                v->err = "b2v_export_halo_device: destination too small";
                out = B2V_ERR_INVALID_ARGUMENT;
            } else {
                e = launch_halo_emit(v->meta, nb, world, d_offs.get(), d_headers, d_payload, cs, v->cfg.color_f64 != 0);
                if (e == cudaSuccess) e = cudaStreamSynchronize(cs);
            }
        }
    }
    if (e != cudaSuccess) {
        v->err = std::string("b2v_export_halo_device: ") + cudaGetErrorString(e);
        return B2V_ERR_CUDA;
    }
    return out;
}

// the unsharded scratch of the halo extraction, with room for `blocks` blocks (recreated larger when needed)
static int ensure_halo_scratch(b2v_volume *v, uint64_t blocks) {
    if (v->halo && v->halo->meta.capacity >= blocks) return B2V_OK;
    b2v_destroy(v->halo);
    v->halo = nullptr;
    const uint64_t cap = std::max<uint64_t>(1024, blocks + blocks / 2);
    if (cap > (1ull << 30)) {
        v->err = "halo extraction: more than 2^30 blocks";
        return B2V_ERR_UNSUPPORTED;
    }
    b2v_config c = v->cfg;
    c.shard_rank = 0;
    c.shard_count = 1;
    c.capacity_blocks = static_cast<uint32_t>(cap);
    c.max_capacity_blocks = 0;
    b2v_volume *h = nullptr;
    const int rc = b2v_create(&c, &h);
    if (rc != B2V_OK) {
        v->err = std::string("halo extraction scratch: ") + (h ? h->err : "invalid configuration");
        b2v_destroy(h);
        return rc;
    }
    v->halo = h;
    return B2V_OK;
}

static int extract_with_halo(b2v_volume *v, bool mesh, int64_t n_records, const int32_t *d_headers,
                             const float *d_payload, int64_t *n_vertices, int64_t *n_triangles) {
    if (n_records < 0 || (n_records > 0 && (!d_headers || !d_payload))) {
        v->err = "b2v_extract_*_with_halo: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    int rc = read_counters(v);
    if (rc == B2V_ERR_CUDA) return rc;
    B2V_CUDA(v, cudaSetDevice(v->cfg.device));
    const uint32_t nb = block_count(v);
    rc = ensure_halo_scratch(v, static_cast<uint64_t>(nb) + static_cast<uint64_t>(n_records));
    if (rc != B2V_OK) return rc;
    b2v_volume *h = v->halo;
    const uint32_t nr = static_cast<uint32_t>(n_records);
    cudaStream_t cs = h->compute;
    DeviceBuffer<uint32_t> d_sizes, d_offs, d_part, d_tot;
    uint32_t head[2] = {nb + nr, 0u};   // the scratch's block count; its error flag after the import
    cudaError_t e = d_sizes.reserve(nr);
    if (e == cudaSuccess) e = d_offs.reserve(nr);
    if (e == cudaSuccess) e = d_part.reserve((nr + 1023) / 1024 + 1);
    if (e == cudaSuccess) e = d_tot.reserve(1);
    if (e == cudaSuccess)
        e = cudaMemsetAsync(h->table.entries, 0xFF, (static_cast<size_t>(h->table.mask) + 1) * sizeof(uint4), cs);
    if (e == cudaSuccess) e = cudaMemsetAsync(h->meta.counters, 0, kNumCounters * sizeof(uint32_t), cs);
    if (e == cudaSuccess)
        e = launch_halo_import(v->meta, nb, d_headers, d_payload, nr, d_sizes.get(), d_offs.get(), d_part.get(),
                               d_tot.get(), h->table, h->meta, cs, v->cfg.color_f64 != 0);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->meta.counters + kCtrPool, &head[0], sizeof(uint32_t), cudaMemcpyHostToDevice, cs);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&head[1], h->meta.counters + kCtrError, sizeof(uint32_t), cudaMemcpyDeviceToHost, cs);
    if (e == cudaSuccess) e = cudaStreamSynchronize(cs);
    if (e != cudaSuccess) {
        v->err = std::string("halo import: ") + cudaGetErrorString(e);
        return B2V_ERR_CUDA;
    }
    if (head[1]) {
        v->err = (head[1] & 4u) ? "halo import: a record has an invalid mask (or another colour precision)"
                 : (head[1] & 8u) ? "halo import: a block key arrived twice (records of another world size?)"
                                  : "halo import: scratch table full";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    rc = extract_common(h, mesh, n_vertices, n_triangles);
    if (rc != B2V_OK) {
        v->err = h->err;
        return rc;
    }
    if (!mesh && nb < h->mb.n_blocks) {
        // the point pass roots at the own blocks only: their points come first (output order is by pool index)
        uint32_t owned = 0;
        B2V_CUDA(v, cudaMemcpy(&owned, h->mb.offs + nb, sizeof(uint32_t), cudaMemcpyDeviceToHost));
        h->last_nv = owned;
        if (n_vertices) *n_vertices = owned;
    }
    v->last_from_halo = true;
    return B2V_OK;
}

extern "C" int b2v_extract_mesh_with_halo(b2v_volume *v, int64_t n_records, const int32_t *d_headers,
                                          const float *d_payload, int64_t *n_vertices, int64_t *n_triangles) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    return extract_with_halo(v, true, n_records, d_headers, d_payload, n_vertices, n_triangles);
}

extern "C" int b2v_extract_points_with_halo(b2v_volume *v, int64_t n_records, const int32_t *d_headers,
                                            const float *d_payload, int64_t *n_points) {
    if (!v) return B2V_ERR_INVALID_ARGUMENT;
    return extract_with_halo(v, false, n_records, d_headers, d_payload, n_points, nullptr);
}

static thread_local std::string g_weld_err;

extern "C" const char *b2v_weld_last_error(void) { return g_weld_err.c_str(); }

extern "C" int b2v_weld_mesh_device(int32_t device, int32_t n_pieces, const int64_t *piece_vertices,
                                    const int64_t *piece_triangles, const double *d_vertices, const double *d_colors,
                                    const int32_t *d_edge_ids, const int32_t *d_triangles, double *d_out_vertices,
                                    double *d_out_colors, int32_t *d_out_edge_ids, int32_t *d_out_triangles,
                                    int64_t *n_out_vertices) {
    g_weld_err.clear();
    if (n_pieces < 1 || !piece_vertices || !piece_triangles || !n_out_vertices) {
        g_weld_err = "b2v_weld_mesh_device: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    std::vector<uint32_t> base(2 * (static_cast<size_t>(n_pieces) + 1), 0u);
    uint64_t nv = 0, nt = 0;
    for (int p = 0; p < n_pieces; ++p) {
        if (piece_vertices[p] < 0 || piece_triangles[p] < 0) {
            g_weld_err = "b2v_weld_mesh_device: negative piece size";
            return B2V_ERR_INVALID_ARGUMENT;
        }
        base[p] = static_cast<uint32_t>(nv);
        base[n_pieces + 1 + p] = static_cast<uint32_t>(nt);
        nv += static_cast<uint64_t>(piece_vertices[p]);
        nt += static_cast<uint64_t>(piece_triangles[p]);
    }
    if (nv >= (1ull << 30) || nt >= (1ull << 31)) {
        g_weld_err = "b2v_weld_mesh_device: mesh too large";
        return B2V_ERR_UNSUPPORTED;
    }
    base[n_pieces] = static_cast<uint32_t>(nv);
    base[2 * static_cast<size_t>(n_pieces) + 1] = static_cast<uint32_t>(nt);
    if ((nv && (!d_vertices || !d_colors || !d_edge_ids || !d_out_vertices || !d_out_colors || !d_out_edge_ids)) ||
        (nt && (!d_triangles || !d_out_triangles))) {
        g_weld_err = "b2v_weld_mesh_device: missing buffers";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    *n_out_vertices = 0;
    if (cudaSetDevice(device) != cudaSuccess) {
        g_weld_err = "b2v_weld_mesh_device: bad device";
        return B2V_ERR_CUDA;
    }
    WeldArgs a{};
    a.nv = static_cast<uint32_t>(nv);
    a.nt = static_cast<uint32_t>(nt);
    a.n_pieces = n_pieces;
    a.vertices = d_vertices;
    a.colors = d_colors;
    a.edge_ids = d_edge_ids;
    a.triangles = d_triangles;
    a.out_vertices = d_out_vertices;
    a.out_colors = d_out_colors;
    a.out_edge_ids = d_out_edge_ids;
    a.out_triangles = d_out_triangles;
    const uint32_t scap = next_pow2(std::max<uint64_t>(1024, 2 * nv));
    a.set.mask = scap - 1;
    DeviceBuffer<uint4> set;
    DeviceBuffer<uint32_t> first, slot_of, keep, newidx, partials, totals, d_base;
    uint32_t host_tot[2] = {0u, 0u};
    cudaStream_t cs = nullptr;
    const size_t n1 = nv ? nv : 1;
    cudaError_t e = cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = set.reserve(scap);
    if (e == cudaSuccess) e = first.reserve(scap);
    if (e == cudaSuccess) e = slot_of.reserve(n1);
    if (e == cudaSuccess) e = keep.reserve(n1);
    if (e == cudaSuccess) e = newidx.reserve(n1);
    if (e == cudaSuccess) e = partials.reserve((n1 + 1023) / 1024);
    if (e == cudaSuccess) e = totals.reserve(2);
    if (e == cudaSuccess) e = d_base.reserve(base.size());
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(d_base.get(), base.data(), base.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, cs);
    a.set.entries = set.get();
    a.first = first.get();
    a.slot_of = slot_of.get();
    a.keep = keep.get();
    a.newidx = newidx.get();
    a.partials = partials.get();
    a.totals = totals.get();
    a.vbase = d_base.get();
    a.tbase = d_base.get() + n_pieces + 1;
    if (e == cudaSuccess) e = launch_weld(a, cs);
    if (e == cudaSuccess) e = cudaMemcpyAsync(host_tot, a.totals, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, cs);
    if (e == cudaSuccess) e = cudaStreamSynchronize(cs);
    if (cs) cudaStreamDestroy(cs);
    if (e != cudaSuccess) {
        g_weld_err = std::string("b2v_weld_mesh_device: ") + cudaGetErrorString(e);
        return B2V_ERR_CUDA;
    }
    if (host_tot[1]) {
        g_weld_err = "b2v_weld_mesh_device: edge-id set full";
        return B2V_ERR_CUDA;
    }
    *n_out_vertices = nv ? host_tot[0] : 0;
    return B2V_OK;
}

// ---- depth shadow filter (b2v_prep.cu) -------------------------------------------------------

extern "C" int b2v_filter_shadow_points(const float *depth, int32_t height, int32_t width, int32_t delta_x,
                                        int32_t delta_y, float fill_value, float *out, int32_t device) {
    if (!depth || !out || height <= 0 || width <= 0 || delta_x < 0 || delta_y < 0 || delta_x >= width ||
        delta_y >= height)
        return B2V_ERR_INVALID_ARGUMENT;
    if (cudaSetDevice(device) != cudaSuccess) return B2V_ERR_CUDA;
    const size_t pixels = static_cast<size_t>(height) * width;
    const bool din = is_device_pointer(depth), dout = is_device_pointer(out);
    DeviceBuffer<float> d_in, d_out;
    DeviceBuffer<uint8_t> scratch;
    cudaError_t e = scratch.reserve(kShadowScratchBytes);
    if (e == cudaSuccess && !din) {
        e = d_in.reserve(pixels);
        if (e == cudaSuccess) e = cudaMemcpy(d_in.get(), depth, pixels * sizeof(float), cudaMemcpyHostToDevice);
    }
    if (e == cudaSuccess && !dout) e = d_out.reserve(pixels);
    if (e == cudaSuccess)
        e = launch_filter_shadow_points(din ? depth : d_in.get(), height, width, delta_x, delta_y, fill_value,
                                        dout ? out : d_out.get(), scratch.get(), nullptr);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess && !dout) e = cudaMemcpy(out, d_out.get(), pixels * sizeof(float), cudaMemcpyDeviceToHost);
    return e == cudaSuccess ? B2V_OK : B2V_ERR_CUDA;
}
