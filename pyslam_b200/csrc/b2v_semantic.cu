// b2v_semantic.cu — semantic voxel-block grids on sm_90a (SURVEY.md §8(f) rank 2, Appendix D).
//
// Replaces, for the `integrate(points, colors, class_ids, instance_ids, depths)` path and its read-outs,
//   VoxelBlockSemanticGrid               = VoxelBlockSemanticGridT<VoxelSemanticData>               (voting)
//   VoxelBlockSemanticProbabilisticGrid  = VoxelBlockSemanticGridT<VoxelSemanticDataProbabilistic>  (Bayesian)
// (cpp/volumetric/voxel_block_semantic_grid.h:118-121; voxel data: voxel_data_semantic.h:106-199, 249-672;
//  integrate: voxel_block_grid.hpp:12-112, 220-288, 524-614; get_voxels :717-819).
//
// Both label rules are ORDER DEPENDENT in the reference (the voting counter is a sequential state machine; the
// Bayesian argmax keeps the earlier label on ties; float sums round in input order).  The reference's
// deterministic build processes the points of one call in input order, so this implementation does the same
// per voxel:
//   1. insert   one thread per point: block key (bit-exact, in the point's own precision) -> 128-bit-CAS table
//   2. keys     one thread per point: sort key = pool_index * B^3 + local voxel index
//   3. sort     stable LSD radix sort of (key, point index) pairs (cub::DeviceRadixSort - library code)
//   4. runs     the first element of every run of equal keys walks its run in input order and applies the
//               reference's per-observation update: count, position_sum (float64), color_sum (float32), labels
// => counts, sums, labels and log-evidence are bit-identical to the sequential reference.  Only exp / log of the
// confidence read-out are evaluated in float64 and rounded (glibc's expf / logf are within 1 ulp of that).
//
// Bayesian labels: the reference keeps a std::map<(object, class), float> per voxel (typically 1-5 entries);
// here a voxel has kSemLabels = 8 fixed slots.  Without an overflow label store (the default) a ninth distinct pair
// evicts the slot with the least evidence that is not the current argmax (the first on ties) and bumps the overflow
// counter (b2v_sgrid_label_overflows); tests/test_gpu_semantic_edges.py checks the evicted slot.  With a store
// (b2v_sgrid_set_label_overflow) a voxel links chunks of 8 more pairs from a grid-wide pool and never evicts below
// the store's ceiling, so it holds the reference's unbounded map.  The store is a compile-time flag (kChain) of the
// kernels that touch label pairs: their kChain = false instantiations are the grid without a store.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <map>
#include <new>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/b2v.h"
#include "b2v_block_grid.cuh"
#include "b2v_scan.cuh"

namespace b2v {

constexpr int kSemLabels = B2V_SEM_MAX_LABELS;
constexpr float kBaseLogProb = 0.10536051565782628f;  // voxel_data_semantic.h:287, -log(0.9)
constexpr int kSemArrays = 11;   // per-voxel arrays of a Bayesian grid (a voting grid has the first 6)
static_assert(kSemArrays <= kMaxBlockArrays, "a block upload carries every array");

// the block index as the semantic kernels read it: BlockIndex without the shard fields, which only the block insert
// reads (the 24-byte layout keeps sem_runs_kernel's label slots in a local-memory frame, as before the shard fields)
struct SemBlockIndex {
    int4 *block_keys;
    uint32_t *counters;
    uint32_t capacity, pool_capacity;
};

struct SemGrid {
    SemBlockIndex index;
    int32_t *count;     // [V]            V = capacity * B^3, voxel id = pool index * B^3 + lx + B ly + B^2 lz
    double *pos;        // [V][3]
    float *col;         // [V][3]
    int32_t *obj, *cls; // [V]            current label (voting) / cached argmax (Bayesian)
    int32_t *counter;   // [V]            voting: confidence counter; Bayesian: number of label slots in use
    float *ml_logp;     // [V]            Bayesian: evidence of the argmax
    float *conf;        // [V]            Bayesian: cached confidence
    int32_t *lab_obj, *lab_cls;  // [V][kSemLabels]
    float *lab_logp;             // [V][kSemLabels]
    int32_t kind;
    float depth_threshold, depth_decay_rate;
};

// ---- overflow label store ----------------------------------------------------------------------------------------
// Pair s of a voxel (insertion order) is in-voxel slot s for s < kSemLabels, else entry (s - kSemLabels) % 8 of the
// ((s - kSemLabels) / 8)-th chunk of the voxel's chain.  Chunks are taken from the pool's free list first, then fresh
// from its mapped storage; edits that reset a voxel or collapse its labels push its chain onto the free list.
constexpr int kChunkPairs = 8;
constexpr uint64_t kMaxLabelChunks = 1ull << 25;   // 2^28 overflow pairs, 4 GiB of chunks
struct alignas(16) LabelChunk {
    int32_t obj[kChunkPairs], cls[kChunkPairs];
    float logp[kChunkPairs];
    uint32_t next;   // 1 + index of the next chunk of the chain, 0: the last
    uint32_t pad[7];
};
static_assert(sizeof(LabelChunk) == 128, "chunk layout");

enum LabelCounter : int {
    kLcFree = 0,        // chunks on the free list
    kLcFresh = 1,       // chunks ever taken from the storage (in use = fresh - free)
    kLcTaken = 2,       // chunks requested by the runs of the current pass
    kLcFirstFail = 3,   // the least request start of a run that got none (UINT_MAX: none)
    kLcListed = 4,      // runs listed for the replay
    kLcFull = 5,        // a run could not have chunks and no growth could give them: it evicted
    kLcNum = 8
};

struct LabelStore {
    uint32_t *head;           // [V] 1 + index of the voxel's first chunk, 0: none (zeroed memory is the cleared state)
    LabelChunk *chunks;       // [mapped]
    uint32_t *free_list;      // [mapped], kLcFree of them in use
    uint32_t *ctr;            // LabelCounter
    uint32_t *list;           // sorted position of the head of each run that found no chunks
    const uint32_t *replay;   // non-NULL: thread r updates the run starting at replay[r], r < n_replay
    uint32_t n_replay;
    uint32_t mapped;          // chunks with storage
    int32_t no_growth;        // the storage cannot grow: a run without chunks evicts instead of waiting for a replay
};

// visit the pairs of a voxel in slot order: f(slot, obj *, cls *, logp *) returns true to stop
template <typename F>
__device__ __forceinline__ void for_each_pair(const LabelStore &S, int32_t *lo, int32_t *lc, float *lp, int nl,
                                              uint32_t head, F f) {
    const int nr = nl < kSemLabels ? nl : kSemLabels;
    for (int s = 0; s < nr; ++s)
        if (f(s, lo + s, lc + s, lp + s)) return;
    LabelChunk *c = nullptr;
    for (int s = kSemLabels; s < nl; ++s) {
        const int e = (s - kSemLabels) & (kChunkPairs - 1);
        if (e == 0) c = S.chunks + ((c ? c->next : head) - 1);
        if (f(s, c->obj + e, c->cls + e, c->logp + e)) return;
    }
}

// push the voxel's chain onto the free list
template <bool kChain> __device__ __forceinline__ void sem_release_labels(const LabelStore &S, uint32_t v) {
    if constexpr (kChain) {
        uint32_t link = S.head[v];
        if (link == 0) return;
        S.head[v] = 0;
        while (link != 0) {
            const uint32_t c = link - 1;
            link = S.chunks[c].next;
            S.free_list[atomicAdd(S.ctr + kLcFree, 1u)] = c;
        }
    }
}

// ---- 2. sort keys: BlockGridCore::sort_voxels (b2v_grid.cu) ------------------------------------------------
// Only points whose block has a pool index in [lo, hi) get a key; the others get kBadVid, sort last and are left out
// by the runs.  The first pass of a call covers the blocks with storage, [0, pool_capacity); after a growth the
// keys -> sort -> runs passes are replayed over the blocks that just got storage.

// ---- fused front-end: depth2pointcloud + world transform of one labelled RGBD frame ------------------------
// (pyslam/utilities/depth.py:45-85; pyslam/dense/volumetric_integrator_voxel_semantic_grid.py:392-453).  One
// thread per pixel writes the point record the reference front-end would have produced for it; invalid pixels
// are masked instead of compacted - their sort key is kBadVid, so the per-voxel order of the valid ones is the
// row-major pixel order, i.e. the reference's point order.
__global__ void __launch_bounds__(256)
sem_rgbd_points_kernel(const RgbdParams P, const float *__restrict__ depth, const uint8_t *__restrict__ rgb,
                       const int32_t *__restrict__ class_img, const int32_t *__restrict__ object_img,
                       float *__restrict__ pts, float *__restrict__ cols, int32_t *__restrict__ cls,
                       int32_t *__restrict__ inst, float *__restrict__ depths, uint8_t *__restrict__ valid) {
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
    if (class_img) cls[i] = class_img[i];
    if (object_img) inst[i] = object_img[i];
    depths[i] = depth[i];  // points[:, 2] narrowed back to float32 (:408-409) is the depth itself
}

// ---- 4. per-voxel sequential update ------------------------------------------------------------------------
struct SemInputs {
    const void *pts;      // float or double [n][3]
    const void *cols;     // nullptr, float [n][3] or uint8 [n][3]
    const int32_t *cls;   // nullptr or [n]
    const int32_t *inst;  // nullptr or [n]
    const float *depths;  // nullptr or [n]
    int32_t pts_f64, cols_u8;
};

__device__ __forceinline__ float exp_rn(float x) { return __double2float_rn(exp(static_cast<double>(x))); }
__device__ __forceinline__ float log_rn(float x) { return __double2float_rn(log(static_cast<double>(x))); }

// log_add_exp (voxel_data_semantic.h:626-635)
__device__ __forceinline__ float log_add_exp(float a, float b) {
    const float ninf = __uint_as_float(0xFF800000u);
    if (a == ninf) return b;
    if (b == ninf) return a;
    const float m = fmaxf(a, b);
    return __fadd_rn(m, log_rn(__fadd_rn(exp_rn(__fsub_rn(a, m)), exp_rn(__fsub_rn(b, m)))));
}

// confidence of the argmax: exp(max - logsumexp) with the sum folded in std::map order, i.e. ascending
// (object, class) (voxel_data_semantic.h:561-570, 607-624)
__device__ float bayes_confidence(const int32_t *lo, const int32_t *lc, const float *lp, int nl, int mo, int mc,
                                  float mlp) {
    if (mo == -1 || mc == -1 || nl == 0) return 0.0f;
    float sum = __uint_as_float(0xFF800000u);
    long long prev = LLONG_MIN;
    for (int k = 0; k < nl; ++k) {  // selection in key order; nl <= 8
        long long best = LLONG_MAX;
        int bi = -1;
        for (int j = 0; j < nl; ++j) {
            const long long key = (static_cast<long long>(lo[j]) << 32) + (static_cast<long long>(lc[j]) + 0x80000000LL);
            if (key > prev && key < best) {
                best = key;
                bi = j;
            }
        }
        if (bi < 0) break;
        prev = best;
        sum = log_add_exp(sum, lp[bi]);
    }
    return exp_rn(__fsub_rn(mlp, sum));
}

// the same over every pair of a voxel with an overflow chain
__device__ float bayes_confidence_chain(const LabelStore &S, int32_t *lo, int32_t *lc, float *lp, int nl,
                                        uint32_t head, int mo, int mc, float mlp) {
    if (mo == -1 || mc == -1 || nl == 0) return 0.0f;
    float sum = __uint_as_float(0xFF800000u);
    long long prev = LLONG_MIN;
    for (int k = 0; k < nl; ++k) {
        long long best = LLONG_MAX;
        float bl = 0.0f;
        for_each_pair(S, lo, lc, lp, nl, head, [&](int, const int32_t *o, const int32_t *c, const float *l) {
            const long long key = (static_cast<long long>(*o) << 32) + (static_cast<long long>(*c) + 0x80000000LL);
            if (key > prev && key < best) {
                best = key;
                bl = *l;
            }
            return false;
        });
        if (best == LLONG_MAX) break;
        prev = best;
        sum = log_add_exp(sum, bl);
    }
    return exp_rn(__fsub_rn(mlp, sum));
}

// one Bayesian observation (object oo, class oc, evidence w) of a voxel with an overflow chain that can hold `cap`
// pairs: the update of sem_runs_kernel over all of its pairs.  A new pair past `cap` evicts the weakest pair that is
// not the argmax, the first in slot order on ties.
__device__ __forceinline__ void bayes_observe_chain(const LabelStore &S, int32_t *lo, int32_t *lc, float *lp, int &nl,
                                                    uint32_t head, int cap, int32_t oo, int32_t oc, float w,
                                                    int32_t count, int32_t &obj, int32_t &cls, float &mlp,
                                                    uint32_t *overflows) {
    int32_t *po = nullptr, *pc = nullptr;
    float *pl = nullptr;
    for_each_pair(S, lo, lc, lp, nl, head, [&](int, int32_t *o, int32_t *c, float *l) {
        if (*o != oo || *c != oc) return false;
        po = o, pc = c, pl = l;
        return true;
    });
    // slot s for a new pair (pl == nullptr before)
    auto at = [&](int s) {
        if (s < kSemLabels) {
            po = lo + s, pc = lc + s, pl = lp + s;
            return;
        }
        LabelChunk *c = S.chunks + (head - 1);
        for (int q = (s - kSemLabels) / kChunkPairs; q > 0; --q) c = S.chunks + (c->next - 1);
        const int e = (s - kSemLabels) & (kChunkPairs - 1);
        po = c->obj + e, pc = c->cls + e, pl = c->logp + e;
    };
    if (count == 0) {  // initialize_semantics_log_prob: map[key] = w, argmax = key
        if (pl == nullptr) {
            at(nl < cap ? nl++ : 0);
            *po = oo, *pc = oc;
        }
        *pl = w;
        obj = oo, cls = oc, mlp = w;
    } else if (pl != nullptr) {  // known pair: accumulate; a strictly larger value takes the argmax
        *pl = __fadd_rn(*pl, w);
        if (*po == obj && *pc == cls) {
            mlp = *pl;
        } else if (*pl > mlp) {
            mlp = *pl;
            obj = oo, cls = oc;
        }
    } else {  // new pair
        if (nl < cap) {
            at(nl++);
        } else {  // out of slots: evict the weakest pair that is not the argmax
            float least = 0.0f;
            for_each_pair(S, lo, lc, lp, nl, head, [&](int, int32_t *o, int32_t *c, float *l) {
                if (!(*o == obj && *c == cls) && (pl == nullptr || *l < least)) {
                    po = o, pc = c, pl = l;
                    least = *l;
                }
                return false;
            });
            atomicAdd(overflows, 1u);
        }
        *po = oo, *pc = oc, *pl = w;
        if (w > mlp) {
            mlp = w;
            obj = oo, cls = oc;
        }
    }
}

// Chunks for the run of voxel v at sorted positions [j0, ...) before it applies anything: the run counts the distinct
// pairs it adds to the voxel's nl pairs and, if they pass what its chain holds, takes the missing chunks with one
// atomic and links them to the chain.  Returns the pairs the chain then holds (kSemLabels + 8 per chunk), or -1 when
// the run got no chunks and must wait for the replay (it is listed).  Without growth (S.no_growth) such a run keeps
// its chain and evicts.
__device__ int sem_take_chunks(const LabelStore &S, const uint32_t *vid, const uint32_t *order, int64_t n, int64_t j0,
                               const SemInputs &in, int32_t *lo, int32_t *lc, float *lp, int nl, uint32_t &head) {
    const uint32_t v = vid[j0];
    int chunks = 0;
    uint32_t tail = 0;   // 1 + index of the chain's last chunk
    for (uint32_t link = head; link != 0; link = S.chunks[link - 1].next) {
        tail = link;
        ++chunks;
    }
    int added = 0;
    for (int64_t j = j0; j < n && vid[j] == v; ++j) {
        const uint32_t i = order[j];
        const int32_t oc = in.cls[i], oo = in.inst ? in.inst[i] : 0;
        bool seen = false;
        for (int64_t q = j - 1; q >= j0 && !seen; --q) {   // earlier in the run (the previous one first)
            const uint32_t iq = order[q];
            seen = in.cls[iq] == oc && (in.inst ? in.inst[iq] : 0) == oo;
        }
        if (!seen)
            for_each_pair(S, lo, lc, lp, nl, head, [&](int, const int32_t *o, const int32_t *c, const float *) {
                seen = *o == oo && *c == oc;
                return seen;
            });
        added += seen ? 0 : 1;
    }
    const int have = kSemLabels + kChunkPairs * chunks;
    const int over = nl + added - have;
    if (over <= 0) return have;
    const uint32_t need = static_cast<uint32_t>((over + kChunkPairs - 1) / kChunkPairs);
    const uint32_t n_free = S.ctr[kLcFree], fresh = S.ctr[kLcFresh];
    const uint32_t t = atomicAdd(S.ctr + kLcTaken, need);
    if (static_cast<uint64_t>(t) + need > static_cast<uint64_t>(n_free) + (S.mapped - fresh)) {
        atomicMin(S.ctr + kLcFirstFail, t);
        if (S.no_growth) {
            atomicOr(S.ctr + kLcFull, 1u);
            return have;
        }
        S.list[atomicAdd(S.ctr + kLcListed, 1u)] = static_cast<uint32_t>(j0);
        return -1;
    }
    for (uint32_t x = t; x < t + need; ++x) {   // free list from the top, then fresh chunks
        const uint32_t c = x < n_free ? S.free_list[n_free - 1 - x] : fresh + (x - n_free);
        S.chunks[c].next = 0;
        if (tail == 0) head = c + 1;
        else S.chunks[tail - 1].next = c + 1;
        tail = c + 1;
    }
    return have + kChunkPairs * static_cast<int>(need);
}

template <bool kChain>
__global__ void __launch_bounds__(128)
sem_runs_kernel(const uint32_t *__restrict__ vid, const uint32_t *__restrict__ order, const int64_t n,
                const SemInputs in, const SemGrid G, const LabelStore S) {
    int64_t j0 = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if constexpr (kChain) {
        if (S.replay != nullptr) {
            if (j0 >= S.n_replay) return;
            j0 = S.replay[j0];
        }
    }
    if (j0 >= n) return;
    const uint32_t v = vid[j0];
    if (v == kBadVid || (j0 > 0 && vid[j0 - 1] == v)) return;  // not the head of a run

    int32_t count = G.count[v];
    double px = G.pos[3 * static_cast<size_t>(v) + 0], py = G.pos[3 * static_cast<size_t>(v) + 1],
           pz = G.pos[3 * static_cast<size_t>(v) + 2];
    float cr = G.col[3 * static_cast<size_t>(v) + 0], cg = G.col[3 * static_cast<size_t>(v) + 1],
          cb = G.col[3 * static_cast<size_t>(v) + 2];
    int32_t obj = G.obj[v], cls = G.cls[v], ctr = G.counter[v];
    const bool bayes = G.kind == B2V_SEM_PROBABILISTIC;
    const bool semantics = in.cls != nullptr && in.cols != nullptr;  // no colours => positions only (hpp:228-231)
    float mlp = 0.0f;
    int32_t lo[kSemLabels], lc[kSemLabels];
    float lp[kSemLabels];
    int nl = 0;
    if (bayes && semantics) {
        mlp = G.ml_logp[v];
        nl = ctr;
        for (int k = 0; k < kSemLabels; ++k) {
            lo[k] = G.lab_obj[static_cast<size_t>(v) * kSemLabels + k];
            lc[k] = G.lab_cls[static_cast<size_t>(v) * kSemLabels + k];
            lp[k] = G.lab_logp[static_cast<size_t>(v) * kSemLabels + k];
        }
    }
    uint32_t head = 0;
    int cap = kSemLabels;   // pairs the voxel can hold in this run
    if constexpr (kChain) {
        if (bayes && semantics) {
            head = S.head[v];
            cap = sem_take_chunks(S, vid, order, n, j0, in, lo, lc, lp, nl, head);
            if (cap < 0) return;   // nothing written: the replay applies the whole run
        }
    }

    for (int64_t j = j0; j < n && vid[j] == v; ++j) {
        const uint32_t i = order[j];
        double x, y, z;
        if (in.pts_f64) {
            const double *p = static_cast<const double *>(in.pts) + 3 * static_cast<size_t>(i);
            x = p[0], y = p[1], z = p[2];
        } else {
            const float *p = static_cast<const float *>(in.pts) + 3 * static_cast<size_t>(i);
            x = p[0], y = p[1], z = p[2];
        }
        px = __dadd_rn(px, x);  // voxel_data.h:53-57
        py = __dadd_rn(py, y);
        pz = __dadd_rn(pz, z);
        if (in.cols != nullptr) {  // voxel_data.h:79-90
            float r, g, b;
            if (in.cols_u8) {
                const uint8_t *c = static_cast<const uint8_t *>(in.cols) + 3 * static_cast<size_t>(i);
                r = color_value(c[0]), g = color_value(c[1]), b = color_value(c[2]);
            } else {
                const float *c = static_cast<const float *>(in.cols) + 3 * static_cast<size_t>(i);
                r = c[0], g = c[1], b = c[2];
            }
            cr = __fadd_rn(cr, r);
            cg = __fadd_rn(cg, g);
            cb = __fadd_rn(cb, b);
        }
        if (semantics) {
            const int32_t oc = in.cls[i];
            const int32_t oo = in.inst ? in.inst[i] : 0;  // no instance ids: object id 0 (hpp:259-286)
            const bool has_depth = in.depths != nullptr;
            const float depth = has_depth ? in.depths[i] : 0.0f;
            if (!bayes) {
                // voting (voxel_data_semantic.h:153-198): observations at depth >= threshold are ignored
                if (!has_depth || depth < G.depth_threshold) {
                    if (count == 0) {
                        obj = oo, cls = oc, ctr = 1;
                    } else if (obj == oo && cls == oc) {
                        ++ctr;
                    } else if (--ctr <= 0) {
                        obj = oo, cls = oc, ctr = 1;
                    }
                }
            } else {
                // Bayesian (voxel_data_semantic.h:312-451): evidence w * -log(0.9), w = 1 up to the depth threshold,
                // exp(-(depth - threshold) * rate) beyond it
                float w = kBaseLogProb;
                if (has_depth && !(depth <= G.depth_threshold))
                    w = __fmul_rn(exp_rn(__fmul_rn(-__fsub_rn(depth, G.depth_threshold), G.depth_decay_rate)),
                                  kBaseLogProb);
                if constexpr (kChain) {
                    bayes_observe_chain(S, lo, lc, lp, nl, head, cap, oo, oc, w, count, obj, cls, mlp,
                                        G.index.counters + kBgLabelOverflow);
                    ++count;
                    continue;
                }
                int k = 0;
                while (k < nl && !(lo[k] == oo && lc[k] == oc)) ++k;
                if (count == 0) {  // initialize_semantics_log_prob: map[key] = w, argmax = key
                    if (k == nl) {
                        k = nl < kSemLabels ? nl++ : 0;
                        lo[k] = oo, lc[k] = oc;
                    }
                    lp[k] = w;
                    obj = oo, cls = oc, mlp = w;
                } else if (k < nl) {  // known pair: accumulate; a strictly larger value takes the argmax
                    lp[k] = __fadd_rn(lp[k], w);
                    if (lo[k] == obj && lc[k] == cls) {
                        mlp = lp[k];
                    } else if (lp[k] > mlp) {
                        mlp = lp[k];
                        obj = oo, cls = oc;
                    }
                } else {  // new pair
                    if (nl < kSemLabels) {
                        k = nl++;
                    } else {  // out of slots: evict the weakest pair that is not the argmax
                        k = -1;
                        for (int q = 0; q < kSemLabels; ++q)
                            if (!(lo[q] == obj && lc[q] == cls) && (k < 0 || lp[q] < lp[k])) k = q;
                        atomicAdd(G.index.counters + kBgLabelOverflow, 1u);
                    }
                    lo[k] = oo, lc[k] = oc, lp[k] = w;
                    if (w > mlp) {
                        mlp = w;
                        obj = oo, cls = oc;
                    }
                }
            }
        }
        ++count;
    }

    G.count[v] = count;
    G.pos[3 * static_cast<size_t>(v) + 0] = px;
    G.pos[3 * static_cast<size_t>(v) + 1] = py;
    G.pos[3 * static_cast<size_t>(v) + 2] = pz;
    G.col[3 * static_cast<size_t>(v) + 0] = cr;
    G.col[3 * static_cast<size_t>(v) + 1] = cg;
    G.col[3 * static_cast<size_t>(v) + 2] = cb;
    if (semantics) {
        G.obj[v] = obj;
        G.cls[v] = cls;
        if (!bayes) {
            G.counter[v] = ctr;
        } else {
            G.counter[v] = nl;
            G.ml_logp[v] = mlp;
            for (int k = 0; k < kSemLabels; ++k) {
                G.lab_obj[static_cast<size_t>(v) * kSemLabels + k] = lo[k];
                G.lab_cls[static_cast<size_t>(v) * kSemLabels + k] = lc[k];
                G.lab_logp[static_cast<size_t>(v) * kSemLabels + k] = lp[k];
            }
            if constexpr (kChain) {
                S.head[v] = head;
                G.conf[v] = bayes_confidence_chain(S, lo, lc, lp, nl, head, obj, cls, mlp);
            } else {
                G.conf[v] = bayes_confidence(lo, lc, lp, nl, obj, cls, mlp);
            }
        }
    }
}

// ---- read-outs -------------------------------------------------------------------------------------------------
__device__ __forceinline__ float sem_confidence(const SemGrid &G, uint32_t v, int32_t count) {
    if (count == 0) return 0.0f;
    if (G.kind == B2V_SEM_PROBABILISTIC) return G.conf[v];
    // voting (voxel_data_semantic.h:117-132): min(1, counter / count)
    return fminf(1.0f, __fdiv_rn(static_cast<float>(G.counter[v]), static_cast<float>(count)));
}

template <bool kChain>
__device__ __forceinline__ void sem_reset_voxel(const SemGrid &G, const LabelStore &S, uint32_t v) {  // ::reset()
    sem_release_labels<kChain>(S, v);
    G.count[v] = 0;
    for (int a = 0; a < 3; ++a) {
        G.pos[3 * static_cast<size_t>(v) + a] = 0.0;
        G.col[3 * static_cast<size_t>(v) + a] = 0.0f;
    }
    G.obj[v] = -1;
    G.cls[v] = -1;
    G.counter[v] = 0;
    if (G.kind == B2V_SEM_PROBABILISTIC) {
        G.ml_logp[v] = __uint_as_float(0xFF800000u);
        G.conf[v] = 0.0f;
    }
}

// op 0: remove_low_count_voxels(a)  1: remove_low_confidence_segments(a)  2: remove_segment(a)
// op 3: merge_segments(a, b)  (voxel_block_grid.hpp:625-647; voxel_block_semantic_grid.hpp:101-183)
// Per-voxel passes: one 512-thread CTA per 512 pool voxels (cta_voxel), so voxel id = blockIdx.x * 512 + threadIdx.x
// whatever B; nv (the voxels of the blocks in use) bounds the last CTA when B < 8 and is not read at B >= 8.
template <int L, bool kChain>
__global__ void __launch_bounds__(kVox)
sem_edit_kernel(const SemGrid G, const int op, const int a, const int b, const uint32_t nv, const LabelStore S) {
    const uint32_t v = blockIdx.x * kVox + threadIdx.x;
    if (3 * L < 9 && v >= nv) return;
    const int c = G.count[v];
    if (op == 0) {
        if (c < a) sem_reset_voxel<kChain>(G, S, v);
    } else if (op == 1) {
        if (sem_confidence(G, v, c) < static_cast<float>(a)) sem_reset_voxel<kChain>(G, S, v);
    } else if (op == 2) {
        if (G.obj[v] == a) sem_reset_voxel<kChain>(G, S, v);
    } else if (G.obj[v] == b) {
        G.obj[v] = a;  // set_object_id
        if (G.kind == B2V_SEM_PROBABILISTIC) {
            sem_release_labels<kChain>(S, v);
            // force_label_distribution (voxel_data_semantic.h:589-605): a single pair with log-probability 0
            const int32_t cl = G.cls[v];
            if (a >= 0 && cl >= 0) {
                G.counter[v] = 1;
                G.lab_obj[static_cast<size_t>(v) * kSemLabels] = a;
                G.lab_cls[static_cast<size_t>(v) * kSemLabels] = cl;
                G.lab_logp[static_cast<size_t>(v) * kSemLabels] = 0.0f;
                G.ml_logp[v] = 0.0f;
                G.conf[v] = 1.0f;
            } else {
                G.counter[v] = 0;
                G.ml_logp[v] = __uint_as_float(0xFF800000u);
                G.conf[v] = 0.0f;
            }
        }
    }
}

// ---- spatial filter: read-outs, carve and instance -> object association ----------------------------------------
// the key range, then the fine test (box or frustum) on the voxel's float64 mean position.  Empty voxels never qualify
// (get_voxels_in_bb, voxel_block_grid.hpp:822-1016; iterate_voxels_in_camera_frustrum, :1336-1460).
template <int L>
__device__ __forceinline__ bool sem_in_region(const SemGrid &G, const GridQuery &Q, uint32_t b, int t, ImagePoint *ip) {
    const int4 key = G.index.block_keys[b];
    if (!block_in_range<L>(Q, key)) return false;
    const uint32_t v = b * GridBlock<L>::kVox + t;
    const int c = G.count[v];
    if (c < 1 || !voxel_in_range<L>(Q, key, t)) return false;
    const double dc = static_cast<double>(c);
    double p[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) p[a] = __ddiv_rn(G.pos[3 * static_cast<size_t>(v) + a], dc);
    return region_contains(Q, p, ip);
}

// the read-out filter: count >= min_count and confidence >= min_conf (voxel_block_grid.hpp:797-803), then in box and
// frustum mode (get_voxels_in_bb, get_voxels_in_camera_frustrum :1019-1195) the spatial filter.  A voxel of a block
// past nb (the last CTA of a pass at B < 8) is never kept.
template <int L>
__device__ __forceinline__ bool sem_keep(const SemGrid &G, const GridQuery &Q, uint32_t b, int t, uint32_t nb,
                                         float min_conf, float *conf_out) {
    if (3 * L < 9 && b >= nb) {
        *conf_out = 0.0f;
        return false;
    }
    const uint32_t v = b * GridBlock<L>::kVox + t;
    const int c = G.count[v];
    const float conf = sem_confidence(G, v, c);
    *conf_out = conf;
    if (!(c >= Q.min_count && conf >= min_conf)) return false;
    if (Q.mode == kQueryAll) return true;
    ImagePoint ip;
    return sem_in_region<L>(G, Q, b, t, &ip);
}

template <int L>
__global__ void __launch_bounds__(kVox)
sem_count_kernel(const SemGrid G, const GridQuery Q, const float min_conf, uint32_t *__restrict__ sums,
                 const uint32_t nb) {
    __shared__ uint32_t s_warp[16];
    float conf;
    uint32_t b;
    int t;
    cta_voxel<L>(&b, &t);
    block_count_512(sem_keep<L>(G, Q, b, t, nb, min_conf, &conf), s_warp, sums + blockIdx.x);
}

template <int L>
__global__ void __launch_bounds__(kVox)
sem_emit_kernel(const SemGrid G, const GridQuery Q, const float min_conf,
                const uint32_t *__restrict__ offs, double *__restrict__ out_pts, float *__restrict__ out_cols,
                int32_t *__restrict__ out_cls, int32_t *__restrict__ out_obj, float *__restrict__ out_conf,
                const uint32_t nb) {
    __shared__ uint32_t s_warp[16];
    const uint32_t v = blockIdx.x * kVox + threadIdx.x;
    float conf;
    uint32_t b;
    int t;
    cta_voxel<L>(&b, &t);
    const bool keep = sem_keep<L>(G, Q, b, t, nb, min_conf, &conf);
    const size_t pos = offs[blockIdx.x] + block_excl_scan_512(keep ? 1u : 0u, s_warp);
    if (!keep) return;
    const int c = G.count[v];
    const double dc = static_cast<double>(c);
    const float fc = static_cast<float>(c);
    for (int a = 0; a < 3; ++a) {  // voxel_data.h:58-69, 98-109: sum / (T)count, zero for an empty voxel
        out_pts[3 * pos + a] = c ? __ddiv_rn(G.pos[3 * static_cast<size_t>(v) + a], dc) : 0.0;
        out_cols[3 * pos + a] = c ? __fdiv_rn(G.col[3 * static_cast<size_t>(v) + a], fc) : 0.0f;
    }
    out_cls[pos] = G.cls[v];
    out_obj[pos] = G.obj[v];
    out_conf[pos] = conf;
}

// set_object_id (voxel_data_semantic.h:135, 455-460): the Bayesian voxel collapses onto the forced pair
template <bool kChain>
__device__ __forceinline__ void sem_set_object_id(const SemGrid &G, const LabelStore &S, uint32_t v, int32_t id) {
    G.obj[v] = id;
    if (G.kind == B2V_SEM_PROBABILISTIC) {
        sem_release_labels<kChain>(S, v);
        const int32_t cl = G.cls[v];
        if (id >= 0 && cl >= 0) {
            G.counter[v] = 1;
            G.lab_obj[static_cast<size_t>(v) * kSemLabels] = id;
            G.lab_cls[static_cast<size_t>(v) * kSemLabels] = cl;
            G.lab_logp[static_cast<size_t>(v) * kSemLabels] = 0.0f;
            G.ml_logp[v] = 0.0f;
            G.conf[v] = 1.0f;
        } else {
            G.counter[v] = 0;
            G.ml_logp[v] = __uint_as_float(0xFF800000u);
            G.conf[v] = 0.0f;
        }
    }
}

// carve (voxel_grid_carving.h:47-80): reset voxels in front of the observed surface by more than the threshold;
// the depth image is indexed with truncated pixel coordinates, like at<float>(v, u)
template <int L, bool kChain>
__global__ void __launch_bounds__(kVox)
sem_carve_kernel(const SemGrid G, const GridQuery Q, const float *__restrict__ depth, const float thr,
                 const uint32_t nb, const LabelStore S) {
    uint32_t b;
    int t;
    cta_voxel<L>(&b, &t);
    if (3 * L < 9 && b >= nb) return;
    ImagePoint ip;
    if (!sem_in_region<L>(G, Q, b, t, &ip)) return;
    const float image_depth = depth[static_cast<size_t>(static_cast<int>(ip.v)) * Q.W + static_cast<int>(ip.u)];
    if (image_depth <= 0.0f || !isfinite(image_depth)) return;
    if (ip.depth < image_depth - thr) sem_reset_voxel<kChain>(G, S, blockIdx.x * kVox + threadIdx.x);
}

// process_point of assign_object_ids_to_instance_ids (voxel_semantic_data_association.h:171-229): every voxel in
// the frustum whose class equals the pixel's class and that lies on the observed surface votes
// "image instance id -> my object id".  Voxels without an object id are recorded as pending (pend[v] = instance
// id).  The records are reduced on the device to sorted (instance, object, count) triples, from which the host
// builds the instance -> object map.
constexpr int32_t kAssocPending = B2V_ASSOC_PENDING;
static_assert(kAssocPending == INT_MIN, "the pending marker sorts before every object id");

// vote record (instance, object) as one sort key: sign bits flipped, so unsigned order is (instance, object) order
__device__ __forceinline__ unsigned long long assoc_key(int32_t inst, int32_t obj) {
    return static_cast<unsigned long long>(static_cast<uint32_t>(inst) ^ 0x80000000u) << 32 |
           (static_cast<uint32_t>(obj) ^ 0x80000000u);
}

template <int L, bool kChain>
__global__ void __launch_bounds__(kVox)
sem_assoc_kernel(const SemGrid G, const GridQuery Q, const int32_t *__restrict__ class_img,
                 const int32_t *__restrict__ inst_img, const float *__restrict__ depth_img, const float thr,
                 const int do_carving, int32_t *__restrict__ pend, unsigned long long *__restrict__ records,
                 uint32_t *__restrict__ n_records, const uint32_t cap_records, const uint32_t nb,
                 const LabelStore S) {
    uint32_t b;
    int t;
    cta_voxel<L>(&b, &t);
    if (3 * L < 9 && b >= nb) return;
    ImagePoint ip;
    if (!sem_in_region<L>(G, Q, b, t, &ip)) return;
    const uint32_t v = blockIdx.x * kVox + threadIdx.x;
    const size_t px = static_cast<size_t>(static_cast<int>(ip.v)) * Q.W + static_cast<int>(ip.u);
    const int32_t image_class = class_img[px];
    if (image_class < 0) return;
    const int32_t point_class = G.cls[v];
    if (point_class < 0 || point_class != image_class) return;
    const int32_t image_instance = inst_img[px];
    if (image_instance < 0) return;
    int32_t point_object = G.obj[v];
    if (depth_img != nullptr) {
        const float image_depth = depth_img[px];
        if (image_depth <= 0.0f || !isfinite(image_depth)) return;
        if (do_carving && ip.depth < image_depth - thr) {
            sem_reset_voxel<kChain>(G, S, v);
            return;
        }
        if (ip.depth > image_depth + thr) return;
    }
    if (point_object < 0) {
        if (image_instance == 0) {
            point_object = 0;
            sem_set_object_id<kChain>(G, S, v, 0);
        } else {
            point_object = kAssocPending;  // one new object id per instance id, handed out by the host
            pend[v] = image_instance;
        }
    }
    const uint32_t r = atomicAdd(n_records, 1u);
    if (r < cap_records) records[r] = assoc_key(image_instance, point_object);
}

// the runs of the sorted records -> triples int32 [n_runs][3] = {instance, object or kAssocPending, count}
__global__ void __launch_bounds__(256)
sem_assoc_triples_kernel(const unsigned long long *__restrict__ keys, const uint32_t *__restrict__ counts,
                         const uint32_t *__restrict__ n_runs, int32_t *__restrict__ triples) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *n_runs) return;
    const unsigned long long k = keys[i];
    triples[3 * static_cast<size_t>(i) + 0] = static_cast<int32_t>(static_cast<uint32_t>(k >> 32) ^ 0x80000000u);
    triples[3 * static_cast<size_t>(i) + 1] = static_cast<int32_t>(static_cast<uint32_t>(k) ^ 0x80000000u);
    triples[3 * static_cast<size_t>(i) + 2] = static_cast<int32_t>(counts[i]);
}

// deferred assignment (voxel_semantic_data_association.h:354-370): pending voxels take their instance's final id
template <int L, bool kChain>
__global__ void __launch_bounds__(kVox)
sem_assoc_apply_kernel(const SemGrid G, const int32_t *__restrict__ pend, const int32_t *__restrict__ map_inst,
                       const int32_t *__restrict__ map_obj, const int n_map, const uint32_t nv, const LabelStore S) {
    const uint32_t v = blockIdx.x * kVox + threadIdx.x;
    if (3 * L < 9 && v >= nv) return;
    const int32_t inst = pend[v];
    if (inst < 0) return;
    int lo = 0, hi = n_map - 1;
    while (lo <= hi) {  // map_inst is sorted
        const int mid = (lo + hi) >> 1;
        const int32_t m = map_inst[mid];
        if (m == inst) {
            if (map_obj[mid] >= 0) sem_set_object_id<kChain>(G, S, v, map_obj[mid]);
            return;
        }
        if (m < inst) lo = mid + 1; else hi = mid - 1;
    }
}

// the non-zero fields of a cleared voxel, for the voxels [v0, v1)
__global__ void sem_fill_kernel(const SemGrid G, const size_t v0, const size_t v1) {
    for (size_t v = v0 + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < v1;
         v += static_cast<size_t>(gridDim.x) * blockDim.x) {
        G.obj[v] = -1;
        G.cls[v] = -1;
        if (G.kind == B2V_SEM_PROBABILISTIC) G.ml_logp[v] = __uint_as_float(0xFF800000u);
    }
}

}  // namespace b2v

// ====================================================================================================================
// host side: the C ABI of include/b2v.h (b2v_sgrid_*)
// ====================================================================================================================
using namespace b2v;

struct b2v_sgrid : BlockGridCore {
    SemGrid G{};   // G.index is not kept: dev() fills it in
    // each per-voxel array of G is a reservation for index.capacity blocks with storage mapped on demand (a fixed grid
    // maps it whole at create); index.pool_capacity is the least any array holds
    VmmRange store[kSemArrays];
    // staging of the points of one call (float or double points, float or uint8 colours)
    DeviceBuffer<double> d_pts;
    DeviceBuffer<float> d_cols, d_depths;
    DeviceBuffer<int32_t> d_cls, d_inst;
    DeviceBuffer<uint8_t> d_valid;   // per-point mask of the fused RGBD front-end; its size is the staging capacity
    // instance -> object association: votes (records -> sort -> runs -> triples), then resolve
    DeviceBuffer<int32_t> d_pend;                  // [voxels] instance id of a pending voxel, else -1
    DeviceBuffer<unsigned long long> d_records;    // [voxels] vote records (sort keys)
    DeviceBuffer<uint32_t> d_n_records;            // [2] records, runs
    DeviceBuffer<unsigned long long> d_runs;       // [votes capacity] run keys
    DeviceBuffer<uint32_t> d_run_counts;           // [votes capacity]
    DeviceBuffer<int32_t> d_triples;               // [votes capacity][3]
    DeviceBuffer<uint8_t> d_votes_tmp;
    DeviceBuffer<unsigned long long> d_sorted;     // [votes capacity] sort buffer; its size is the votes capacity
    int64_t n_triples = 0;
    // every call that may change a voxel bumps `generation`; resolve needs the votes of the current state
    uint64_t generation = 0, votes_generation = 0;
    bool votes_ready = false;
    uint32_t votes_blocks = 0;                       // blocks d_pend covers
    int32_t next_object_id = 1;  // VoxelSemanticSharedData::next_object_id (process-wide in the reference)
    std::vector<int32_t> map_inst, map_obj;
    bool has_instance_map = false;   // the last association succeeded (map_inst / map_obj are its map)
    DeviceBuffer<int32_t> d_map;     // its map_inst then map_obj on the device
    // read-out
    DeviceBuffer<double> d_out_pts;
    DeviceBuffer<float> d_out_cols, d_out_conf;
    DeviceBuffer<int32_t> d_out_cls;
    DeviceBuffer<int32_t> d_out_obj;   // its size is the read-out capacity
    int64_t last_n = 0;
    // overflow label store (b2v_sgrid_set_label_overflow): lab_max_chunks 0 = none, the kernels' kChain = false
    uint32_t lab_max_chunks = 0;
    uint32_t lab_mapped = 0;          // chunks with storage (the mapped granules may hold more)
    int64_t lab_growths = 0;
    bool lab_full = false;            // a run of the current call evicted for want of chunks past the ceiling
    std::string lab_map_err;          // the chunk storage of the current call failed to grow (device memory)
    VmmRange lab_head;                // [voxels] chain heads, mapped with the per-voxel arrays
    VmmRange lab_chunks, lab_free;    // [lab_max_chunks] chunks and free list, mapped on demand
    DeviceBuffer<uint32_t> d_lab_ctr;   // LabelCounter
    DeviceBuffer<uint32_t> d_lab_list;  // runs listed for the replay; its size is their capacity

    SemGrid dev() const {   // the kernels' view
        SemGrid d = G;
        d.index = SemBlockIndex{index.block_keys, index.counters, index.capacity, index.pool_capacity};
        return d;
    }
    LabelStore labels() const {   // the store as the kernels see it (all NULL without one)
        LabelStore s{};
        if (lab_max_chunks == 0) return s;
        s.head = reinterpret_cast<uint32_t *>(lab_head.va);
        s.chunks = reinterpret_cast<LabelChunk *>(lab_chunks.va);
        s.free_list = reinterpret_cast<uint32_t *>(lab_free.va);
        s.ctr = d_lab_ctr.get();
        s.list = d_lab_list.get();
        s.mapped = lab_mapped;
        s.no_growth = lab_mapped >= lab_max_chunks ? 1 : 0;
        return s;
    }
};

// f(block size, chain flag) as integral constants: the kernels of the grid's block size and label store
template <typename F> static void sgrid_dispatch(const b2v_sgrid *g, F &&f) {
    g->dispatch([&](auto l) {
        if (g->lab_max_chunks) f(l, std::true_type{});
        else f(l, std::false_type{});
    });
}

static bool sgrid_map_labels(b2v_sgrid *g, uint64_t chunks, std::string *err);
static int sgrid_set_labels(b2v_sgrid *g, const char *fn, int64_t n_blocks, const int32_t *keys4, const int32_t *n_over,
                            const int32_t *obj, const int32_t *cls, const float *logp);

// an empty store: no chain, no chunk taken
static int sgrid_label_reset(b2v_sgrid *g, size_t nv) {
    static const uint32_t init[kLcNum] = {0, 0, 0, UINT32_MAX, 0, 0, 0, 0};
    if (nv) B2V_CUDA(g, cudaMemsetAsync(reinterpret_cast<void *>(g->lab_head.va), 0, nv * sizeof(uint32_t), g->stream));
    B2V_CUDA(g, cudaMemcpyAsync(g->d_lab_ctr.get(), init, sizeof(init), cudaMemcpyHostToDevice, g->stream));
    return B2V_OK;
}

extern "C" const char *b2v_sgrid_last_error(const b2v_sgrid *g) { return g ? g->err.c_str() : "null grid"; }

static int sgrid_clear_device(b2v_sgrid *g, uint32_t used_blocks) {
    const size_t nv = static_cast<size_t>(used_blocks) * g->block_voxels();
    const int rc = g->clear_index();
    if (rc != B2V_OK || nv == 0) return rc;
    B2V_CUDA(g, cudaMemsetAsync(g->G.count, 0, nv * sizeof(int32_t), g->stream));
    B2V_CUDA(g, cudaMemsetAsync(g->G.pos, 0, nv * 3 * sizeof(double), g->stream));
    B2V_CUDA(g, cudaMemsetAsync(g->G.col, 0, nv * 3 * sizeof(float), g->stream));
    B2V_CUDA(g, cudaMemsetAsync(g->G.counter, 0, nv * sizeof(int32_t), g->stream));
    if (g->G.kind == B2V_SEM_PROBABILISTIC) B2V_CUDA(g, cudaMemsetAsync(g->G.conf, 0, nv * sizeof(float), g->stream));
    sem_fill_kernel<<<592, 256, 0, g->stream>>>(g->dev(), 0, nv);
    B2V_CUDA(g, cudaGetLastError());
    return g->lab_max_chunks ? sgrid_label_reset(g, nv) : B2V_OK;
}

// the per-voxel arrays of the grid's kind and the bytes each holds per voxel
struct SemArray {
    void **ptr;
    size_t voxel_bytes;
};
static int sgrid_arrays(b2v_sgrid *g, SemArray out[kSemArrays]) {
    SemGrid &G = g->G;
    const SemArray all[kSemArrays] = {
        {reinterpret_cast<void **>(&G.count), sizeof(int32_t)},
        {reinterpret_cast<void **>(&G.pos), 3 * sizeof(double)},
        {reinterpret_cast<void **>(&G.col), 3 * sizeof(float)},
        {reinterpret_cast<void **>(&G.obj), sizeof(int32_t)},
        {reinterpret_cast<void **>(&G.cls), sizeof(int32_t)},
        {reinterpret_cast<void **>(&G.counter), sizeof(int32_t)},
        {reinterpret_cast<void **>(&G.ml_logp), sizeof(float)},
        {reinterpret_cast<void **>(&G.conf), sizeof(float)},
        {reinterpret_cast<void **>(&G.lab_obj), kSemLabels * sizeof(int32_t)},
        {reinterpret_cast<void **>(&G.lab_cls), kSemLabels * sizeof(int32_t)},
        {reinterpret_cast<void **>(&G.lab_logp), kSemLabels * sizeof(float)},
    };
    const int n = G.kind == B2V_SEM_PROBABILISTIC ? kSemArrays : 6;
    for (int k = 0; k < n; ++k) out[k] = all[k];
    return n;
}

// map (zeroed) storage for at least `blocks` blocks in every array; index.pool_capacity becomes the least any array
// holds.
// Voxels entering the storage are set to the cleared state by the caller.  False if a mapping failed.
static bool sgrid_map_storage(b2v_sgrid *g, uint64_t blocks, std::string *err) {
    SemArray arr[kSemArrays];
    const int na = sgrid_arrays(g, arr);
    bool ok = true;
    uint64_t storage = g->index.capacity;
    for (int k = 0; k < na; ++k) {
        const size_t block_bytes = arr[k].voxel_bytes * g->block_voxels();
        ok = ok && vmm_map(&g->store[k], static_cast<size_t>(blocks) * block_bytes, g->stream, err);
        storage = std::min<uint64_t>(storage, g->store[k].mapped / block_bytes);
    }
    if (g->lab_max_chunks) {
        const size_t block_bytes = sizeof(uint32_t) * g->block_voxels();
        ok = ok && vmm_map(&g->lab_head, static_cast<size_t>(blocks) * block_bytes, g->stream, err);
        storage = std::min<uint64_t>(storage, g->lab_head.mapped / block_bytes);
    }
    g->index.pool_capacity = static_cast<uint32_t>(storage);
    return ok;
}

// the storage growth of BlockGridCore::resolve / upload_blocks
static auto sgrid_grow_storage(b2v_sgrid *g) {
    return [g](uint64_t blocks) {
        std::string map_err;   // a failed mapping surfaces as "block pool full"
        sgrid_map_storage(g, blocks, &map_err);
    };
}

extern "C" int b2v_sgrid_create_ex(double voxel_size, int32_t block_size, uint32_t capacity_blocks,
                                   uint32_t max_capacity_blocks, int32_t kind, int32_t device, b2v_sgrid **out) {
    if (!out) return B2V_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    // the sort key pool_index * B^3 + voxel must stay below kBadVid: at most 2^31 / B^3 blocks (2^22 at B = 8)
    if (!BlockGridCore::valid_args(voxel_size, block_size, capacity_blocks, max_capacity_blocks) ||
        capacity_blocks > BlockGridCore::max_blocks(BlockGridCore::log2_block_size(block_size)) ||
        (kind != B2V_SEM_VOTING && kind != B2V_SEM_PROBABILISTIC))
        return B2V_ERR_INVALID_ARGUMENT;
    b2v_sgrid *g = new (std::nothrow) b2v_sgrid();
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    g->G.kind = kind;
    g->frame_labels = true;
    // class defaults (voxel_data_semantic.h:107-108, 251-254)
    g->G.depth_threshold = kind == B2V_SEM_VOTING ? 10.0f : 5.0f;
    g->G.depth_decay_rate = 0.07f;
    *out = g;
    int rc = g->create(voxel_size, block_size, capacity_blocks, max_capacity_blocks, device);
    if (rc != B2V_OK) return rc;
    SemArray arr[kSemArrays];
    const int na = sgrid_arrays(g, arr);
    for (int k = 0; k < na; ++k) {
        if (!vmm_reserve(&g->store[k], static_cast<size_t>(g->index.capacity) * g->block_voxels() * arr[k].voxel_bytes, device,
                         &g->err))
            return B2V_ERR_CUDA;
        *arr[k].ptr = reinterpret_cast<void *>(g->store[k].va);
    }
    if (!sgrid_map_storage(g, capacity_blocks, &g->err)) return B2V_ERR_CUDA;
    g->index.pool_capacity = capacity_blocks;   // the rest of the last granules is used only after a growth
    rc = sgrid_clear_device(g, capacity_blocks);
    if (rc != B2V_OK) return rc;
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    return B2V_OK;
}

extern "C" int b2v_sgrid_destroy(b2v_sgrid *g) {
    if (!g) return B2V_OK;
    g->destroy();
    delete g;
    return B2V_OK;
}

extern "C" int b2v_sgrid_set_shard(b2v_sgrid *g, int32_t shard_rank, int32_t shard_count) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->set_shard(shard_rank, shard_count);
}

extern "C" int b2v_sgrid_set_label_overflow(b2v_sgrid *g, uint64_t max_pairs, uint64_t initial_pairs) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (max_pairs == 0) return B2V_OK;
    const uint64_t chunks = (max_pairs + kChunkPairs - 1) / kChunkPairs;
    if (g->G.kind != B2V_SEM_PROBABILISTIC || g->lab_max_chunks != 0 || chunks > kMaxLabelChunks) {
        g->err = g->G.kind != B2V_SEM_PROBABILISTIC ? "b2v_sgrid_set_label_overflow: the voting grid has no label set"
                 : g->lab_max_chunks ? "b2v_sgrid_set_label_overflow: the store is already set"
                                     : "b2v_sgrid_set_label_overflow: more than 2^28 overflow pairs";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    B2V_CUDA(g, cudaSetDevice(g->device));
    int rc = g->fetch_counters();
    if (rc != B2V_OK) return rc;
    if (g->h_counters[kBgPool] != 0) {
        g->err = "b2v_sgrid_set_label_overflow: only on a grid without blocks";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    const size_t head_block = sizeof(uint32_t) * g->block_voxels();
    B2V_CUDA(g, g->d_lab_ctr.reserve(kLcNum));
    if (!vmm_reserve(&g->lab_head, static_cast<size_t>(g->index.capacity) * head_block, g->device, &g->err) ||
        !vmm_reserve(&g->lab_chunks, static_cast<size_t>(chunks) * sizeof(LabelChunk), g->device, &g->err) ||
        !vmm_reserve(&g->lab_free, static_cast<size_t>(chunks) * sizeof(uint32_t), g->device, &g->err) ||
        !vmm_map(&g->lab_head, static_cast<size_t>(g->index.pool_capacity) * head_block, g->stream, &g->err))
        return B2V_ERR_CUDA;
    g->lab_max_chunks = static_cast<uint32_t>(chunks);
    const uint64_t first = std::max<uint64_t>(1, (initial_pairs + kChunkPairs - 1) / kChunkPairs);
    if (!sgrid_map_labels(g, first, &g->err)) return B2V_ERR_CUDA;
    rc = sgrid_label_reset(g, 0);
    if (rc != B2V_OK) return rc;
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    return B2V_OK;
}

extern "C" int b2v_sgrid_label_storage(b2v_sgrid *g, int64_t *chunks_used, int64_t *chunks_mapped,
                                       int64_t *chunks_max, int64_t *growths) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    uint32_t c[kLcNum] = {};
    if (g->lab_max_chunks) {
        B2V_CUDA(g, cudaMemcpyAsync(c, g->d_lab_ctr.get(), sizeof(c), cudaMemcpyDeviceToHost, g->stream));
        B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    }
    if (chunks_used) *chunks_used = static_cast<int64_t>(c[kLcFresh]) - c[kLcFree];
    if (chunks_mapped) *chunks_mapped = g->lab_mapped;
    if (chunks_max) *chunks_max = g->lab_max_chunks;
    if (growths) *growths = g->lab_growths;
    return B2V_OK;
}

extern "C" int b2v_sgrid_clear(b2v_sgrid *g) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    ++g->generation;
    int rc = g->fetch_counters();
    if (rc != B2V_OK) return rc;
    rc = sgrid_clear_device(g, g->block_count());   // the storage is kept
    if (rc != B2V_OK) return rc;
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    return B2V_OK;
}

extern "C" int b2v_sgrid_set_depth_threshold(b2v_sgrid *g, float depth_threshold) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    g->G.depth_threshold = depth_threshold;
    return B2V_OK;
}

extern "C" int b2v_sgrid_set_depth_decay_rate(b2v_sgrid *g, float depth_decay_rate) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (g->G.kind == B2V_SEM_PROBABILISTIC) g->G.depth_decay_rate = depth_decay_rate;  // semantic_grid.hpp:31-36
    return B2V_OK;
}

static int sgrid_ensure_stage(b2v_sgrid *g, size_t n) {
    if (n <= g->d_valid.size()) return B2V_OK;
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    g->d_valid = {};   // reserved last: it holds the capacity only once every staging buffer does
    const size_t cap = n + n / 4 + 1024;
    B2V_CUDA(g, g->d_pts.reserve(cap * 3));
    B2V_CUDA(g, g->d_cols.reserve(cap * 3));
    B2V_CUDA(g, g->d_cls.reserve(cap));
    B2V_CUDA(g, g->d_inst.reserve(cap));
    B2V_CUDA(g, g->d_depths.reserve(cap));
    const int rc = g->reserve_sort(cap);
    if (rc != B2V_OK) return rc;
    B2V_CUDA(g, g->d_valid.reserve(cap));
    return B2V_OK;
}

// map chunk storage for at least `chunks` chunks (at most the ceiling); false if a mapping failed
static bool sgrid_map_labels(b2v_sgrid *g, uint64_t chunks, std::string *err) {
    chunks = std::min<uint64_t>(chunks, g->lab_max_chunks);
    const bool ok = vmm_map(&g->lab_chunks, static_cast<size_t>(chunks) * sizeof(LabelChunk), g->stream, err) &&
                    vmm_map(&g->lab_free, static_cast<size_t>(chunks) * sizeof(uint32_t), g->stream, err);
    const uint64_t held = std::min<uint64_t>(g->lab_chunks.mapped / sizeof(LabelChunk),
                                             g->lab_free.mapped / sizeof(uint32_t));
    g->lab_mapped = static_cast<uint32_t>(std::max<uint64_t>(g->lab_mapped, std::min(chunks, held)));
    return ok;
}

// After a runs pass with a label store: the chunks its runs took leave the free list or the fresh storage, the pass
// counters are re-armed, and *listed is the number of runs that got none.  *wanted: the chunks the storage must hold
// for their replay.  Synchronises.
static int sgrid_label_settle(b2v_sgrid *g, uint32_t *listed, uint64_t *wanted) {
    uint32_t c[kLcNum];
    B2V_CUDA(g, cudaMemcpyAsync(c, g->d_lab_ctr.get(), sizeof(c), cudaMemcpyDeviceToHost, g->stream));
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    // the runs that got chunks requested exactly [0, first fail) of the pass's requests
    const uint32_t used = std::min(c[kLcTaken], c[kLcFirstFail]);
    const uint32_t from_free = std::min(used, c[kLcFree]);
    c[kLcFree] -= from_free;
    c[kLcFresh] += used - from_free;
    *wanted = c[kLcFresh] + std::max<int64_t>(0, static_cast<int64_t>(c[kLcTaken] - used) - c[kLcFree]);
    *listed = c[kLcListed];
    g->lab_full = g->lab_full || c[kLcFull] != 0;
    c[kLcTaken] = 0;
    c[kLcFirstFail] = UINT32_MAX;
    c[kLcListed] = 0;
    c[kLcFull] = 0;
    B2V_CUDA(g, cudaMemcpyAsync(g->d_lab_ctr.get(), c, sizeof(c), cudaMemcpyHostToDevice, g->stream));
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    return B2V_OK;
}

// sem_runs_kernel with a label store: the runs that found no chunks write nothing and are listed; the storage then
// grows to hold them (at least doubling, at most the ceiling) and they are replayed over the same sorted pairs.  A
// voxel's run is its only update in the pass, so the replay applies it from the state before the pass.  Past the
// ceiling the replayed runs that still find no chunks evict (g->lab_full).
static int sgrid_runs_chain(b2v_sgrid *g, int64_t n, const SemInputs &in) {
    cudaStream_t s = g->stream;
    if (g->d_lab_list.size() < static_cast<size_t>(n)) {
        B2V_CUDA(g, cudaStreamSynchronize(s));
        B2V_CUDA(g, g->d_lab_list.reserve(static_cast<size_t>(n) + n / 4 + 1024));
    }
    sem_runs_kernel<true><<<static_cast<unsigned>((n + 127) / 128), 128, 0, s>>>(
        g->sort.vid[1].get(), g->sort.ord[1].get(), n, in, g->dev(), g->labels());
    B2V_CUDA(g, cudaGetLastError());
    uint32_t listed = 0;
    uint64_t wanted = 0;
    int rc = sgrid_label_settle(g, &listed, &wanted);
    if (rc != B2V_OK || listed == 0) return rc;
    if (wanted > g->lab_mapped && g->lab_mapped < g->lab_max_chunks) {
        // a failed mapping still replays (the runs without chunks evict), then the call reports the device error
        const uint32_t old = g->lab_mapped;
        std::string map_err;
        if (!sgrid_map_labels(g, std::max<uint64_t>(wanted, 2ull * old), &map_err) && g->lab_map_err.empty())
            g->lab_map_err = "label storage could not grow: " + map_err;
        if (g->lab_mapped > old) ++g->lab_growths;
    }
    LabelStore S = g->labels();
    S.replay = g->d_lab_list.get();
    S.n_replay = listed;
    S.no_growth = 1;
    sem_runs_kernel<true><<<(listed + 127) / 128, 128, 0, s>>>(g->sort.vid[1].get(), g->sort.ord[1].get(), n, in,
                                                              g->dev(), S);
    B2V_CUDA(g, cudaGetLastError());
    return sgrid_label_settle(g, &listed, &wanted);
}

// keys -> sort -> runs over the staged point records, for the points whose block's pool index lies in [lo, hi)
static int sgrid_apply(b2v_sgrid *g, int64_t n, const SemInputs &in, const uint8_t *valid, uint32_t lo, uint32_t hi) {
    cudaStream_t s = g->stream;
    B2V_CUDA(g, g->sort_voxels(in.pts, in.pts_f64 != 0, valid, n, lo, hi));
    if (g->lab_max_chunks) return sgrid_runs_chain(g, n, in);
    sem_runs_kernel<false><<<static_cast<unsigned>((n + 127) / 128), 128, 0, s>>>(
        g->sort.vid[1].get(), g->sort.ord[1].get(), n, in, g->dev(), LabelStore{});
    B2V_CUDA(g, cudaGetLastError());
    return B2V_OK;
}

// insert -> keys -> sort -> runs over the staged point records (valid: optional per-point mask).  A growable grid
// resolves an overflow before returning (BlockGridCore::resolve): the new voxels are set to the cleared state and
// keys -> sort -> runs is replayed over the blocks that just got storage, from the same staged inputs, so every voxel
// is updated from the cleared state in input order (the sort is stable) and the grid equals one created at the
// maximum.  The staged inputs must stay alive until the call ends.
static int sgrid_fuse_staged(b2v_sgrid *g, int64_t n, const SemInputs &in, const uint8_t *valid) {
    ++g->generation;
    g->lab_full = false;
    g->lab_map_err.clear();
    B2V_CUDA(g, launch_point_insert(in.pts, in.pts_f64 != 0, valid, n, g->inv_voxel_size, g->log2_block, g->table,
                                    g->index, g->stream));
    const int rc = sgrid_apply(g, n, in, valid, 0, g->index.pool_capacity);
    if (rc != B2V_OK || !g->growable) return rc;
    return g->resolve(sgrid_grow_storage(g), [&](uint32_t lo, uint32_t hi) {
        sem_fill_kernel<<<592, 256, 0, g->stream>>>(g->dev(), static_cast<size_t>(lo) * g->block_voxels(),
                                                    static_cast<size_t>(hi) * g->block_voxels());
        B2V_CUDA(g, cudaGetLastError());
        return sgrid_apply(g, n, in, valid, lo, hi);
    });
}

// end of an integrate call: the counters, then B2V_ERR_CUDA if the label storage failed to grow, or "label storage
// full" if a voxel evicted past the store's ceiling
static int sgrid_finish(b2v_sgrid *g) {
    const int rc = g->read_counters();
    if (rc != B2V_OK) return rc;
    if (!g->lab_map_err.empty()) {
        g->err = g->lab_map_err;
        return B2V_ERR_CUDA;
    }
    if (!g->lab_full) return rc;
    g->err = "label storage full";
    return B2V_ERR_CAPACITY;
}

extern "C" int b2v_sgrid_integrate(b2v_sgrid *g, int64_t n, const void *points, int32_t points_f64,
                                   const void *colors, int32_t colors_u8, const int32_t *class_ids,
                                   const int32_t *instance_ids, const float *depths) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (n < 0 || (n > 0 && !points) || n > 0x7FFFFFF0LL) {
        g->err = "b2v_sgrid_integrate: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    if (instance_ids && !class_ids) {  // voxel_block_grid.hpp:43-46
        g->err = "instance_ids but no class_ids is not supported";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    if (n == 0) return B2V_OK;
    B2V_CUDA(g, cudaSetDevice(g->device));
    int rc = sgrid_ensure_stage(g, static_cast<size_t>(n));
    if (rc != B2V_OK) return rc;
    const size_t m = static_cast<size_t>(n);
    cudaStream_t s = g->stream;
    B2V_CUDA(g, cudaMemcpyAsync(g->d_pts.get(), points, m * 3 * (points_f64 ? sizeof(double) : sizeof(float)),
                               cudaMemcpyDefault, s));
    if (colors)
        B2V_CUDA(g, cudaMemcpyAsync(g->d_cols.get(), colors, m * 3 * (colors_u8 ? 1 : sizeof(float)), cudaMemcpyDefault, s));
    if (class_ids) B2V_CUDA(g, cudaMemcpyAsync(g->d_cls.get(), class_ids, m * sizeof(int32_t), cudaMemcpyDefault, s));
    if (instance_ids) B2V_CUDA(g, cudaMemcpyAsync(g->d_inst.get(), instance_ids, m * sizeof(int32_t), cudaMemcpyDefault, s));
    if (depths) B2V_CUDA(g, cudaMemcpyAsync(g->d_depths.get(), depths, m * sizeof(float), cudaMemcpyDefault, s));
    SemInputs in{};
    in.pts = g->d_pts.get();
    in.cols = colors ? g->d_cols.get() : nullptr;
    in.cls = class_ids ? g->d_cls.get() : nullptr;
    in.inst = instance_ids ? g->d_inst.get() : nullptr;
    in.depths = depths ? g->d_depths.get() : nullptr;
    in.pts_f64 = points_f64 ? 1 : 0;
    in.cols_u8 = colors_u8 ? 1 : 0;
    rc = sgrid_fuse_staged(g, n, in, nullptr);
    if (rc != B2V_OK) return rc;
    return sgrid_finish(g);  // also the completion fence: the inputs are free when this returns
}

extern "C" int b2v_sgrid_integrate_rgbd(b2v_sgrid *g, const float *depth, const uint8_t *color,
                                        const int32_t *class_image, const int32_t *object_image, int32_t height,
                                        int32_t width, const double K[4], const double Twc[16], float max_depth,
                                        float min_depth, int32_t use_depths, int32_t filter_shadow_points) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (!depth || !color || !K || !Twc || height <= 0 || width <= 0 || (object_image && !class_image)) {
        g->err = "b2v_sgrid_integrate_rgbd: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    const float *d_depth = depth;
    const uint8_t *d_rgb = color;
    const int32_t *d_cls = class_image, *d_obj = object_image;
    // semantic_grid.py:332-341: everything downstream sees the filtered depth
    int rc = g->stage_input("b2v_sgrid_integrate_rgbd", height, width, filter_shadow_points != 0, &d_depth, &d_rgb,
                            &d_cls, &d_obj);
    if (rc != B2V_OK) return rc;
    const int64_t n = static_cast<int64_t>(height) * width;
    rc = sgrid_ensure_stage(g, static_cast<size_t>(n));
    if (rc != B2V_OK) return rc;
    const RgbdParams P = rgbd_params(K, Twc, min_depth, max_depth, height, width);
    sem_rgbd_points_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, g->stream>>>(
        P, d_depth, d_rgb, d_cls, d_obj, reinterpret_cast<float *>(g->d_pts.get()), g->d_cols.get(), g->d_cls.get(),
        g->d_inst.get(), g->d_depths.get(), g->d_valid.get());
    B2V_CUDA(g, cudaGetLastError());
    SemInputs in{};
    in.pts = g->d_pts.get();
    in.cols = g->d_cols.get();
    in.cls = class_image ? g->d_cls.get() : nullptr;
    in.inst = object_image ? g->d_inst.get() : nullptr;
    in.depths = use_depths ? g->d_depths.get() : nullptr;
    rc = sgrid_fuse_staged(g, n, in, g->d_valid.get());
    if (rc != B2V_OK) return rc;
    return sgrid_finish(g);
}

extern "C" int64_t b2v_sgrid_num_blocks(b2v_sgrid *g) {
    if (!g) return -1;
    if (g->fetch_counters() != B2V_OK) return -1;
    return g->block_count();
}

extern "C" int b2v_sgrid_capacity(b2v_sgrid *g, int64_t *capacity_blocks, int64_t *growths) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->capacity(capacity_blocks, growths);
}

extern "C" int b2v_sgrid_label_overflows(b2v_sgrid *g, uint64_t *out) {
    if (!g || !out) return B2V_ERR_INVALID_ARGUMENT;
    if (b2v_sgrid_num_blocks(g) < 0) return B2V_ERR_CUDA;
    *out = g->h_counters[kBgLabelOverflow];
    return B2V_OK;
}

static int64_t sgrid_run_readout(b2v_sgrid *g, const GridQuery &q, float min_confidence) {
    const int64_t nb64 = b2v_sgrid_num_blocks(g);
    if (nb64 < 0) {
        g->err = "semantic read-out: device error";
        return -1;
    }
    const uint32_t nb = static_cast<uint32_t>(nb64);
    g->last_n = 0;
    if (nb == 0) return 0;
    auto fail = [&](cudaError_t e) {
        g->err = std::string("semantic read-out: ") + cudaGetErrorString(e);
        return static_cast<int64_t>(-1);
    };
    const uint32_t nc = g->voxel_ctas(nb);
    if (g->ensure_scan(nc) != B2V_OK) return -1;
    g->dispatch([&](auto l) {
        sem_count_kernel<decltype(l)::value><<<nc, kVox, 0, g->stream>>>(g->dev(), q, min_confidence, g->d_sums.get(),
                                                                        nb);
    });
    uint32_t total = 0;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = g->scan_total(nc, &total);
    if (e != cudaSuccess) return fail(e);
    if (total > g->d_out_obj.size()) {
        g->d_out_obj = {};   // reserved last: it holds the capacity only once every read-out buffer does
        const size_t cap = static_cast<size_t>(total) + total / 4 + 1024;
        if ((e = g->d_out_pts.reserve(cap * 3)) != cudaSuccess) return fail(e);
        if ((e = g->d_out_cols.reserve(cap * 3)) != cudaSuccess) return fail(e);
        if ((e = g->d_out_conf.reserve(cap)) != cudaSuccess) return fail(e);
        if ((e = g->d_out_cls.reserve(cap)) != cudaSuccess) return fail(e);
        if ((e = g->d_out_obj.reserve(cap)) != cudaSuccess) return fail(e);
    }
    if (total) {
        g->dispatch([&](auto l) {
            sem_emit_kernel<decltype(l)::value><<<nc, kVox, 0, g->stream>>>(
                g->dev(), q, min_confidence, g->d_offs.get(), g->d_out_pts.get(), g->d_out_cols.get(),
                g->d_out_cls.get(), g->d_out_obj.get(), g->d_out_conf.get(), nb);
        });
        if ((e = cudaGetLastError()) != cudaSuccess) return fail(e);
    }
    g->last_n = total;
    return total;
}

extern "C" int64_t b2v_sgrid_get_voxels(b2v_sgrid *g, int32_t min_count, float min_confidence) {
    if (!g) return -1;
    return sgrid_run_readout(g, g->all_query(min_count), min_confidence);
}

extern "C" int64_t b2v_sgrid_get_voxels_in_bb(b2v_sgrid *g, const double bbox[6], int32_t min_count,
                                              float min_confidence) {
    if (!g || !bbox) return -1;
    return sgrid_run_readout(g, g->box_query(bbox, min_count), min_confidence);
}

extern "C" int64_t b2v_sgrid_get_voxels_in_frustum(b2v_sgrid *g, const float K[4], int32_t width, int32_t height,
                                                   const double Tcw[16], float depth_max, float depth_min,
                                                   int32_t min_count, float min_confidence) {
    if (!g || !K || !Tcw || width <= 0 || height <= 0) return -1;
    return sgrid_run_readout(g, g->frustum_query(K, width, height, Tcw, depth_max, depth_min, min_count),
                             min_confidence);
}

extern "C" int b2v_sgrid_copy_voxels(b2v_sgrid *g, double *points, float *colors, int32_t *class_ids,
                                     int32_t *object_ids, float *confidences) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    const size_t n = static_cast<size_t>(g->last_n);
    B2V_CUDA(g, cudaSetDevice(g->device));
    if (n) {
        if (points) B2V_CUDA(g, cudaMemcpyAsync(points, g->d_out_pts.get(), n * 3 * sizeof(double), cudaMemcpyDefault, g->stream));
        if (colors) B2V_CUDA(g, cudaMemcpyAsync(colors, g->d_out_cols.get(), n * 3 * sizeof(float), cudaMemcpyDefault, g->stream));
        if (class_ids) B2V_CUDA(g, cudaMemcpyAsync(class_ids, g->d_out_cls.get(), n * sizeof(int32_t), cudaMemcpyDefault, g->stream));
        if (object_ids) B2V_CUDA(g, cudaMemcpyAsync(object_ids, g->d_out_obj.get(), n * sizeof(int32_t), cudaMemcpyDefault, g->stream));
        if (confidences) B2V_CUDA(g, cudaMemcpyAsync(confidences, g->d_out_conf.get(), n * sizeof(float), cudaMemcpyDefault, g->stream));
    }
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    return B2V_OK;
}

static int sgrid_edit(b2v_sgrid *g, int op, int a, int b) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    ++g->generation;
    const int64_t nb = b2v_sgrid_num_blocks(g);
    if (nb < 0) return B2V_ERR_CUDA;
    if (nb == 0) return B2V_OK;
    const uint32_t nbu = static_cast<uint32_t>(nb);
    sgrid_dispatch(g, [&](auto l, auto c) {
        sem_edit_kernel<decltype(l)::value, decltype(c)::value><<<g->voxel_ctas(nbu), kVox, 0, g->stream>>>(
            g->dev(), op, a, b, nbu * g->block_voxels(), g->labels());
    });
    B2V_CUDA(g, cudaGetLastError());
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    return B2V_OK;
}

extern "C" int b2v_sgrid_remove_low_count_voxels(b2v_sgrid *g, int32_t min_count) { return sgrid_edit(g, 0, min_count, 0); }
extern "C" int b2v_sgrid_remove_low_confidence_segments(b2v_sgrid *g, int32_t min_confidence) {
    return sgrid_edit(g, 1, min_confidence, 0);
}
extern "C" int b2v_sgrid_remove_segment(b2v_sgrid *g, int32_t object_id) { return sgrid_edit(g, 2, object_id, 0); }
extern "C" int b2v_sgrid_merge_segments(b2v_sgrid *g, int32_t object_id1, int32_t object_id2) {
    return sgrid_edit(g, 3, object_id1, object_id2);
}

// ---- carve / instance -> object association -------------------------------------------------------------------------
extern "C" int b2v_sgrid_carve(b2v_sgrid *g, const float K[4], int32_t width, int32_t height, const double Tcw[16],
                               float depth_max, float depth_min, const float *depth, float depth_threshold) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (!K || !Tcw || !depth || width <= 0 || height <= 0) {
        g->err = "b2v_sgrid_carve: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    ++g->generation;
    const int64_t nb = b2v_sgrid_num_blocks(g);
    if (nb < 0) return B2V_ERR_CUDA;
    if (nb == 0) return B2V_OK;
    const float *d_depth = depth;
    const int rc = g->stage_input("b2v_sgrid_carve", height, width, false, &d_depth);
    if (rc != B2V_OK) return rc;
    const GridQuery q = g->frustum_query(K, width, height, Tcw, depth_max, depth_min, 1);
    const uint32_t nbu = static_cast<uint32_t>(nb);
    sgrid_dispatch(g, [&](auto l, auto c) {
        sem_carve_kernel<decltype(l)::value, decltype(c)::value><<<g->voxel_ctas(nbu), kVox, 0, g->stream>>>(
            g->dev(), q, d_depth, depth_threshold, nbu, g->labels());
    });
    B2V_CUDA(g, cudaGetLastError());
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    return B2V_OK;
}

extern "C" int b2v_sgrid_set_next_object_id(b2v_sgrid *g, int32_t next_object_id) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    g->next_object_id = next_object_id;
    return B2V_OK;
}

extern "C" int32_t b2v_sgrid_get_next_object_id(const b2v_sgrid *g) { return g ? g->next_object_id : -1; }

// votes of the association: sem_assoc_kernel (pending marks, optional carving), then the records reduced on the
// device to sorted unique (instance, object or kAssocPending, count) triples in d_triples.  `fn` names the call in
// err.  Returns the number of triples, or -1.
static int64_t sgrid_assoc_votes(b2v_sgrid *g, const char *fn, const float K[4], int32_t width, int32_t height,
                                 const double Tcw[16], float depth_max, float depth_min, const int32_t *class_image,
                                 const int32_t *instance_image, const float *depth_image, float depth_threshold,
                                 int32_t do_carving) {
    g->map_inst.clear();
    g->map_obj.clear();
    g->has_instance_map = false;
    g->votes_ready = false;
    g->n_triples = 0;
    if (!K || !Tcw || !class_image || !instance_image || width <= 0 || height <= 0) {
        g->err = std::string(fn) + ": bad arguments";
        return -1;
    }
    const int64_t nb = b2v_sgrid_num_blocks(g);
    if (nb < 0) return -1;
    const size_t nv = static_cast<size_t>(nb) * g->block_voxels();
    ++g->generation;   // carving, and object id 0 for instance 0, change voxels
    uint32_t counts[2] = {0, 0};   // records, runs
    if (nb > 0) {
        const float *d_depth = depth_image;
        const int32_t *d_cls = class_image, *d_inst = instance_image;
        if (g->stage_input(fn, height, width, false, &d_depth, nullptr, &d_cls, &d_inst) != B2V_OK) return -1;
        cudaStream_t s = g->stream;
        cudaError_t e = g->d_pend.reserve(nv);
        if (e == cudaSuccess) e = g->d_records.reserve(nv);
        if (e == cudaSuccess) e = g->d_n_records.reserve(2);
        uint32_t *const n_records = g->d_n_records.get();
        if (e == cudaSuccess) e = cudaMemsetAsync(g->d_pend.get(), 0xFF, nv * sizeof(int32_t), s);
        if (e == cudaSuccess) e = cudaMemsetAsync(n_records, 0, 2 * sizeof(uint32_t), s);
        if (e == cudaSuccess) {
            const GridQuery q = g->frustum_query(K, width, height, Tcw, depth_max, depth_min, 1);
            const uint32_t nbu = static_cast<uint32_t>(nb);
            sgrid_dispatch(g, [&](auto l, auto c) {
                sem_assoc_kernel<decltype(l)::value, decltype(c)::value><<<g->voxel_ctas(nbu), kVox, 0, s>>>(
                    g->dev(), q, d_cls, d_inst, d_depth, depth_threshold, (do_carving && depth_image) ? 1 : 0,
                    g->d_pend.get(), g->d_records.get(), n_records, static_cast<uint32_t>(nv), nbu, g->labels());
            });
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync(counts, n_records, sizeof(uint32_t), cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        const uint32_t n_rec = counts[0];
        if (e == cudaSuccess && n_rec > g->d_sorted.size()) {   // sort and run buffers sized by the records, not the voxels
            g->d_sorted = {};   // reserved last: it holds the capacity only once every buffer of the votes does
            const size_t cap = std::min<size_t>(nv, static_cast<size_t>(n_rec) + n_rec / 4 + 1024);
            e = g->d_runs.reserve(cap);
            if (e == cudaSuccess) e = g->d_run_counts.reserve(cap);
            if (e == cudaSuccess) e = g->d_triples.reserve(3 * cap);
            size_t sort_bytes = 0, rle_bytes = 0;
            cub::DoubleBuffer<unsigned long long> db(g->d_records.get(), g->d_sorted.get());
            if (e == cudaSuccess)
                e = cub::DeviceRadixSort::SortKeys(nullptr, sort_bytes, db, static_cast<int>(cap), 0, 64, s);
            if (e == cudaSuccess)
                e = cub::DeviceRunLengthEncode::Encode(nullptr, rle_bytes, g->d_records.get(), g->d_runs.get(),
                                                       g->d_run_counts.get(), n_records + 1, static_cast<int>(cap), s);
            if (e == cudaSuccess) e = g->d_votes_tmp.reserve(std::max(sort_bytes, rle_bytes));
            if (e == cudaSuccess) e = g->d_sorted.reserve(cap);
        }
        if (e == cudaSuccess && n_rec) {
            // all 64 bits: the triples come out in ascending (instance, object) order, kAssocPending first
            cub::DoubleBuffer<unsigned long long> db(g->d_records.get(), g->d_sorted.get());
            size_t tmp = g->d_votes_tmp.size();
            e = cub::DeviceRadixSort::SortKeys(g->d_votes_tmp.get(), tmp, db, static_cast<int>(n_rec), 0, 64, s);
            tmp = g->d_votes_tmp.size();
            if (e == cudaSuccess)
                e = cub::DeviceRunLengthEncode::Encode(g->d_votes_tmp.get(), tmp, db.Current(), g->d_runs.get(),
                                                       g->d_run_counts.get(), n_records + 1, static_cast<int>(n_rec), s);
            if (e == cudaSuccess) {
                sem_assoc_triples_kernel<<<(n_rec + 255) / 256, 256, 0, s>>>(g->d_runs.get(), g->d_run_counts.get(),
                                                                             n_records + 1, g->d_triples.get());
                e = cudaGetLastError();
            }
            if (e == cudaSuccess)
                e = cudaMemcpyAsync(counts + 1, n_records + 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, s);
            if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        }
        if (e != cudaSuccess) {
            g->err = std::string(fn) + ": device pass: " + cudaGetErrorString(e);
            return -1;
        }
    }
    g->n_triples = counts[1];
    g->votes_blocks = static_cast<uint32_t>(nb);
    g->votes_generation = g->generation;
    g->votes_ready = true;
    return g->n_triples;
}

extern "C" int64_t b2v_sgrid_assoc_votes(b2v_sgrid *g, const float K[4], int32_t width, int32_t height,
                                         const double Tcw[16], float depth_max, float depth_min,
                                         const int32_t *class_image, const int32_t *instance_image,
                                         const float *depth_image, float depth_threshold, int32_t do_carving) {
    if (!g) return -1;
    return sgrid_assoc_votes(g, "b2v_sgrid_assoc_votes", K, width, height, Tcw, depth_max, depth_min, class_image,
                             instance_image, depth_image, depth_threshold, do_carving);
}

extern "C" int b2v_sgrid_copy_assoc_votes(b2v_sgrid *g, int32_t *triples) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (!g->votes_ready) {
        g->err = "b2v_sgrid_copy_assoc_votes: no votes (run b2v_sgrid_assoc_votes first)";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    if (g->n_triples == 0) return B2V_OK;
    if (!triples) {
        g->err = "b2v_sgrid_copy_assoc_votes: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    B2V_CUDA(g, cudaSetDevice(g->device));
    B2V_CUDA(g, cudaMemcpyAsync(triples, g->d_triples.get(), static_cast<size_t>(g->n_triples) * 3 * sizeof(int32_t),
                                cudaMemcpyDefault, g->stream));
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    return B2V_OK;
}

// resolve of the association from the triples of every rank; `fn` names the call in err
static int64_t sgrid_assoc_resolve(b2v_sgrid *g, const char *fn, const int32_t *triples, int64_t n_triples,
                                   int32_t width, int32_t height, const int32_t *class_image,
                                   const int32_t *instance_image, float min_vote_ratio, int32_t min_votes) {
    if (n_triples < 0 || (n_triples > 0 && !triples) || !class_image || !instance_image || width <= 0 ||
        height <= 0) {
        g->err = std::string(fn) + ": bad arguments";
        return -1;
    }
    if (!g->votes_ready || g->votes_generation != g->generation) {
        g->err = std::string(fn) + ": no votes of the grid's current state (an integrate, edit or clear, or an "
                                   "earlier resolve, followed the votes)";
        return -1;
    }
    g->votes_ready = false;
    auto fail = [&](const char *what, cudaError_t e) {
        g->err = std::string(fn) + ": " + what + ": " + cudaGetErrorString(e);
        return static_cast<int64_t>(-1);
    };
    cudaError_t e = cudaSetDevice(g->device);
    // host copies of the label images: the map must cover every (instance >= 0, class >= 0) pixel (:322-352)
    const size_t pixels = static_cast<size_t>(width) * height;
    std::vector<int32_t> h_cls(pixels), h_inst(pixels), t(static_cast<size_t>(n_triples) * 3);
    if (e == cudaSuccess) e = cudaMemcpy(h_cls.data(), class_image, pixels * sizeof(int32_t), cudaMemcpyDefault);
    if (e == cudaSuccess) e = cudaMemcpy(h_inst.data(), instance_image, pixels * sizeof(int32_t), cudaMemcpyDefault);
    if (e != cudaSuccess) return fail("label images", e);
    if (n_triples && (e = cudaMemcpy(t.data(), triples, t.size() * sizeof(int32_t), cudaMemcpyDefault)) != cudaSuccess)
        return fail("votes", e);

    // votes: instance id -> (object id -> count), summed over the triples of every rank; pending voxels vote for
    // their instance's NEW object id, handed out here in ascending instance-id order (the reference hands them out in
    // block-iteration order, :118-141).  The counts are integers, so the sums equal the unsharded counts exactly.
    std::map<int32_t, std::map<int32_t, int64_t>> votes;
    std::map<int32_t, int32_t> new_id;
    for (size_t i = 0; i < t.size(); i += 3)
        if (t[i + 1] == kAssocPending) new_id.emplace(t[i], 0);
    for (auto &kv : new_id) kv.second = g->next_object_id++;
    for (size_t i = 0; i < t.size(); i += 3)
        votes[t[i]][t[i + 1] == kAssocPending ? new_id[t[i]] : t[i + 1]] += t[i + 2];
    std::map<int32_t, int32_t> result;
    for (const auto &[inst, ov] : votes) {  // :287-320
        int64_t max_votes = 0, total = 0;
        int32_t winner = -1;
        for (const auto &[obj, cnt] : ov) {
            total += cnt;
            if (cnt > max_votes) {
                max_votes = cnt;
                winner = obj;
            }
        }
        if (total < min_votes || static_cast<float>(max_votes) / static_cast<float>(total) < min_vote_ratio)
            result[inst] = -1;
        else
            result[inst] = winner;
    }
    int32_t prev = -1;   // labelled pixels come in runs of one instance; repeating an entry changes nothing
    for (size_t i = 0; i < pixels; ++i) {  // :322-352: every labelled instance of the image gets an entry
        const int32_t inst = h_inst[i];
        if (inst < 0 || h_cls[i] < 0 || inst == prev) continue;
        prev = inst;
        if (inst == 0)
            result[0] = 0;
        else
            result.try_emplace(inst, -1);   // no node allocated for an instance already present
    }
    for (const auto &[inst, obj] : result) {
        g->map_inst.push_back(inst);
        g->map_obj.push_back(obj);
    }
    // the map on the device, for the deferred assignment below and for b2v_sgrid_remap_instance_ids
    const size_t m = g->map_inst.size();
    if (2 * m > g->d_map.size()) {
        e = cudaStreamSynchronize(g->stream);
        if (e == cudaSuccess) e = g->d_map.reserve(2 * m);
    }
    int32_t *const d_map = g->d_map.get();
    if (e == cudaSuccess && m)
        e = cudaMemcpyAsync(d_map, g->map_inst.data(), m * sizeof(int32_t), cudaMemcpyHostToDevice, g->stream);
    if (e == cudaSuccess && m)
        e = cudaMemcpyAsync(d_map + m, g->map_obj.data(), m * sizeof(int32_t), cudaMemcpyHostToDevice, g->stream);
    if (e == cudaSuccess && !new_id.empty() && g->votes_blocks > 0) {  // deferred assignment of this grid's pending voxels
        ++g->generation;
        sgrid_dispatch(g, [&](auto l, auto c) {
            sem_assoc_apply_kernel<decltype(l)::value, decltype(c)::value>
                <<<g->voxel_ctas(g->votes_blocks), kVox, 0, g->stream>>>(g->dev(), g->d_pend.get(), d_map, d_map + m,
                                                                        static_cast<int>(m),
                                                                        g->votes_blocks * g->block_voxels(),
                                                                        g->labels());
        });
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(g->stream);
    if (e != cudaSuccess) return fail("instance map", e);
    g->has_instance_map = true;
    return static_cast<int64_t>(m);
}

extern "C" int64_t b2v_sgrid_assoc_resolve(b2v_sgrid *g, const int32_t *triples, int64_t n_triples, int32_t width,
                                           int32_t height, const int32_t *class_image, const int32_t *instance_image,
                                           float min_vote_ratio, int32_t min_votes) {
    if (!g) return -1;
    return sgrid_assoc_resolve(g, "b2v_sgrid_assoc_resolve", triples, n_triples, width, height, class_image,
                               instance_image, min_vote_ratio, min_votes);
}

// the unsharded association: the votes, then the resolve of this grid's own triples
extern "C" int64_t b2v_sgrid_assign_object_ids_to_instance_ids(
    b2v_sgrid *g, const float K[4], int32_t width, int32_t height, const double Tcw[16], float depth_max,
    float depth_min, const int32_t *class_image, const int32_t *instance_image, const float *depth_image,
    float depth_threshold, int32_t do_carving, float min_vote_ratio, int32_t min_votes) {
    if (!g) return -1;
    const char *fn = "b2v_sgrid_assign_object_ids_to_instance_ids";
    const int64_t n = sgrid_assoc_votes(g, fn, K, width, height, Tcw, depth_max, depth_min, class_image,
                                        instance_image, depth_image, depth_threshold, do_carving);
    if (n < 0) return -1;
    return sgrid_assoc_resolve(g, fn, g->d_triples.get(), n, width, height, class_image, instance_image, min_vote_ratio,
                               min_votes);
}

extern "C" int b2v_sgrid_set_rectification(b2v_sgrid *g, const float *map_x, const float *map_y, int32_t height,
                                           int32_t width, int32_t swap_rb) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->set_rectification(map_x, map_y, height, width, swap_rb);
}

extern "C" int b2v_sgrid_set_frame(b2v_sgrid *g, const void *depth, int32_t depth_u16, float depth_scale,
                                   const uint8_t *color, const int32_t *class_image, const int32_t *instance_image,
                                   int32_t height, int32_t width, int32_t filter_shadow_points, b2v_frame *out) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->set_frame(depth, depth_u16 != 0, depth_scale, color, class_image, instance_image, height, width,
                        filter_shadow_points != 0, out);
}

extern "C" int b2v_sgrid_set_frame_store(b2v_sgrid *g, int32_t max_frames) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->set_frame_store(max_frames);
}

extern "C" int b2v_sgrid_frame_store_clear(b2v_sgrid *g) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->set_frame_store(g->frame_store.max);
}

extern "C" int b2v_sgrid_frame_store_last(b2v_sgrid *g, int32_t *slot) {
    if (!g || !slot) return B2V_ERR_INVALID_ARGUMENT;
    *slot = g->frame_store.last.empty() ? -1 : g->frame_store.last[0];
    return B2V_OK;
}

extern "C" int b2v_sgrid_frame_store_stats(b2v_sgrid *g, int64_t *frames, int64_t *bytes) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (frames) *frames = g->frame_store.count;
    if (bytes) *bytes = static_cast<int64_t>(g->frame_store.range.mapped);
    return B2V_OK;
}

extern "C" int b2v_sgrid_stage_stored(b2v_sgrid *g, int32_t slot, b2v_frame *out) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    return g->stage_stored(slot, out);
}

extern "C" int b2v_sgrid_remap_instance_ids(b2v_sgrid *g, const int32_t **object_image) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    const b2v_frame &f = g->frame.staged;
    if (!object_image || !f.instance_image || !g->has_instance_map) {
        g->err = !g->has_instance_map ? "b2v_sgrid_remap_instance_ids: no instance map (run an association first)"
                                      : "b2v_sgrid_remap_instance_ids: no staged instance image";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    B2V_CUDA(g, cudaSetDevice(g->device));
    const size_t m = g->map_inst.size();   // the association left its map in d_map
    B2V_CUDA(g, launch_remap_instance_ids(f.instance_image, static_cast<size_t>(f.height) * f.width, g->d_map.get(),
                                          g->d_map.get() + m, static_cast<int>(m), g->frame.obj.get(), g->stream));
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    *object_image = g->frame.obj.get();
    return B2V_OK;
}

extern "C" int b2v_sgrid_copy_instance_map(b2v_sgrid *g, int32_t *instance_ids, int32_t *object_ids) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    for (size_t i = 0; i < g->map_inst.size(); ++i) {
        if (instance_ids) instance_ids[i] = g->map_inst[i];
        if (object_ids) object_ids[i] = g->map_obj[i];
    }
    return B2V_OK;
}

// ---- raw block export / upload (map state) --------------------------------------------------------------------------
extern "C" int64_t b2v_sgrid_export_blocks(b2v_sgrid *g, int32_t *keys4, int32_t *count, double *pos_sum, float *col_sum,
                                           int32_t *object_id, int32_t *class_id, int32_t *counter, float *ml_logp,
                                           float *conf, int32_t *lab_obj, int32_t *lab_cls, float *lab_logp) {
    if (!g) return -1;
    const int64_t nb = b2v_sgrid_num_blocks(g);
    if (nb <= 0) return nb;
    void *const out[kSemArrays] = {count, pos_sum, col_sum, object_id, class_id, counter, ml_logp, conf,
                                   lab_obj, lab_cls, lab_logp};
    SemArray arr[kSemArrays];
    const int na = sgrid_arrays(g, arr);
    cudaError_t e = cudaSuccess;
    if (keys4)
        e = cudaMemcpyAsync(keys4, g->index.block_keys, static_cast<size_t>(nb) * sizeof(int4), cudaMemcpyDeviceToHost,
                            g->stream);
    for (int k = 0; k < na && e == cudaSuccess; ++k)
        if (out[k])
            e = cudaMemcpyAsync(out[k], *arr[k].ptr, static_cast<size_t>(nb) * g->block_voxels() * arr[k].voxel_bytes,
                                cudaMemcpyDeviceToHost, g->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(g->stream);
    if (e != cudaSuccess) {
        g->err = std::string("b2v_sgrid_export_blocks: ") + cudaGetErrorString(e);
        return -1;
    }
    return nb;
}

extern "C" int b2v_sgrid_upload_blocks(b2v_sgrid *g, int64_t n_blocks, const int32_t *keys4, const int32_t *count,
                                       const double *pos_sum, const float *col_sum, const int32_t *object_id,
                                       const int32_t *class_id, const int32_t *counter, const float *ml_logp,
                                       const float *conf, const int32_t *lab_obj, const int32_t *lab_cls,
                                       const float *lab_logp) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    const void *const in[kSemArrays] = {count, pos_sum, col_sum, object_id, class_id, counter, ml_logp, conf,
                                        lab_obj, lab_cls, lab_logp};
    SemArray arr[kSemArrays];
    const int na = sgrid_arrays(g, arr);
    bool bad = n_blocks < 0 || n_blocks > INT32_MAX || (n_blocks > 0 && !keys4);
    for (int k = 0; k < na; ++k) bad = bad || (n_blocks > 0 && !in[k]);
    if (bad) {
        g->err = "b2v_sgrid_upload_blocks: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    // the uploaded voxels are a new state: votes taken before are stale and remap_instance_ids needs a new association
    ++g->generation;
    g->has_instance_map = false;
    if (n_blocks == 0) return B2V_OK;
    B2V_CUDA(g, cudaSetDevice(g->device));
    BlockArrays a{};
    a.n_arrays = na;
    for (int k = 0; k < na; ++k) {
        a.dst[k] = *arr[k].ptr;
        a.src[k] = in[k];
        a.block_bytes[k] = static_cast<uint32_t>(arr[k].voxel_bytes * g->block_voxels());
    }
    int rc = g->upload_blocks(n_blocks, keys4, a, sgrid_grow_storage(g), [&](uint32_t lo, uint32_t hi) {
        // the cleared state for the voxels that just got storage
        sem_fill_kernel<<<592, 256, 0, g->stream>>>(g->dev(), static_cast<size_t>(lo) * g->block_voxels(),
                                                    static_cast<size_t>(hi) * g->block_voxels());
        B2V_CUDA(g, cudaGetLastError());
        return B2V_OK;
    });
    if (rc != B2V_OK) return rc;
    if (g->lab_max_chunks) {   // the uploaded voxels hold their in-voxel pairs only until b2v_sgrid_upload_labels
        rc = sgrid_set_labels(g, "b2v_sgrid_upload_blocks", n_blocks, keys4, nullptr, nullptr, nullptr, nullptr);
        if (rc != B2V_OK) return rc;
    }
    return g->read_counters();
}

// ---- overflow label pairs of the map state ------------------------------------------------------------------------
// Host copies of what the label store's host passes read: per-voxel counters and chain heads of the nb blocks in use,
// the store's counters, every chunk ever taken and the free list.
struct LabelHost {
    int64_t nb = 0;
    std::vector<int32_t> counter;
    std::vector<uint32_t> head, free_list;
    std::vector<LabelChunk> chunks;
    uint32_t ctr[kLcNum] = {};
};

static int sgrid_fetch_labels(b2v_sgrid *g, LabelHost *h) {
    h->nb = b2v_sgrid_num_blocks(g);
    if (h->nb < 0) return B2V_ERR_CUDA;
    const size_t nv = static_cast<size_t>(h->nb) * g->block_voxels();
    h->counter.resize(nv);
    h->head.resize(nv);
    B2V_CUDA(g, cudaMemcpyAsync(h->ctr, g->d_lab_ctr.get(), sizeof(h->ctr), cudaMemcpyDeviceToHost, g->stream));
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    h->chunks.resize(h->ctr[kLcFresh]);
    h->free_list.resize(h->ctr[kLcFree]);
    if (nv) {
        B2V_CUDA(g, cudaMemcpyAsync(h->counter.data(), g->G.counter, nv * sizeof(int32_t), cudaMemcpyDeviceToHost,
                                    g->stream));
        B2V_CUDA(g, cudaMemcpyAsync(h->head.data(), reinterpret_cast<const void *>(g->lab_head.va),
                                    nv * sizeof(uint32_t), cudaMemcpyDeviceToHost, g->stream));
    }
    if (!h->chunks.empty())
        B2V_CUDA(g, cudaMemcpyAsync(h->chunks.data(), reinterpret_cast<const void *>(g->lab_chunks.va),
                                    h->chunks.size() * sizeof(LabelChunk), cudaMemcpyDeviceToHost, g->stream));
    if (!h->free_list.empty())
        B2V_CUDA(g, cudaMemcpyAsync(h->free_list.data(), reinterpret_cast<const void *>(g->lab_free.va),
                                    h->free_list.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, g->stream));
    B2V_CUDA(g, cudaStreamSynchronize(g->stream));
    return B2V_OK;
}

// The uploaded blocks `keys4` [n][4] that the grid holds get their overflow pairs: each voxel's chain goes back to the
// pool, its counter keeps its in-voxel pairs (at most B2V_SEM_MAX_LABELS) and, if n_over is not NULL, it takes a new
// chain of n_over[voxel] pairs from obj / cls / logp (slot order; the pairs of blocks the grid does not hold are
// skipped).  Checks first and changes nothing on a bad argument or when the pool's ceiling cannot hold the pairs.
static int sgrid_set_labels(b2v_sgrid *g, const char *fn, int64_t n_blocks, const int32_t *keys4, const int32_t *n_over,
                            const int32_t *obj, const int32_t *cls, const float *logp) {
    const size_t nvb = g->block_voxels();
    LabelHost h;
    int rc = sgrid_fetch_labels(g, &h);
    if (rc != B2V_OK) return rc;
    // pool index of every block in use, by key
    std::vector<int4> hk(static_cast<size_t>(h.nb));
    if (h.nb) {
        B2V_CUDA(g, cudaMemcpy(hk.data(), g->index.block_keys, hk.size() * sizeof(int4), cudaMemcpyDeviceToHost));
    }
    std::map<std::tuple<int32_t, int32_t, int32_t>, uint32_t> pool;
    for (int64_t b = 0; b < h.nb; ++b) pool[{hk[b].x, hk[b].y, hk[b].z}] = static_cast<uint32_t>(b);
    std::vector<int64_t> idx(static_cast<size_t>(n_blocks), -1);
    for (int64_t b = 0; b < n_blocks; ++b) {
        const auto it = pool.find({keys4[4 * b], keys4[4 * b + 1], keys4[4 * b + 2]});
        if (it != pool.end()) idx[b] = it->second;
    }
    // checks: counts, and the chunks the new chains need against what the pool can give once the old ones are back
    uint64_t need = 0, released = 0;
    for (int64_t b = 0; b < n_blocks; ++b)
        for (size_t t = 0; t < nvb; ++t) {
            const int32_t m = n_over ? n_over[b * nvb + t] : 0;
            if (m < 0 || (m > 0 && idx[b] >= 0 && h.counter[idx[b] * nvb + t] < kSemLabels)) {
                g->err = std::string(fn) + ": overflow pairs of a voxel without " + std::to_string(kSemLabels) +
                         " in-voxel pairs, or a negative count";
                return B2V_ERR_INVALID_ARGUMENT;
            }
            if (idx[b] < 0) continue;
            need += (static_cast<uint64_t>(m) + kChunkPairs - 1) / kChunkPairs;
            for (uint32_t l = h.head[idx[b] * nvb + t]; l != 0; l = h.chunks[l - 1].next) ++released;
        }
    if (need > static_cast<uint64_t>(h.ctr[kLcFree]) + released + (g->lab_max_chunks - h.ctr[kLcFresh])) {
        g->err = std::string(fn) + ": label storage full";
        return B2V_ERR_CAPACITY;
    }
    // release, then new chains: chunks from the free list first, then fresh ones
    size_t pos = 0;
    for (int64_t b = 0; b < n_blocks; ++b)
        for (size_t t = 0; t < nvb; ++t) {
            const int32_t m = n_over ? n_over[b * nvb + t] : 0;
            if (idx[b] < 0) {
                pos += static_cast<size_t>(m);
                continue;
            }
            const size_t v = idx[b] * nvb + t;
            for (uint32_t l = h.head[v]; l != 0; l = h.chunks[l - 1].next) h.free_list.push_back(l - 1);
            h.head[v] = 0;
            h.counter[v] = std::min(h.counter[v], static_cast<int32_t>(kSemLabels)) + m;
            uint32_t tail = 0;
            for (int32_t e = 0; e < m; ++e, ++pos) {
                if (e % kChunkPairs == 0) {
                    uint32_t c;
                    if (!h.free_list.empty()) {
                        c = h.free_list.back();
                        h.free_list.pop_back();
                    } else {
                        c = static_cast<uint32_t>(h.chunks.size());
                        h.chunks.emplace_back();
                    }
                    h.chunks[c] = LabelChunk{};
                    if (tail) h.chunks[tail - 1].next = c + 1;
                    else h.head[v] = c + 1;
                    tail = c + 1;
                }
                LabelChunk &c = h.chunks[tail - 1];
                c.obj[e % kChunkPairs] = obj[pos];
                c.cls[e % kChunkPairs] = cls[pos];
                c.logp[e % kChunkPairs] = logp[pos];
            }
        }
    if (h.chunks.size() > g->lab_mapped) {   // a growth of the chunk storage, counted as the runs' growths are
        const uint32_t old = g->lab_mapped;
        std::string map_err;
        if (!sgrid_map_labels(g, h.chunks.size(), &map_err)) {
            g->err = std::string(fn) + ": label storage could not grow: " + map_err;
            return B2V_ERR_CUDA;
        }
        if (g->lab_mapped > old) ++g->lab_growths;
    }
    h.ctr[kLcFree] = static_cast<uint32_t>(h.free_list.size());
    h.ctr[kLcFresh] = static_cast<uint32_t>(h.chunks.size());
    const size_t nv = h.counter.size();
    if (nv) {
        B2V_CUDA(g, cudaMemcpy(g->G.counter, h.counter.data(), nv * sizeof(int32_t), cudaMemcpyHostToDevice));
        B2V_CUDA(g, cudaMemcpy(reinterpret_cast<void *>(g->lab_head.va), h.head.data(), nv * sizeof(uint32_t),
                               cudaMemcpyHostToDevice));
    }
    if (!h.chunks.empty())
        B2V_CUDA(g, cudaMemcpy(reinterpret_cast<void *>(g->lab_chunks.va), h.chunks.data(),
                               h.chunks.size() * sizeof(LabelChunk), cudaMemcpyHostToDevice));
    if (!h.free_list.empty())
        B2V_CUDA(g, cudaMemcpy(reinterpret_cast<void *>(g->lab_free.va), h.free_list.data(),
                               h.free_list.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    B2V_CUDA(g, cudaMemcpy(g->d_lab_ctr.get(), h.ctr, sizeof(h.ctr), cudaMemcpyHostToDevice));
    return B2V_OK;
}

extern "C" int64_t b2v_sgrid_export_labels(b2v_sgrid *g, int32_t *n_over, int32_t *obj, int32_t *cls, float *logp) {
    if (!g) return -1;
    const size_t nvb = g->block_voxels();
    if (g->lab_max_chunks == 0) {   // no store: no overflow pairs
        const int64_t nb = b2v_sgrid_num_blocks(g);
        if (nb > 0 && n_over) std::fill(n_over, n_over + static_cast<size_t>(nb) * nvb, 0);
        return nb < 0 ? -1 : 0;
    }
    LabelHost h;
    if (sgrid_fetch_labels(g, &h) != B2V_OK) return -1;
    int64_t total = 0;
    for (size_t v = 0; v < h.counter.size(); ++v) {
        const int32_t m = h.counter[v] > kSemLabels ? h.counter[v] - kSemLabels : 0;
        if (n_over) n_over[v] = m;
        int32_t e = 0;
        for (uint32_t l = h.head[v]; l != 0 && e < m; l = h.chunks[l - 1].next)
            for (int k = 0; k < kChunkPairs && e < m; ++k, ++e) {
                if (obj) obj[total + e] = h.chunks[l - 1].obj[k];
                if (cls) cls[total + e] = h.chunks[l - 1].cls[k];
                if (logp) logp[total + e] = h.chunks[l - 1].logp[k];
            }
        total += m;
    }
    return total;
}

extern "C" int b2v_sgrid_upload_labels(b2v_sgrid *g, int64_t n_blocks, const int32_t *keys4, const int32_t *n_over,
                                       const int32_t *obj, const int32_t *cls, const float *logp) {
    if (!g) return B2V_ERR_INVALID_ARGUMENT;
    if (n_blocks < 0 || (n_blocks > 0 && (!keys4 || !n_over))) {
        g->err = "b2v_sgrid_upload_labels: bad arguments";
        return B2V_ERR_INVALID_ARGUMENT;
    }
    const size_t nv = static_cast<size_t>(n_blocks) * g->block_voxels();
    int64_t total = 0;
    for (size_t v = 0; v < nv; ++v) total += n_over[v] > 0 ? n_over[v] : 0;
    if (total == 0) return B2V_OK;
    if (g->lab_max_chunks == 0 || !obj || !cls || !logp) {
        g->err = g->lab_max_chunks == 0 ? "b2v_sgrid_upload_labels: overflow pairs for a grid without a label store"
                                        : "b2v_sgrid_upload_labels: bad arguments";
        return g->lab_max_chunks == 0 ? B2V_ERR_CAPACITY : B2V_ERR_INVALID_ARGUMENT;
    }
    B2V_CUDA(g, cudaSetDevice(g->device));
    ++g->generation;
    return sgrid_set_labels(g, "b2v_sgrid_upload_labels", n_blocks, keys4, n_over, obj, cls, logp);
}
