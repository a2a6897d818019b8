// b2v_prep.cu — per-frame depth preparation on the GPU (SURVEY.md §8 row a2, "next" row f#1).
//
// filter_shadow_points (pyslam/utilities/depth.py:103-146): remove the ghost points on depth
// discontinuities.  delta_y = |d[r+2,c] - d[r,c]|, delta_x = |d[r,c+2] - d[r,c]|; the threshold is
// 3 * 1.4826 * median(all positive deltas) (float32 arithmetic, like numpy on float32 input); a pixel is
// set to fill_value if any delta it takes part in exceeds the threshold.
//
// The global median is an exact order statistic: a 3-pass radix select over the float bit patterns
// (positive floats order like their bits), entirely on the device.  For an even count numpy averages the
// two middle elements in float32; both ranks are selected in the same passes.
#include "b2v_internal.h"

namespace b2v {

struct SelectState {
    uint32_t prefix[2];  // bits fixed so far, for rank 0 (lower middle) and rank 1 (upper middle)
    uint32_t rank[2];    // residual rank inside the prefix bucket
    uint32_t total;      // number of positive deltas
    float threshold;     // 3 * 1.4826 * median
};

__device__ __forceinline__ bool delta_at(const float *__restrict__ d, int H, int W, int dx, int dy, int64_t i,
                                         float *out) {
    // index space: first the (H - dy) * W vertical deltas, then the H * (W - dx) horizontal ones
    const int64_t ny = dy > 0 ? static_cast<int64_t>(H - dy) * W : 0;
    if (i < ny) {
        *out = fabsf(__fsub_rn(d[i + static_cast<int64_t>(dy) * W], d[i]));
        return true;
    }
    const int64_t j = i - ny;
    const int wx = W - dx;
    if (dx > 0 && j < static_cast<int64_t>(H) * wx) {
        const int r = static_cast<int>(j / wx), c = static_cast<int>(j % wx);
        const int64_t p = static_cast<int64_t>(r) * W + c;
        *out = fabsf(__fsub_rn(d[p + dx], d[p]));
        return true;
    }
    return false;
}

// pass p in {0,1,2}: digit widths 11, 11, 10 bits from the top
__device__ __forceinline__ void digit_layout(int pass, int *shift, uint32_t *nbins, uint32_t *hi_mask) {
    if (pass == 0) {
        *shift = 21;
        *nbins = 2048;
        *hi_mask = 0u;
    } else if (pass == 1) {
        *shift = 10;
        *nbins = 2048;
        *hi_mask = 0xFFE00000u;
    } else {
        *shift = 0;
        *nbins = 1024;
        *hi_mask = 0xFFFFFC00u;
    }
}

__global__ void __launch_bounds__(256)
shadow_hist_kernel(const float *__restrict__ depth, int H, int W, int dx, int dy, int pass,
                   const SelectState *__restrict__ st, uint32_t *__restrict__ hist) {
    // per-CTA histograms in shared memory (the positive deltas of an image crowd into a few bins: global atomics
    // on them serialise), flushed once
    __shared__ uint32_t s_h[4096];
    for (int i = threadIdx.x; i < 4096; i += blockDim.x) s_h[i] = 0u;
    __syncthreads();
    int shift;
    uint32_t nbins, hi_mask;
    digit_layout(pass, &shift, &nbins, &hi_mask);
    const int64_t n = (dy > 0 ? static_cast<int64_t>(H - dy) * W : 0) + (dx > 0 ? static_cast<int64_t>(H) * (W - dx) : 0);
    const uint32_t p0 = pass ? st->prefix[0] : 0u, p1 = pass ? st->prefix[1] : 0u;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        float v;
        if (!delta_at(depth, H, W, dx, dy, i, &v) || !(v > 0.0f)) continue;  // delta_values[delta_values > 0]
        const uint32_t bits = __float_as_uint(v);
        const uint32_t digit = (bits >> shift) & (nbins - 1);
        if ((bits & hi_mask) == p0) atomicAdd(s_h + digit, 1u);
        if ((bits & hi_mask) == p1) atomicAdd(s_h + 2048 + digit, 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 4096; i += blockDim.x)
        if (s_h[i]) atomicAdd(hist + i, s_h[i]);
}

// one block: walk the two histograms, fix the next digit of both ranks, clear the histograms.  The walk is a
// block-wide scan: thread t owns 8 consecutive bins of each histogram.
__global__ void __launch_bounds__(256)
shadow_pick_kernel(int pass, SelectState *st, uint32_t *hist) {
    __shared__ uint32_t s_part[2][256];
    __shared__ uint32_t s_total;
    int shift;
    uint32_t nbins, hi_mask;
    digit_layout(pass, &shift, &nbins, &hi_mask);
    const int t = threadIdx.x;
    uint32_t mine[2][8];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        uint32_t sum = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t b = static_cast<uint32_t>(t) * 8u + j;
            mine[k][j] = b < nbins ? hist[2048 * k + b] : 0u;
            sum += mine[k][j];
        }
        s_part[k][t] = sum;
    }
    __syncthreads();
    if (t == 0) {  // 256 partial sums: exclusive prefixes in place (tiny, serial)
        for (int k = 0; k < 2; ++k) {
            uint32_t run = 0;
            for (int i = 0; i < 256; ++i) {
                const uint32_t v = s_part[k][i];
                s_part[k][i] = run;
                run += v;
            }
            if (k == 0) s_total = run;
        }
        if (pass == 0) {
            const uint32_t total = s_total;
            st->total = total;
            st->rank[0] = total ? (total - 1) / 2 : 0;  // numpy median: mean of elements (n-1)//2 and n//2
            st->rank[1] = total / 2;
            st->prefix[0] = st->prefix[1] = 0;
        }
    }
    __syncthreads();
    const uint32_t ranks[2] = {st->rank[0], st->rank[1]};
    __syncthreads();  // every thread has read the ranks before the owner of the crossing bin rewrites them
    // the bin b with  sum(h[0..b)) <= rank < sum(h[0..b]), or the last bin (the serial walk's stopping rule)
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const uint32_t r = ranks[k];
        uint32_t before = s_part[k][t];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t b = static_cast<uint32_t>(t) * 8u + j;
            if (b < nbins) {
                const bool last = b + 1 == nbins;
                if (r >= before && (r < before + mine[k][j] || last)) {
                    st->rank[k] = r - before;
                    st->prefix[k] |= b << shift;
                }
            }
            before += mine[k][j];
        }
    }
    __syncthreads();
    if (t == 0 && pass == 2) {
        const float a = __uint_as_float(st->prefix[0]), b = __uint_as_float(st->prefix[1]);
        // np.median -> mean of the two middle values in float32; then float32(1.4826) * mad; then 3 * sigma
        const float mad = st->total ? __fmul_rn(__fadd_rn(a, b), 0.5f) : __uint_as_float(0x7FC00000u);
        st->threshold = __fmul_rn(3.0f, __fmul_rn(1.4826f, mad));
    }
    for (uint32_t i = threadIdx.x; i < 4096; i += blockDim.x) hist[i] = 0;
}

__global__ void shadow_mask_kernel(const float *__restrict__ depth, int H, int W, int dx, int dy, float fill,
                                   const SelectState *__restrict__ st, float *__restrict__ out) {
    const int64_t n = static_cast<int64_t>(H) * W;
    const float thr = st->threshold;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int r = static_cast<int>(i / W), c = static_cast<int>(i % W);
        const float d = depth[i];
        bool m = false;
        if (dy > 0) {
            if (r >= dy) m |= fabsf(__fsub_rn(d, depth[i - static_cast<int64_t>(dy) * W])) > thr;
            if (r < H - dy) m |= fabsf(__fsub_rn(depth[i + static_cast<int64_t>(dy) * W], d)) > thr;
        }
        if (dx > 0) {
            if (c >= dx) m |= fabsf(__fsub_rn(d, depth[i - dx])) > thr;
            if (c < W - dx) m |= fabsf(__fsub_rn(depth[i + dx], d)) > thr;
        }
        out[i] = m ? fill : d;
    }
}

// scratch: sizeof(SelectState) + 4096 * 4 bytes of device memory, zero-initialised by the caller once
cudaError_t launch_filter_shadow_points(const float *depth, int H, int W, int dx, int dy, float fill, float *out,
                                        void *scratch, cudaStream_t stream) {
    SelectState *st = static_cast<SelectState *>(scratch);
    uint32_t *hist = reinterpret_cast<uint32_t *>(static_cast<char *>(scratch) + 64);
    cudaError_t e = cudaMemsetAsync(scratch, 0, 64 + 4096 * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    for (int pass = 0; pass < 3; ++pass) {
        shadow_hist_kernel<<<296, 256, 0, stream>>>(depth, H, W, dx, dy, pass, st, hist);
        shadow_pick_kernel<<<1, 256, 0, stream>>>(pass, st, hist);
    }
    shadow_mask_kernel<<<296, 256, 0, stream>>>(depth, H, W, dx, dy, fill, st, out);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// undistort / rectify: cv2.remap with the precomputed maps of initUndistortRectifyMap
// (pyslam/dense/volumetric_integrator_base.py:1017-1054: colour INTER_LINEAR, depth and labels
// INTER_NEAREST, constant zero border).  OpenCV's fixed-point arithmetic is reproduced exactly:
//   linear (8-bit): sx = round_half_even(mapx * 32), pixel = sx >> 5, fraction a = sx & 31;
//                   weights (32-ay)(32-ax)*32, ... (sum 32768); out = (sum w*p + 16384) >> 15
//   nearest:        pixel = round_half_even(mapx)
// A NaN map coordinate converts to INT_MIN, as OpenCV's cvRound does on x86 (cvtss2si), so the pixel lies outside
// the image and takes the zero border; the PTX conversion alone would give 0 and read column / row 0.
// ------------------------------------------------------------------------------------------------
constexpr int kNanMapCoord = INT_MIN;

__global__ void remap_u8c3_linear_kernel(const uint8_t *__restrict__ src, int H, int W,
                                         const float *__restrict__ mapx, const float *__restrict__ mapy,
                                         uint8_t *__restrict__ dst, int swap_rb) {
    const int64_t n = static_cast<int64_t>(H) * W;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const float fx = __fmul_rn(mapx[i], 32.0f), fy = __fmul_rn(mapy[i], 32.0f);
        const int sx = isnan(fx) ? kNanMapCoord : __float2int_rn(fx), sy = isnan(fy) ? kNanMapCoord : __float2int_rn(fy);
        const int x0 = sx >> 5, y0 = sy >> 5, ax = sx & 31, ay = sy & 31;
        const int w00 = (32 - ay) * (32 - ax) * 32, w01 = (32 - ay) * ax * 32, w10 = ay * (32 - ax) * 32,
                  w11 = ay * ax * 32;
        int acc[3] = {16384, 16384, 16384};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int x = x0 + (t & 1), y = y0 + (t >> 1);
            const int w = t == 0 ? w00 : (t == 1 ? w01 : (t == 2 ? w10 : w11));
            if (x >= 0 && x < W && y >= 0 && y < H && w) {  // BORDER_CONSTANT, value 0
                const uint8_t *p = src + (static_cast<int64_t>(y) * W + x) * 3;
                acc[0] += w * p[0];
                acc[1] += w * p[1];
                acc[2] += w * p[2];
            }
        }
        uint8_t *o = dst + i * 3;
        o[swap_rb ? 2 : 0] = static_cast<uint8_t>(acc[0] >> 15);
        o[1] = static_cast<uint8_t>(acc[1] >> 15);
        o[swap_rb ? 0 : 2] = static_cast<uint8_t>(acc[2] >> 15);
    }
}

__global__ void remap_b32_nearest_kernel(const uint32_t *__restrict__ src, int H, int W,
                                         const float *__restrict__ mapx, const float *__restrict__ mapy,
                                         uint32_t *__restrict__ dst) {
    const int64_t n = static_cast<int64_t>(H) * W;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int x = isnan(mapx[i]) ? kNanMapCoord : __float2int_rn(mapx[i]),
                  y = isnan(mapy[i]) ? kNanMapCoord : __float2int_rn(mapy[i]);
        dst[i] = (x >= 0 && x < W && y >= 0 && y < H) ? src[static_cast<int64_t>(y) * W + x] : 0u;
    }
}

// raw 16-bit depth -> metres: float(u16) * scale, one float32 rounding (numpy: depth.astype(float32) * factor)
__global__ void depth_u16_to_f32_kernel(const uint16_t *__restrict__ src, float *__restrict__ dst, const size_t n,
                                        const float scale) {
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<size_t>(gridDim.x) * blockDim.x)
        dst[i] = __fmul_rn(static_cast<float>(src[i]), scale);
}

// instance id -> object id of the last association; one binary search over the sorted map per pixel
__global__ void remap_instance_ids_kernel(const int32_t *__restrict__ src, const size_t n,
                                          const int32_t *__restrict__ map_inst, const int32_t *__restrict__ map_obj,
                                          const int n_map, int32_t *__restrict__ dst) {
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int32_t id = src[i];
        int32_t out = -1;
        int lo = 0, hi = n_map - 1;
        while (lo <= hi) {
            const int mid = (lo + hi) >> 1;
            const int32_t m = __ldg(map_inst + mid);
            if (m == id) {
                out = __ldg(map_obj + mid);
                break;
            }
            if (m < id) lo = mid + 1; else hi = mid - 1;
        }
        dst[i] = out;
    }
}

// ------------------------------------------------------------------------------------------------
// frame-store records of the grids (b2v_internal.h, launch_grid_frame_pack): one thread per group of 4 pixels, with
// 16-byte loads and stores of depth, filtered depth, labels and records (colour: three 4-byte words); the pixels of a
// last partial group one by one.  Word 1 of a record: r | g << 8 | b << 16 | flags << 24.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t record_word1(float d, float f, uint32_t rgb) {
    return rgb | (__float_as_uint(f) != __float_as_uint(d) ? 1u << 24 : 0u);
}

template <bool Labels>
__global__ void __launch_bounds__(256)
grid_frame_pack_kernel(const float *__restrict__ depth, const float *__restrict__ filtered,
                       const uint8_t *__restrict__ rgb, const int32_t *__restrict__ cls,
                       const int32_t *__restrict__ inst, const size_t n, uint32_t *__restrict__ rec) {
    constexpr int kWords = Labels ? 4 : 2;   // record words per pixel
    const size_t groups = (n + 3) / 4;
    for (size_t q = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; q < groups;
         q += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t p0 = 4 * q;
        uint32_t *r = rec + p0 * kWords;
        if (p0 + 4 <= n) {
            const float4 d = __ldg(reinterpret_cast<const float4 *>(depth + p0));
            const float4 f = filtered ? __ldg(reinterpret_cast<const float4 *>(filtered + p0)) : d;
            const uint32_t *cw = reinterpret_cast<const uint32_t *>(rgb + 3 * p0);
            const uint32_t w0 = __ldg(cw), w1 = __ldg(cw + 1), w2 = __ldg(cw + 2);
            const uint32_t c0 = w0 & 0xFFFFFFu, c1 = (w0 >> 24) | ((w1 & 0xFFFFu) << 8),
                           c2 = (w1 >> 16) | ((w2 & 0xFFu) << 16), c3 = w2 >> 8;
            const uint4 a = make_uint4(__float_as_uint(d.x), record_word1(d.x, f.x, c0), __float_as_uint(d.y),
                                       record_word1(d.y, f.y, c1));
            const uint4 b = make_uint4(__float_as_uint(d.z), record_word1(d.z, f.z, c2), __float_as_uint(d.w),
                                       record_word1(d.w, f.w, c3));
            if constexpr (Labels) {
                if (cls) {
                    const int4 k = __ldg(reinterpret_cast<const int4 *>(cls + p0));
                    const int4 m = inst ? __ldg(reinterpret_cast<const int4 *>(inst + p0)) : make_int4(0, 0, 0, 0);
                    uint4 *o = reinterpret_cast<uint4 *>(r);
                    o[0] = make_uint4(a.x, a.y, k.x, m.x);
                    o[1] = make_uint4(a.z, a.w, k.y, m.y);
                    o[2] = make_uint4(b.x, b.y, k.z, m.z);
                    o[3] = make_uint4(b.z, b.w, k.w, m.w);
                } else {   // the label half is not written
                    uint2 *o = reinterpret_cast<uint2 *>(r);
                    o[0] = make_uint2(a.x, a.y);
                    o[2] = make_uint2(a.z, a.w);
                    o[4] = make_uint2(b.x, b.y);
                    o[6] = make_uint2(b.z, b.w);
                }
            } else {
                reinterpret_cast<uint4 *>(r)[0] = a;
                reinterpret_cast<uint4 *>(r)[1] = b;
            }
        } else {
            for (size_t p = p0; p < n; ++p, r += kWords) {
                const float d = depth[p], f = filtered ? filtered[p] : d;
                const uint8_t *c = rgb + 3 * p;
                r[0] = __float_as_uint(d);
                r[1] = record_word1(d, f, c[0] | (static_cast<uint32_t>(c[1]) << 8) | (static_cast<uint32_t>(c[2]) << 16));
                if constexpr (Labels) {
                    if (cls) {
                        r[2] = static_cast<uint32_t>(cls[p]);
                        r[3] = inst ? static_cast<uint32_t>(inst[p]) : 0u;
                    }
                }
            }
        }
    }
}

// the bits of the filtered depth: -1.0f where the filter set the pixel, else the depth's bits (NaN payloads included)
__device__ __forceinline__ uint32_t record_filtered(uint32_t w0, uint32_t w1) {
    return (w1 >> 24) & 1u ? 0xBF800000u : w0;
}

template <bool Labels>
__global__ void __launch_bounds__(256)
grid_frame_unpack_kernel(const uint32_t *__restrict__ rec, const size_t n, float *__restrict__ depth,
                         float *__restrict__ filtered, uint8_t *__restrict__ rgb, int32_t *__restrict__ cls,
                         int32_t *__restrict__ inst) {
    constexpr int kWords = Labels ? 4 : 2;
    const size_t groups = (n + 3) / 4;
    for (size_t q = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; q < groups;
         q += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t p0 = 4 * q;
        const uint32_t *r = rec + p0 * kWords;
        if (p0 + 4 <= n) {
            uint4 px[4];   // {depth bits, word 1, class, instance} of each pixel
            if constexpr (Labels) {
                const uint4 *in = reinterpret_cast<const uint4 *>(r);
#pragma unroll
                for (int k = 0; k < 4; ++k) px[k] = __ldg(in + k);
            } else {
                const uint4 a = __ldg(reinterpret_cast<const uint4 *>(r)), b = __ldg(reinterpret_cast<const uint4 *>(r) + 1);
                px[0] = make_uint4(a.x, a.y, 0, 0);
                px[1] = make_uint4(a.z, a.w, 0, 0);
                px[2] = make_uint4(b.x, b.y, 0, 0);
                px[3] = make_uint4(b.z, b.w, 0, 0);
            }
            *reinterpret_cast<uint4 *>(depth + p0) = make_uint4(px[0].x, px[1].x, px[2].x, px[3].x);
            if (filtered)
                *reinterpret_cast<uint4 *>(filtered + p0) =
                    make_uint4(record_filtered(px[0].x, px[0].y), record_filtered(px[1].x, px[1].y),
                                record_filtered(px[2].x, px[2].y), record_filtered(px[3].x, px[3].y));
            const uint32_t c0 = px[0].y & 0xFFFFFFu, c1 = px[1].y & 0xFFFFFFu, c2 = px[2].y & 0xFFFFFFu,
                           c3 = px[3].y & 0xFFFFFFu;
            uint32_t *cw = reinterpret_cast<uint32_t *>(rgb + 3 * p0);
            cw[0] = c0 | (c1 << 24);
            cw[1] = (c1 >> 8) | (c2 << 16);
            cw[2] = (c2 >> 16) | (c3 << 8);
            if constexpr (Labels) {
                if (cls) *reinterpret_cast<uint4 *>(cls + p0) = make_uint4(px[0].z, px[1].z, px[2].z, px[3].z);
                if (inst) *reinterpret_cast<uint4 *>(inst + p0) = make_uint4(px[0].w, px[1].w, px[2].w, px[3].w);
            }
        } else {
            for (size_t p = p0; p < n; ++p, r += kWords) {
                const uint32_t w0 = r[0], w1 = r[1];
                depth[p] = __uint_as_float(w0);
                if (filtered) filtered[p] = __uint_as_float(record_filtered(w0, w1));
                rgb[3 * p] = static_cast<uint8_t>(w1);
                rgb[3 * p + 1] = static_cast<uint8_t>(w1 >> 8);
                rgb[3 * p + 2] = static_cast<uint8_t>(w1 >> 16);
                if constexpr (Labels) {
                    if (cls) cls[p] = static_cast<int32_t>(r[2]);
                    if (inst) inst[p] = static_cast<int32_t>(r[3]);
                }
            }
        }
    }
}

static unsigned record_ctas(size_t pixels) {
    return static_cast<unsigned>(std::min<size_t>((pixels + 4 * 256 - 1) / (4 * 256), 2368));
}

cudaError_t launch_grid_frame_pack(const float *depth, const float *filtered, const uint8_t *rgb, const int32_t *cls,
                                   const int32_t *inst, size_t pixels, bool labels, void *rec, cudaStream_t stream) {
    if (pixels == 0) return cudaSuccess;
    uint32_t *r = static_cast<uint32_t *>(rec);
    if (labels)
        grid_frame_pack_kernel<true><<<record_ctas(pixels), 256, 0, stream>>>(depth, filtered, rgb, cls, inst, pixels, r);
    else
        grid_frame_pack_kernel<false><<<record_ctas(pixels), 256, 0, stream>>>(depth, filtered, rgb, nullptr, nullptr,
                                                                                pixels, r);
    return cudaGetLastError();
}

cudaError_t launch_grid_frame_unpack(const void *rec, size_t pixels, bool labels, float *depth, float *filtered,
                                     uint8_t *rgb, int32_t *cls, int32_t *inst, cudaStream_t stream) {
    if (pixels == 0) return cudaSuccess;
    const uint32_t *r = static_cast<const uint32_t *>(rec);
    if (labels)
        grid_frame_unpack_kernel<true><<<record_ctas(pixels), 256, 0, stream>>>(r, pixels, depth, filtered, rgb, cls,
                                                                                 inst);
    else
        grid_frame_unpack_kernel<false><<<record_ctas(pixels), 256, 0, stream>>>(r, pixels, depth, filtered, rgb,
                                                                                  nullptr, nullptr);
    return cudaGetLastError();
}

cudaError_t launch_remap_instance_ids(const int32_t *src, size_t n, const int32_t *map_inst, const int32_t *map_obj,
                                      int n_map, int32_t *dst, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    remap_instance_ids_kernel<<<1184, 256, 0, stream>>>(src, n, map_inst, map_obj, n_map, dst);
    return cudaGetLastError();
}

cudaError_t launch_depth_u16_to_f32(const uint16_t *src, float *dst, size_t n, float scale, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    depth_u16_to_f32_kernel<<<1184, 256, 0, stream>>>(src, dst, n, scale);
    return cudaGetLastError();
}

cudaError_t launch_remap_u8c3_linear(const uint8_t *src, int H, int W, const float *mapx, const float *mapy,
                                     uint8_t *dst, int swap_rb, cudaStream_t stream) {
    remap_u8c3_linear_kernel<<<296, 256, 0, stream>>>(src, H, W, mapx, mapy, dst, swap_rb);
    return cudaGetLastError();
}

cudaError_t launch_remap_b32_nearest(const void *src, int H, int W, const float *mapx, const float *mapy, void *dst,
                                     cudaStream_t stream) {
    remap_b32_nearest_kernel<<<296, 256, 0, stream>>>(static_cast<const uint32_t *>(src), H, W, mapx, mapy,
                                                      static_cast<uint32_t *>(dst));
    return cudaGetLastError();
}

}  // namespace b2v
