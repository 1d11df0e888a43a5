// annotation.cu -- the per-pixel passes of the reference's imsegm/annotation.py:
//   colour histogram over 2^24 packed-RGB bins and its compaction (unique_image_colors :46-68, image_frequent_colors :163-193,
//   group_images_frequent_colors :196-223)
//   palette exact match / L1-nearest index (convert_img_colors_to_labels[_reverted] :71-125, image_color_2_labels :226-249,
//   quantize_image_nearest_color :252-276, the valid map of quantize_image_nearest_pixel :289-321)
//   label -> colour gather (convert_img_labels_to_colors :128-160 and the last step of both quantisers)
//   value gather at the nearest-site index of isb_edt_2d_indices (image_inpaint_pixels :279-286)
#include <algorithm>
#include <type_traits>

#include "compact.cuh"
#include "run_flush.cuh"

namespace {

constexpr int HIST_PER = 16;             // pixels per thread, consecutive lanes on consecutive pixels
constexpr unsigned FULL = 0xffffffffu;
constexpr unsigned NO_KEY = 0xffffffffu; // past the end of the image (packed colours are < 2^24)
constexpr int PAL_MAX = 1024;
constexpr int PAL_ROW_MAX = 32;          // bytes of one gathered colour: 4 channels of 8 bytes

__device__ __forceinline__ unsigned pixel_key(const uint8_t* __restrict__ img, long long i, int C)
{
    const uint8_t* p = img + i * C;
    if (C == 1) return (unsigned)p[0] * 0x010101u;                  // grey as PIL's convert('RGB') expands it
    return ((unsigned)p[0] << 16) | ((unsigned)p[1] << 8) | p[2];   // the alpha of RGBA does not count
}

// every lane keeps a run of one colour over its pixels, which lie 32 apart (flush_run): a single-colour image issues one atomic per
// 32 * HIST_PER pixels
__global__ void __launch_bounds__(256) k_color_hist(const uint8_t* __restrict__ img, long long n, int C, unsigned long long* __restrict__ hist)
{
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long base = warp * 32LL * HIST_PER + (threadIdx.x & 31);
    if (warp * 32LL * HIST_PER >= n) return;                         // uniform over the warp
    const auto add = [hist](unsigned key, unsigned s) { atomicAdd(hist + key, (unsigned long long)s); };
    unsigned cur = NO_KEY, cnt = 0;
    for (int k = 0; k < HIST_PER; ++k) {
        const long long i = base + 32LL * k;
        const unsigned key = i < n ? pixel_key(img, i, C) : NO_KEY;
        flush_run(key != cur && cnt != 0, cur, cnt, add);
        if (key != cur) { cur = key; cnt = 0; }
        if (key != NO_KEY) ++cnt;
    }
    flush_run(cnt != 0, cur, cnt, add);
}

__global__ void __launch_bounds__(CPT_THREADS) k_hist_write(const unsigned long long* __restrict__ hist, long long n,
                                                            const long long* __restrict__ tile_off, int32_t* __restrict__ colors,
                                                            int64_t* __restrict__ counts)
{
    const long long beg = (long long)blockIdx.x * CPT_TILE + (long long)threadIdx.x * CPT_PER;
    int total;
    long long o = tile_off[blockIdx.x] + cta_exclusive_sum<CPT_THREADS>(thread_count(hist, beg, n), total);
    for (int k = 0; k < CPT_PER; ++k) {
        const long long i = beg + k;
        if (i < n && hist[i]) {
            colors[o] = (int32_t)i;
            counts[o] = (int64_t)hist[i];
            ++o;
        }
    }
}

__device__ __forceinline__ void block_add(unsigned long long v, unsigned long long* __restrict__ total)
{
    for (int o = 16; o; o >>= 1) v += __shfl_down_sync(FULL, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(total, v);
}

// exact (mode 0: the LAST equal entry, -1 when none) or L1-nearest (mode 1: the FIRST entry of least distance) palette index of every
// pixel, then labels = values[index] when a value table is given.  uint8: pixel and entries packed one channel per byte, |a - b|
// summed by __vsadu4 (exact integers).  float64: |p_c - e_c| added channel by channel from 0 as numpy's sum does; a NaN distance
// is the minimum at its first occurrence (np.argmin).
template <typename T>
__global__ void __launch_bounds__(256) k_palette(const T* __restrict__ img, long long n, int C, const T* __restrict__ pal, int P, int mode,
                                                 const int64_t* __restrict__ values, int64_t* __restrict__ labels, uint8_t* __restrict__ matched,
                                                 unsigned long long* __restrict__ unmatched)
{
    constexpr bool U8 = sizeof(T) == 1;
    __shared__ typename std::conditional<U8, unsigned, double>::type sp[U8 ? PAL_MAX : PAL_MAX * 4];
    for (int j = threadIdx.x; j < P; j += blockDim.x) {
        if constexpr (U8) {
            unsigned q = 0;
            for (int c = 0; c < C; ++c) q |= (unsigned)pal[j * C + c] << (8 * c);
            sp[j] = q;
        } else {
            for (int c = 0; c < C; ++c) sp[j * C + c] = pal[j * C + c];
        }
    }
    __syncthreads();
    unsigned long long miss = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        int best = -1;
        if constexpr (U8) {
            unsigned q = 0;
            for (int c = 0; c < C; ++c) q |= (unsigned)img[i * C + c] << (8 * c);
            if (mode == 0) {
                for (int j = P - 1; j >= 0; --j)
                    if (sp[j] == q) { best = j; break; }
            } else {
                unsigned bd = 0xffffffffu;
                for (int j = 0; j < P; ++j) {
                    const unsigned d = __vsadu4(sp[j], q);
                    if (d < bd) { bd = d; best = j; }
                }
            }
        } else {
            double px[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) px[c] = c < C ? img[i * C + c] : 0.0;
            if (mode == 0) {
                for (int j = P - 1; j >= 0 && best < 0; --j) {
                    bool eq = true;
#pragma unroll
                    for (int c = 0; c < 4; ++c) eq = eq && (c >= C || px[c] == sp[j * C + c]);
                    if (eq) best = j;
                }
            } else {
                double bd = 0.0;
                for (int j = 0; j < P; ++j) {
                    double d = 0.0;
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        if (c < C) d += fabs(px[c] - sp[j * C + c]);
                    if (d != d) { best = j; break; }
                    if (best < 0 || d < bd) { bd = d; best = j; }
                }
            }
        }
        labels[i] = best < 0 ? -1 : (values ? values[best] : best);
        if (matched) matched[i] = best >= 0;
        miss += best < 0;
    }
    if (unmatched) block_add(miss, unmatched);
}

// out[i] = table[row of label i]: with keys (sorted, unique) the row whose key equals the label (binary search), without them the
// label itself when 0 <= label < P.  A label without a row writes zeros and is counted in *missing.
__global__ void __launch_bounds__(256) k_palette_gather(const int64_t* __restrict__ labels, long long n, const int64_t* __restrict__ keys, int P,
                                                        const uint8_t* __restrict__ table, int row_bytes, uint8_t* __restrict__ out,
                                                        unsigned long long* __restrict__ missing)
{
    __shared__ int64_t sk[PAL_MAX];
    __shared__ __align__(8) uint8_t st[PAL_MAX * PAL_ROW_MAX];
    for (int j = threadIdx.x; j < P; j += blockDim.x) sk[j] = keys ? keys[j] : j;
    for (int e = threadIdx.x; e < P * row_bytes; e += blockDim.x) st[e] = table[e];
    __syncthreads();
    unsigned long long miss = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int64_t lb = labels[i];
        int row = -1;
        if (!keys) {
            if (lb >= 0 && lb < P) row = (int)lb;
        } else {
            int lo = 0, hi = P;                     // first key >= lb
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (sk[mid] < lb) lo = mid + 1; else hi = mid;
            }
            if (lo < P && sk[lo] == lb) row = lo;
        }
        miss += row < 0;
        uint8_t* dst = out + i * row_bytes;
        if (row_bytes % 8 == 0) {
            const uint64_t* s = reinterpret_cast<const uint64_t*>(st + (size_t)max(row, 0) * row_bytes);
            for (int w = 0; w < row_bytes / 8; ++w) reinterpret_cast<uint64_t*>(dst)[w] = row < 0 ? 0 : s[w];
        } else {
            for (int b = 0; b < row_bytes; ++b) dst[b] = row < 0 ? 0 : st[row * row_bytes + b];
        }
    }
    if (missing) block_add(miss, missing);
}

template <typename T>
__global__ void __launch_bounds__(256) k_gather_index(const T* __restrict__ src, const int32_t* __restrict__ index, long long n, T* __restrict__ out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = src[index[i]];
}

unsigned grid_for(long long n)
{
    // grid-stride kernels that stage a table in shared memory: enough CTAs to fill the GPU several times, no more
    return (unsigned)std::min<long long>((n + 255) / 256, 132LL * 16);
}

} // namespace

extern "C" int isb_color_hist(const uint8_t* img, long long n_px, int channels, int accumulate, unsigned long long* hist, isb_stream_t stream)
{
    ISB_REQUIRE(img && hist, "null pointer");
    ISB_REQUIRE(n_px > 0, "bad sizes");
    ISB_REQUIRE(channels == 1 || channels == 3 || channels == 4, "channels must be 1 (grey), 3 (RGB) or 4 (RGBA)");
    cudaStream_t st = (cudaStream_t)stream;
    if (!accumulate) ISB_CUDA_CHECK(cudaMemsetAsync(hist, 0, sizeof(unsigned long long) << 24, st));
    const long long warps = (n_px + 32LL * HIST_PER - 1) / (32LL * HIST_PER);
    k_color_hist<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(img, n_px, channels, hist);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" size_t isb_color_hist_workspace_bytes(void) { return compact_workspace_bytes(1LL << 24); }

extern "C" int isb_color_hist_compact_count(const unsigned long long* hist, void* ws, size_t ws_bytes, long long* total, isb_stream_t stream)
{
    ISB_REQUIRE(hist && ws && total, "null pointer");
    ISB_REQUIRE(ws_bytes >= isb_color_hist_workspace_bytes(), "workspace too small");
    return compact_count(hist, 1LL << 24, ws, (cudaStream_t)stream, total);
}

extern "C" int isb_color_hist_compact_write(const unsigned long long* hist, const void* ws, size_t ws_bytes, int32_t* colors, int64_t* counts,
                                            isb_stream_t stream)
{
    ISB_REQUIRE(hist && ws && colors && counts, "null pointer");
    ISB_REQUIRE(ws_bytes >= isb_color_hist_workspace_bytes(), "workspace too small");
    const long long n = 1LL << 24;
    k_hist_write<<<compact_tiles(n), CPT_THREADS, 0, (cudaStream_t)stream>>>(hist, n, compact_tile_offsets(ws, n), colors, counts);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_palette_map(const void* img, int dtype, long long n_px, int channels, const void* palette, int n_colors, int mode,
                               const int64_t* values, int64_t* labels, uint8_t* matched, unsigned long long* unmatched, isb_stream_t stream)
{
    ISB_REQUIRE(img && palette && labels, "null pointer");
    ISB_REQUIRE(n_px > 0 && n_colors > 0, "bad sizes");
    ISB_REQUIRE(channels >= 1 && channels <= 4, "channels must be 1 .. 4");
    ISB_REQUIRE(dtype == ISB_U8 || dtype == ISB_F64, "the palette kernels take uint8 or float64 pixels");
    ISB_REQUIRE(mode == 0 || mode == 1, "mode must be 0 (exact) or 1 (L1-nearest)");
    if (n_colors > PAL_MAX) {
        isb_set_error("a palette of %d colours is above the limit of %d", n_colors, PAL_MAX);
        return ISB_ERR_UNSUPPORTED;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (unmatched) ISB_CUDA_CHECK(cudaMemsetAsync(unmatched, 0, sizeof(unsigned long long), st));
    if (dtype == ISB_U8)
        k_palette<uint8_t><<<grid_for(n_px), 256, 0, st>>>((const uint8_t*)img, n_px, channels, (const uint8_t*)palette, n_colors, mode, values,
                                                           labels, matched, unmatched);
    else
        k_palette<double><<<grid_for(n_px), 256, 0, st>>>((const double*)img, n_px, channels, (const double*)palette, n_colors, mode, values,
                                                          labels, matched, unmatched);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_palette_gather(const int64_t* labels, long long n_px, const int64_t* keys, int n_colors, const void* table, int row_bytes,
                                  void* out, unsigned long long* missing, isb_stream_t stream)
{
    ISB_REQUIRE(labels && table && out, "null pointer");
    ISB_REQUIRE(n_px > 0 && n_colors > 0, "bad sizes");
    ISB_REQUIRE(row_bytes >= 1 && row_bytes <= PAL_ROW_MAX, "a colour is 1 .. 32 bytes");
    if (n_colors > PAL_MAX) {
        isb_set_error("a palette of %d colours is above the limit of %d", n_colors, PAL_MAX);
        return ISB_ERR_UNSUPPORTED;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (missing) ISB_CUDA_CHECK(cudaMemsetAsync(missing, 0, sizeof(unsigned long long), st));
    k_palette_gather<<<grid_for(n_px), 256, 0, st>>>(labels, n_px, keys, n_colors, (const uint8_t*)table, row_bytes, (uint8_t*)out, missing);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_gather_at_index(const void* src, int elem_bytes, const int32_t* index, long long n, void* out, isb_stream_t stream)
{
    ISB_REQUIRE(src && index && out, "null pointer");
    ISB_REQUIRE(n > 0, "bad sizes");
    const unsigned grid = (unsigned)((n + 255) / 256);
    cudaStream_t st = (cudaStream_t)stream;
    switch (elem_bytes) {
        case 1: k_gather_index<uint8_t><<<grid, 256, 0, st>>>((const uint8_t*)src, index, n, (uint8_t*)out); break;
        case 2: k_gather_index<uint16_t><<<grid, 256, 0, st>>>((const uint16_t*)src, index, n, (uint16_t*)out); break;
        case 4: k_gather_index<uint32_t><<<grid, 256, 0, st>>>((const uint32_t*)src, index, n, (uint32_t*)out); break;
        case 8: k_gather_index<uint64_t><<<grid, 256, 0, st>>>((const uint64_t*)src, index, n, (uint64_t*)out); break;
        default: ISB_REQUIRE(false, "elements are 1, 2, 4 or 8 bytes");
    }
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
