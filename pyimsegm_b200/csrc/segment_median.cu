// segment_median.cu -- per-segment, per-channel MEDIAN of an image, and binary morphology with a disc.
//
// Median: replaces imsegm/descriptors.py:420-455 numpy_img2d_color_median and :651-676 numpy_img3d_gray_median -- pure-Python
// loops in the reference (a list append per pixel and channel, then np.median per label).  Here:
//   1. counting sort of the pixel indices by label (histogram, single-CTA scan, scatter; the order inside a label is irrelevant),
//   2. one CTA per label for all its channels: 8-bit MSB-first radix SELECT on the order-preserving 64-bit image of the doubles --
//      eight passes over the label's pixels find the lower middle value exactly, one more pass finds the upper middle one
//      (np.median averages the two for an even count).  The passes read the label's keys from shared memory, staged once, unless
//      the label is larger than the shared-memory budget; then they read the image.
// Morphology: skimage.morphology.opening(mask, disk(r)) as imsegm/descriptors.py:1873-1876 applies it to the boundary mask of the
// Ray features = grey erosion then grey dilation with a disc footprint, borders reflected (scipy.ndimage default mode).
#include <float.h>
#include "common.cuh"
#include "block_scan.cuh"

namespace {

constexpr int MT = 128;   // threads of a select CTA

__global__ void __launch_bounds__(256) k_med_count(const int* __restrict__ seg, size_t n, int nb, int* __restrict__ counts)
{
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int lb = seg[p];
    if (lb >= 0 && lb < nb) atomicAdd(&counts[lb], 1);
}

// exclusive scan counts[0..nb) -> start[0..nb], cursor = start (single CTA; nb is a superpixel count)
__global__ void __launch_bounds__(1024) k_med_scan(const int* __restrict__ counts, int nb, int* __restrict__ start, int* __restrict__ cursor)
{
    const int total = cta_scan_chunks<1024, int>(nb, [&](int i) { return counts[i]; },
                                                 [&](int i, int s) { start[i] = s; cursor[i] = s; });
    if (threadIdx.x == 0) start[nb] = total;
}

__global__ void __launch_bounds__(256) k_med_scatter(const int* __restrict__ seg, size_t n, int nb, int* __restrict__ cursor, unsigned* __restrict__ order)
{
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int lb = seg[p];
    if (lb >= 0 && lb < nb) order[atomicAdd(&cursor[lb], 1)] = (unsigned)p;
}

// the pixel value as a double, with np.nan_to_num applied in the pixel's own type first when ``clean`` is set
__device__ __forceinline__ double med_load(const void* img, int dtype, size_t i, bool clean)
{
    if (clean && dtype == ISB_F32) {
        const float v = ((const float*)img)[i];
        return isnan(v) ? 0. : (isinf(v) ? (v > 0.f ? (double)FLT_MAX : -(double)FLT_MAX) : (double)v);
    }
    const double v = load_as_f64(img, dtype, i);
    if (clean && dtype == ISB_F64) return isnan(v) ? 0. : (isinf(v) ? (v > 0. ? DBL_MAX : -DBL_MAX) : v);
    return v;
}

struct SelShared {
    int hist[256];
    unsigned long long prefix;
    unsigned long long next;   // smallest key above the selected one
    int k;
    int le;                    // how many keys are <= the selected one
    int nan;                   // how many keys are NaN
};

// the keys of +inf and -inf: a NaN key lies above the first (sign bit clear) or below the second (sign bit set)
constexpr unsigned long long KEY_PINF = 0xFFF0000000000000ull, KEY_NINF = 0x000FFFFFFFFFFFFFull;

// np.median of the n keys key_at(0..n) in the float type of the image (float32 when ``f32``): 8-bit MSB-first radix select of the
// lower middle rank, one more pass for the upper middle one; NaN when any key is NaN.  Every thread of the CTA calls it and gets
// the result.
template <class KeyAt>
__device__ double med_select(const KeyAt& key_at, int n, bool f32, SelShared& s)
{
    const int k_lo = (n - 1) / 2, k_hi = n / 2;
    __syncthreads();                       // the previous call's readers are done with s
    if (threadIdx.x == 0) { s.prefix = 0ull; s.k = k_lo; s.nan = 0; }
    for (int pass = 0; pass < 8; ++pass) {
        const int shift = 56 - 8 * pass;
        for (int i = threadIdx.x; i < 256; i += MT) s.hist[i] = 0;
        __syncthreads();
        const unsigned long long prefix = s.prefix;
        int n_nan = 0;
        for (int i = threadIdx.x; i < n; i += MT) {
            const unsigned long long key = key_at(i);
            if (pass == 0) n_nan += key > KEY_PINF || key < KEY_NINF;
            if (pass == 0 || (key >> (shift + 8)) == (prefix >> (shift + 8))) atomicAdd(&s.hist[(int)((key >> shift) & 255ull)], 1);
        }
        if (pass == 0 && n_nan) atomicAdd(&s.nan, n_nan);
        __syncthreads();
        if (s.nan) return nan("");         // np.median propagates NaN; s.nan is final after the barrier, so every thread returns here
        if (threadIdx.x == 0) {
            int k = s.k, d = 0;
            for (; d < 255; ++d) { if (k < s.hist[d]) break; k -= s.hist[d]; }
            s.k = k;
            s.prefix = prefix | ((unsigned long long)d << shift);
        }
        __syncthreads();
    }
    const unsigned long long sel = s.prefix;    // key of the element of rank k_lo
    const double lo = f64_unordered(sel);
    double hi = lo;
    if (k_hi != k_lo) {
        if (threadIdx.x == 0) { s.next = ~0ull; s.le = 0; }
        __syncthreads();
        int le = 0;
        unsigned long long nx = ~0ull;
        for (int i = threadIdx.x; i < n; i += MT) {
            const unsigned long long key = key_at(i);
            if (key <= sel) ++le; else if (key < nx) nx = key;
        }
        atomicAdd(&s.le, le);
        atomicMin(&s.next, nx);
        __syncthreads();
        if (s.le < k_hi + 1) hi = f64_unordered(s.next);   // the upper middle element is the next larger value
    }
    if (k_hi == k_lo) return lo;           // odd count: the middle value itself (no 0.5 * (v + v), which overflows near DBL_MAX)
    // np.mean of the two middles: summed and halved in the image's float type (u8 / u16 middles add exactly in float64)
    if (f32) return (double)__fmul_rn(__fadd_rn((float)lo, (float)hi), 0.5f);
    return 0.5 * (lo + hi);
}

// one CTA per label serves every channel.  A label of at most ``cap`` pixels stages its C keys per pixel in shared memory once
// and selects there; a larger one (a caller may pass any label map) selects straight from the image, channel after channel.
__global__ void __launch_bounds__(MT) k_med_select(const void* __restrict__ img, int dtype, int C, const int* __restrict__ start,
                                                   const unsigned* __restrict__ order, int cap, int clean, double* __restrict__ out,
                                                   int ld, int col0)
{
    extern __shared__ unsigned long long s_keys[];   // [C][cap]
    __shared__ SelShared s;
    const int lb = blockIdx.x;
    const int beg = start[lb], n = start[lb + 1] - beg;
    double* row = out + (size_t)lb * ld + col0;
    if (n <= 0) { for (int c = threadIdx.x; c < C; c += MT) row[c] = nan(""); return; }
    const unsigned* ord = order + beg;
    const bool f32 = dtype == ISB_F32;
    if (n <= cap) {
        for (int i = threadIdx.x; i < n; i += MT) {
            const size_t p = (size_t)ord[i] * C;
            for (int c = 0; c < C; ++c) s_keys[(size_t)c * cap + i] = f64_ordered(med_load(img, dtype, p + c, clean));
        }
    }
    for (int c = 0; c < C; ++c) {
        double m;
        if (n <= cap) {
            const unsigned long long* keys = s_keys + (size_t)c * cap;
            m = med_select([&](int i) { return keys[i]; }, n, f32, s);      // the first barrier inside also publishes the staged keys
        } else {
            m = med_select([&](int i) { return f64_ordered(med_load(img, dtype, (size_t)ord[i] * C + c, clean)); }, n, f32, s);
        }
        if (clean) {   // the feature table's rules: an infinite median (FLT_MAX + FLT_MAX in float32) -> the largest finite value, -0 -> +0
            if (isinf(m)) m = m > 0 ? DBL_MAX : -DBL_MAX;
            if (m == 0.) m = 0.;
        }
        if (threadIdx.x == 0) row[c] = m;
    }
}

// shared memory of the staged keys (two CTAs of 96 KB per SM)
constexpr int MED_SMEM_BYTES = 96 * 1024;

struct MedWs { int* counts; int* start; int* cursor; unsigned* order; };
static size_t carve_med(MedWs& w, void* ws, size_t bytes, size_t n, int nb)
{
    WsCarver c(ws, bytes);
    w.counts = c.take<int>(nb); w.start = c.take<int>((size_t)nb + 1); w.cursor = c.take<int>(nb); w.order = c.take<unsigned>(n);
    return isb_align(c.off);
}

} // namespace

extern "C" size_t isb_segment_median_workspace_bytes(long long n_px, int nb)
{
    MedWs w;
    return carve_med(w, nullptr, 0, (size_t)n_px, nb);
}

static int segment_median(const void* img, int dtype, const int32_t* seg, long long n_px, int channels, int nb, double* out, int ld,
                          int col0, bool clean, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(img && seg && out && ws, "null pointer");
    ISB_REQUIRE(n_px > 0 && n_px < (1LL << 32) && channels > 0 && channels <= 65535 && nb > 0, "bad sizes");
    ISB_REQUIRE(col0 >= 0 && ld >= col0 + channels, "bad feature table layout");
    ISB_REQUIRE(dtype >= ISB_U8 && dtype <= ISB_F64, "bad dtype");
    static bool smem_set[64] = {};   // per device; set outside any capture: the first call of a configuration always runs eagerly
    int dev = 0;
    ISB_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev >= 64 || !smem_set[dev]) {
        ISB_CUDA_CHECK(cudaFuncSetAttribute(k_med_select, cudaFuncAttributeMaxDynamicSharedMemorySize, MED_SMEM_BYTES));
        if (dev < 64) smem_set[dev] = true;
    }
    const int cap = MED_SMEM_BYTES / (int)(sizeof(unsigned long long) * channels);
    const size_t smem = cap > 0 ? (size_t)MED_SMEM_BYTES : 0;
    MedWs w;
    const size_t need = carve_med(w, ws, ws_bytes, (size_t)n_px, nb);
    ISB_REQUIRE(need <= ws_bytes, "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_STATS, st);
    const size_t n = (size_t)n_px;
    ISB_CUDA_CHECK(cudaMemsetAsync(w.counts, 0, sizeof(int) * (size_t)nb, st));
    k_med_count<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(seg, n, nb, w.counts);
    ISB_LAUNCH_CHECK();
    k_med_scan<<<1, 1024, 0, st>>>(w.counts, nb, w.start, w.cursor);
    ISB_LAUNCH_CHECK();
    k_med_scatter<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(seg, n, nb, w.cursor, w.order);
    ISB_LAUNCH_CHECK();
    k_med_select<<<nb, MT, smem, st>>>(img, dtype, channels, w.start, w.order, cap, int(clean), out, ld, col0);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_segment_median(const void* img, int dtype, const int32_t* seg, long long n_px, int channels, int nb, double* out, void* ws,
                                  size_t ws_bytes, isb_stream_t stream)
{
    return segment_median(img, dtype, seg, n_px, channels, nb, out, channels, 0, false, ws, ws_bytes, stream);
}

extern "C" int isb_segment_median_2d(const void* img, int dtype, const int32_t* seg, int H, int W, int channels, int nb, double* feat, int ld,
                                     int col0, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(H > 0 && W > 0, "bad sizes");
    return segment_median(img, dtype, seg, (long long)H * W, channels, nb, feat, ld, col0, true, ws, ws_bytes, stream);
}
