// slic_prepare.cu -- SLIC pre-pass: min/max -> rescale -> gaussian blur -> rgb2lab -> * 1/compactness -> planar f64.
// The rescale runs in the image's own precision as numpy does it (float32 for a float32 image, float64 otherwise); the
// blur and everything after it run in f64 for every input type.
//
// Replaces (reference call stack, SURVEY.md section 3.1):
//   imsegm/superpixels.py:53-54   img = (img - img.min()) / float(img.max() - img.min())
//   skimage.segmentation.slic:    ndi.gaussian_filter(image[1,H,W,3], [s,s,s,0]);  rgb2lab;  image * (1/compactness)
//
// Every value must be bit-identical to oracle/slic_oracle.c, so all arithmetic below is explicit IEEE
// round-to-nearest double (__dadd_rn/__dmul_rn/__ddiv_rn are never contracted into FMA) in the oracle's order.
// HBM traffic: reads the raw image once (+ halo re-reads served by L2), writes 24 B/px.
#include "common.cuh"

namespace {

struct GaussW { double w[9]; };

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

// cube root, division-free: Newton on y = x^(-1/3) from an exponent-bit seed, then x y^2 and one correction step.
// A fixed sequence of IEEE mul / sub -- the same sequence as oracle/slic_oracle.c (DESIGN.md "deliberate definitions").
__device__ __forceinline__ double det_cbrt(double x)
{
    unsigned long long u = 0x553EF00000000000ull - (unsigned long long)__double_as_longlong(x) / 3ull;
    double y = __longlong_as_double((long long)u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const double y2 = dmul(y, y);
        const double y3 = dmul(y2, y);
        const double t = dmul(x, y3);
        const double w = dsub(4.0, t);
        y = dmul(dmul(y, w), 1.0 / 3.0);
    }
    const double y2 = dmul(y, y);
    double c = dmul(x, y2);
    const double c3 = dmul(dmul(c, c), c);
    c = dsub(c, dmul(dmul(dsub(c3, x), y2), 1.0 / 3.0));
    return c;
}

__device__ __forceinline__ double det_root5(double x)
{
    unsigned long long u = 0x4CB8A99999999800ull - (unsigned long long)__double_as_longlong(x) / 5ull;
    double y = __longlong_as_double((long long)u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const double y2 = dmul(y, y);
        const double y4 = dmul(y2, y2);
        const double y5 = dmul(y4, y);
        const double t = dmul(x, y5);
        const double w = dsub(6.0, t);
        y = dmul(dmul(y, w), 0.2);
    }
    const double y2 = dmul(y, y);
    const double y4 = dmul(y2, y2);
    double r = dmul(x, y4);
    const double r2 = dmul(r, r);
    const double r5 = dmul(dmul(r2, r2), r);
    r = dsub(r, dmul(dmul(dsub(r5, x), y4), 0.2));
    return r;
}

__device__ __forceinline__ double det_pow24(double t)
{
    double r = det_root5(t);
    return dmul(dmul(t, t), dmul(r, r));
}

__device__ __forceinline__ void rgb2lab_px(double r, double g, double b, double& L, double& A, double& B)
{
    double c[3] = { r, g, b };
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        if (c[i] > 0.04045) c[i] = det_pow24(ddiv(dadd(c[i], 0.055), 1.055));
        else c[i] = ddiv(c[i], 12.92);
    }
    double X = dadd(dadd(dmul(c[0], 0.412453), dmul(c[1], 0.357580)), dmul(c[2], 0.180423));
    double Y = dadd(dadd(dmul(c[0], 0.212671), dmul(c[1], 0.715160)), dmul(c[2], 0.072169));
    double Z = dadd(dadd(dmul(c[0], 0.019334), dmul(c[1], 0.119193)), dmul(c[2], 0.950227));
    double f[3] = { ddiv(X, 0.95047), ddiv(Y, 1.0), ddiv(Z, 1.08883) };
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        if (f[i] > 0.008856) f[i] = det_cbrt(f[i]);
        else f[i] = dadd(dmul(7.787, f[i]), ddiv(16.0, 116.0));
    }
    L = dsub(dmul(116.0, f[1]), 16.0);
    A = dmul(500.0, dsub(f[0], f[1]));
    B = dmul(200.0, dsub(f[1], f[2]));
}

// numpy's min / max: a NaN sample makes the result NaN (fmin / fmax would skip it).  A NaN is sticky in both reductions: it wins
// every comparison it takes part in.
__device__ __forceinline__ double nan_min(double a, double b) { return (a < b || a != a) ? a : b; }
__device__ __forceinline__ double nan_max(double a, double b) { return (a > b || a != a) ? a : b; }

__global__ void k_minmax(const void* img, int dtype, size_t n, unsigned long long* mm)
{
    double lo = 1.0 / 0.0, hi = -1.0 / 0.0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        double v = load_as_f64(img, dtype, i);
        lo = nan_min(lo, v);
        hi = nan_max(hi, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo = nan_min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = nan_max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    __shared__ double slo[32], shi[32];
    int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { slo[w] = lo; shi[w] = hi; }
    __syncthreads();
    if (w == 0) {
        int nw = blockDim.x >> 5;
        lo = l < nw ? slo[l] : 1.0 / 0.0;
        hi = l < nw ? shi[l] : -1.0 / 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo = nan_min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
            hi = nan_max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        }
        if (l == 0) {
            // in the ordered map a NaN with the sign bit set is below -inf and one without it above +inf, so the atomics keep it
            if (lo != lo) lo = __longlong_as_double((long long)0xFFF8000000000000ull);
            if (hi != hi) hi = __longlong_as_double(0x7FF8000000000000ll);
            atomicMin(&mm[0], f64_ordered(lo));
            atomicMax(&mm[1], f64_ordered(hi));
        }
    }
}

__global__ void k_minmax_decode(const unsigned long long* mm, double* out)
{
    const double lo = f64_unordered(mm[0]), hi = f64_unordered(mm[1]);
    const double nan = __longlong_as_double(0x7FF8000000000000ll);
    out[0] = lo != lo ? nan : lo;
    out[1] = hi != hi ? nan : hi;
}

// k_blur_lab: one CTA = TX output columns x SH output rows, walked down in chunks of K rows.
//   stage 1  load + rescale + depth axis of the K new input rows into a ring of 2R+K haloed rows (the first chunk fills all 2R+K)
//   stage 2  rows axis: one thread per (channel, haloed column) reads its 2R+K ring samples once into registers, writes K outputs
//   stage 3  cols axis + rgb2lab + ratio for the K x TX output pixels
// Rescale and depth work per output pixel is (SH+2R)(TX+2R)/(SH TX) (1.19x at R=4), the rows axis (TX+2R)/TX (1.06x at R=4).
// The radius is a template parameter so every tap loop unrolls and the weights are read from parameter space.
constexpr int TX = 128, SH = 64, KR = 8, NT = 256;

template <int R>
struct BlurShape {
    static constexpr int IW = TX + 2 * R;   // haloed tile width
    static constexpr int RING = 2 * R + KR; // input rows held at once
    static constexpr size_t smem = sizeof(double) * 3 * ((size_t)RING * IW + (size_t)KR * IW) + sizeof(int) * IW;
};

template <int R>
__global__ void __launch_bounds__(NT, 2) k_blur_lab(const void* __restrict__ img, int dtype, int H, int W, int C,
                                                    const double* __restrict__ minmax, int rescale, GaussW gw, double ratio,
                                                    double* __restrict__ out)
{
    using S = BlurShape<R>;
    constexpr int IW = S::IW, RING = S::RING;
    extern __shared__ double smem[];
    double* s_in = smem;                     // [3][RING][IW]
    double* s_v = smem + 3 * RING * IW;      // [3][KR][IW]
    int* s_gx = (int*)(s_v + 3 * KR * IW);   // [IW] reflected source column of each haloed column
    const int x0 = blockIdx.x * TX, y0 = blockIdx.y * SH;
    const int y_end = min(y0 + SH, H);
    const double mn = minmax[0], mx = minmax[1];
    const bool do_rescale = rescale && (mn != 0.0 || mx != 1.0);
    const double span = dsub(mx, mn);
    // a float32 image is rescaled in float32, as numpy does (img - img.min()) / float(img.max() - img.min()) for it; the
    // extrema are float32 values, so they convert back exactly
    const bool rescale_f32 = dtype == ISB_F32;
    const float mnf = (float)mn, spanf = __fsub_rn((float)mx, mnf);
    const size_t HW = (size_t)H * W;

    for (int ix = threadIdx.x; ix < IW; ix += NT) s_gx[ix] = reflect_index(x0 + ix - R, W);
    __syncthreads();

    // rescale, then the depth axis of skimage's [1,H,W,3] array: all its taps reflect onto the same sample
    auto prep = [&](double v) {
        if (do_rescale) v = rescale_f32 ? (double)__fdiv_rn(__fsub_rn((float)v, mnf), spanf) : ddiv(dsub(v, mn), span);
        if (R > 0) {
            double t = dmul(v, gw.w[0]);
#pragma unroll
            for (int j = R; j >= 1; --j) t = dadd(t, dmul(dadd(v, v), gw.w[j]));
            v = t;
        }
        return v;
    };

    int slot0 = 0; // ring slot of the chunk's first input row
    for (int cy = y0; cy < y_end; cy += KR) {
        // stage 1: input rows [lo, lo + nrow) relative to y0 - R
        const int first = cy == y0;
        const int lo = first ? 0 : cy - y0 + 2 * R, nrow = first ? RING : KR;
        for (int i = threadIdx.x; i < nrow * IW; i += NT) {
            const int row = i / IW, ix = i - row * IW;
            const int ir = lo + row;
            const int gy = reflect_index(y0 - R + ir, H);
            const size_t base = ((size_t)gy * W + s_gx[ix]) * C;
            double* dst = s_in + (ir % RING) * IW + ix;
            if (C == 3) {
#pragma unroll
                for (int c = 0; c < 3; ++c) dst[c * RING * IW] = prep(load_as_f64(img, dtype, base + c));
            } else {
                const double v = prep(load_as_f64(img, dtype, base));
#pragma unroll
                for (int c = 0; c < 3; ++c) dst[c * RING * IW] = v;
            }
        }
        __syncthreads();
        // stage 2: rows axis
        for (int i = threadIdx.x; i < 3 * IW; i += NT) {
            const int c = i / IW, ix = i - c * IW;
            const double* col = s_in + c * RING * IW + ix;
            double w[RING];
#pragma unroll
            for (int k = 0; k < RING; ++k) {
                int s = slot0 + k;
                if (s >= RING) s -= RING;
                w[k] = col[s * IW];
            }
            double* dst = s_v + c * KR * IW + ix;
#pragma unroll
            for (int k = 0; k < KR; ++k) {
                double t = w[k + R];
                if (R > 0) {
                    t = dmul(w[k + R], gw.w[0]);
#pragma unroll
                    for (int j = R; j >= 1; --j) t = dadd(t, dmul(dadd(w[k + R - j], w[k + R + j]), gw.w[j]));
                }
                dst[k * IW] = t;
            }
        }
        __syncthreads();
        // stage 3: cols axis + rgb2lab + scale
        for (int i = threadIdx.x; i < KR * TX; i += NT) {
            const int ty = i / TX, tx = i - ty * TX;
            const int gy = cy + ty, gx = x0 + tx;
            if (gy >= y_end || gx >= W) continue;
            double v[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const double* row = s_v + (c * KR + ty) * IW + tx + R;
                double t = row[0];
                if (R > 0) {
                    t = dmul(row[0], gw.w[0]);
#pragma unroll
                    for (int j = R; j >= 1; --j) t = dadd(t, dmul(dadd(row[-j], row[j]), gw.w[j]));
                }
                v[c] = t;
            }
            double L, A, B;
            rgb2lab_px(v[0], v[1], v[2], L, A, B);
            const size_t p = (size_t)gy * W + gx;
            out[p] = dmul(L, ratio);
            out[HW + p] = dmul(A, ratio);
            out[2 * HW + p] = dmul(B, ratio);
        }
        // the next stage 1 overwrites only ring rows this chunk's stage 2 has finished with (a barrier ago), and the next
        // stage 2 writes s_v only after the barrier that follows the next stage 1
        slot0 += KR;
        if (slot0 >= RING) slot0 -= RING;
    }
}

template <int R>
static int blur_lab_launch(const void* img, int dtype, int H, int W, int C, const double* minmax, int rescale, const GaussW& gw,
                           double ratio, double* out, cudaStream_t st)
{
    const size_t smem = BlurShape<R>::smem;
    if (smem > 48 * 1024) ISB_CUDA_CHECK(cudaFuncSetAttribute(k_blur_lab<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((W + TX - 1) / TX, (H + SH - 1) / SH);
    k_blur_lab<R><<<grid, NT, smem, st>>>(img, dtype, H, W, C, minmax, rescale, gw, ratio, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

static int minmax_launch(const void* img, int dtype, size_t n, double* minmax_out, cudaStream_t st)
{
    // the two ordered-uint64 accumulators live in minmax_out[2..3]
    unsigned long long* mm = (unsigned long long*)(minmax_out + 2);
    ISB_CUDA_CHECK(cudaMemsetAsync(mm, 0xFF, sizeof(unsigned long long), st));
    ISB_CUDA_CHECK(cudaMemsetAsync(mm + 1, 0x00, sizeof(unsigned long long), st));
    int blocks = (int)((n + 256 * 8 - 1) / (256 * 8));
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    k_minmax<<<blocks, 256, 0, st>>>(img, dtype, n, mm);
    ISB_LAUNCH_CHECK();
    k_minmax_decode<<<1, 1, 0, st>>>(mm, minmax_out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

} // namespace

extern "C" int isb_image_minmax(const void* img, int dtype, long long n, double* minmax_out, isb_stream_t stream)
{
    ISB_REQUIRE(img && minmax_out && n > 0, "null pointer or empty image");
    ISB_REQUIRE(dtype >= ISB_U8 && dtype <= ISB_F64, "bad dtype");
    return minmax_launch(img, dtype, (size_t)n, minmax_out, (cudaStream_t)stream);
}

extern "C" int isb_slic_prepare(const void* img, int dtype, int H, int W, int C, const double* w_half, int radius, double ratio,
                                int rescale, double* lab_planar, double* minmax_out, isb_stream_t stream)
{
    ISB_REQUIRE(img && lab_planar && minmax_out, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && (C == 1 || C == 3), "bad image shape (C must be 1 or 3)");
    ISB_REQUIRE(dtype >= ISB_U8 && dtype <= ISB_F64, "bad dtype");
    ISB_REQUIRE(radius >= 0 && radius <= 8 && (radius == 0 || w_half), "gaussian radius must be in [0,8]");
    cudaStream_t st = (cudaStream_t)stream;
    // minmax_out must have room for 4 doubles: [min, max, scratch, scratch]
    ProfScope prof(ISB_PROF_PREPARE, st);
    if (rescale != 2)
        if (int rc = minmax_launch(img, dtype, (size_t)H * W * C, minmax_out, st)) return rc;
    GaussW gw;
    for (int i = 0; i < 9; ++i) gw.w[i] = (i <= radius && w_half) ? w_half[i] : 0.0;
    switch (radius) {
        case 0: return blur_lab_launch<0>(img, dtype, H, W, C, minmax_out, rescale, gw, ratio, lab_planar, st);
        case 1: return blur_lab_launch<1>(img, dtype, H, W, C, minmax_out, rescale, gw, ratio, lab_planar, st);
        case 2: return blur_lab_launch<2>(img, dtype, H, W, C, minmax_out, rescale, gw, ratio, lab_planar, st);
        case 3: return blur_lab_launch<3>(img, dtype, H, W, C, minmax_out, rescale, gw, ratio, lab_planar, st);
        case 4: return blur_lab_launch<4>(img, dtype, H, W, C, minmax_out, rescale, gw, ratio, lab_planar, st);
        case 5: return blur_lab_launch<5>(img, dtype, H, W, C, minmax_out, rescale, gw, ratio, lab_planar, st);
        case 6: return blur_lab_launch<6>(img, dtype, H, W, C, minmax_out, rescale, gw, ratio, lab_planar, st);
        case 7: return blur_lab_launch<7>(img, dtype, H, W, C, minmax_out, rescale, gw, ratio, lab_planar, st);
        default: return blur_lab_launch<8>(img, dtype, H, W, C, minmax_out, rescale, gw, ratio, lab_planar, st);
    }
}
