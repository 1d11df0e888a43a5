// slic_prepare.cu -- SLIC pre-pass: min/max -> rescale -> gaussian blur -> rgb2lab -> * 1/compactness -> planar f64.
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

struct GaussW { double w[9]; int r; };

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

__device__ __forceinline__ int reflect_idx(int i, int n)
{
    if (n == 1) return 0;
    int p = 2 * n;
    i %= p;
    if (i < 0) i += p;
    return (i < n) ? i : (p - 1 - i);
}

__global__ void k_minmax(const void* img, int dtype, size_t n, unsigned long long* mm)
{
    double lo = 1.0 / 0.0, hi = -1.0 / 0.0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        double v = load_as_f64(img, dtype, i);
        lo = fmin(lo, v);
        hi = fmax(hi, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
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
            lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
            hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        }
        if (l == 0) {
            atomicMin(&mm[0], f64_ordered(lo));
            atomicMax(&mm[1], f64_ordered(hi));
        }
    }
}

__global__ void k_minmax_decode(const unsigned long long* mm, double* out)
{
    out[0] = f64_unordered(mm[0]);
    out[1] = f64_unordered(mm[1]);
}

constexpr int TY = 16, TX = 32;

// one CTA = TY x TX output pixels; smem: input tile with halo r (after rescale + depth pass), then row-blurred strip
__global__ void __launch_bounds__(256) k_blur_lab(const void* img, int dtype, int H, int W, int C, const double* minmax,
                                                  int rescale, GaussW gw, double ratio, double* out)
{
    extern __shared__ double smem[];
    const int r = gw.r;
    const int IW = TX + 2 * r, IH = TY + 2 * r;
    double* s_in = smem;               // [3][IH][IW]
    double* s_v = smem + 3 * IH * IW;  // [3][TY][IW]
    const int x0 = blockIdx.x * TX, y0 = blockIdx.y * TY;
    const double mn = minmax[0], mx = minmax[1];
    const bool do_rescale = rescale && (mn != 0.0 || mx != 1.0);
    const double span = dsub(mx, mn);

    for (int i = threadIdx.x; i < IH * IW; i += blockDim.x) {
        int iy = i / IW, ix = i - iy * IW;
        int gy = reflect_idx(y0 + iy - r, H), gx = reflect_idx(x0 + ix - r, W);
        size_t base = ((size_t)gy * W + gx) * C;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            double v = load_as_f64(img, dtype, base + (C == 3 ? c : 0));
            if (do_rescale) v = ddiv(dsub(v, mn), span);
            if (r > 0) {
                // depth axis of skimage's [1,H,W,3] array: all taps reflect onto the same sample
                double t = dmul(v, gw.w[0]);
                for (int j = r; j >= 1; --j) t = dadd(t, dmul(dadd(v, v), gw.w[j]));
                v = t;
            }
            s_in[(c * IH + iy) * IW + ix] = v;
        }
    }
    __syncthreads();
    // rows axis (vertical), for every column of the haloed tile
    for (int i = threadIdx.x; i < 3 * TY * IW; i += blockDim.x) {
        int c = i / (TY * IW), rem = i - c * TY * IW;
        int ty = rem / IW, ix = rem - ty * IW;
        const double* col = s_in + (c * IH + ty + r) * IW + ix;
        double t;
        if (r > 0) {
            t = dmul(col[0], gw.w[0]);
            for (int j = r; j >= 1; --j) t = dadd(t, dmul(dadd(col[-j * IW], col[j * IW]), gw.w[j]));
        } else t = col[0];
        s_v[(c * TY + ty) * IW + ix] = t;
    }
    __syncthreads();
    // cols axis (horizontal) + rgb2lab + scale
    const size_t HW = (size_t)H * W;
    for (int i = threadIdx.x; i < TY * TX; i += blockDim.x) {
        int ty = i / TX, tx = i - ty * TX;
        int gy = y0 + ty, gx = x0 + tx;
        if (gy >= H || gx >= W) continue;
        double v[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double* row = s_v + (c * TY + ty) * IW + tx + r;
            double t;
            if (r > 0) {
                t = dmul(row[0], gw.w[0]);
                for (int j = r; j >= 1; --j) t = dadd(t, dmul(dadd(row[-j], row[j]), gw.w[j]));
            } else t = row[0];
            v[c] = t;
        }
        double L, A, B;
        rgb2lab_px(v[0], v[1], v[2], L, A, B);
        size_t p = (size_t)gy * W + gx;
        out[p] = dmul(L, ratio);
        out[HW + p] = dmul(A, ratio);
        out[2 * HW + p] = dmul(B, ratio);
    }
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
    gw.r = radius;
    for (int i = 0; i < 9; ++i) gw.w[i] = (i <= radius && w_half) ? w_half[i] : 0.0;
    dim3 grid((W + TX - 1) / TX, (H + TY - 1) / TY);
    size_t smem = sizeof(double) * 3 * ((size_t)(TY + 2 * radius) * (TX + 2 * radius) + (size_t)TY * (TX + 2 * radius));
    if (smem > 48 * 1024)
        ISB_CUDA_CHECK(cudaFuncSetAttribute(k_blur_lab, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_blur_lab<<<grid, 256, smem, st>>>(img, dtype, H, W, C, minmax_out, rescale, gw, ratio, lab_planar);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
