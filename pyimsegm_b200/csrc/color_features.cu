// color_features.cu -- the per-pixel inputs of the colour-space groups and of the median / meanGrad statistics, on the device.
//
//   isb_color_convert        pyimsegm_b200/color.py (skimage.color.rgb2hsv / luv / lab / hed / xyz) operation by operation, IEEE
//                            pow / cbrt / log (NOT the division-free forms of slic_prepare.cu, which define SLIC's own rgb2lab)
//   isb_gradient_sum_2d      np.sum(np.gradient(np.nan_to_num(ch)), axis=0) per channel, in the image's float type (descriptors.py
//                            compute_image2d_color_statistic, 'meanGrad')
//   isb_lm_background        the materialised Leung-Malik route (texture.py device_lm_materialised): planar copy of the image
//   isb_lm_battery_response  minus its sigma-150 background, then per battery the strongest response, clip, sum of squares in a fixed
//                            order (block partials, every CTA of the second kernel re-adds them in the same order: no floating atomics,
//                            a rerun gives the same bits) and the log-norm scaling, written interleaved [H, W, 3]
//   isb_lm_battery_partial   the same battery step split for row bands (tiled.py): the responses of a slab and the sum of squares of
//   isb_lm_battery_scale     its owned rows, then -- once the bands' sums are added -- the scaling of a row range with that norm
// Built with -fmad=false like every source here; the gradient spells its rounding out with the _rn intrinsics as well.
#include <float.h>
#include <algorithm>
#include "common.cuh"

namespace {

// hed_from_rgb = np.linalg.inv(rgb_from_hed) (color.py) and np.log(1e-6), to the last printed digit
__constant__ double c_hed_from_rgb[9] = {1.8779827368521353, -1.0076786862855645, -0.5561158181996246,
                                         -0.06590806222356332, 1.1347303724996625, -0.1355217986283712,
                                         -0.6019073634392891, -0.4804141884970579, 1.5735880719641926};
constexpr double kLogAdjust = -13.815510557964274;
__constant__ double c_xyz_from_rgb[9] = {0.412453, 0.357580, 0.180423, 0.212671, 0.715160, 0.072169, 0.019334, 0.119193, 0.950227};
constexpr double kD65x = 0.95047, kD65y = 1., kD65z = 1.08883;
// u0 = 4 * D65[0] / dot([1, 15, 3], D65), v0 = 9 * D65[1] / dot(...), np.finfo(float).eps
constexpr double kU0 = 0.19783982482140777, kV0 = 0.4683363029324097, kEps = 2.220446049250313e-16;

// color.py _as_float: u8 / 255., u16 / 65535., floats widened
__device__ __forceinline__ double as_float(const void* p, int dtype, size_t i)
{
    switch (dtype) {
        case ISB_U8: return __ddiv_rn((double)((const unsigned char*)p)[i], 255.);
        case ISB_U16: return __ddiv_rn((double)((const unsigned short*)p)[i], 65535.);
        case ISB_F32: return (double)((const float*)p)[i];
        default: return ((const double*)p)[i];
    }
}

__device__ __forceinline__ double np_mod1(double x)
{
    double m = fmod(x, 1.);        // numpy's divmod: the remainder takes the divisor's sign, an exact zero is +0
    if (m != 0.) { if (m < 0.) m = __dadd_rn(m, 1.); }
    else m = 0.;
    return m;
}

__device__ __forceinline__ double nan0(double v) { return isnan(v) ? 0. : v; }

__device__ __forceinline__ double srgb_linear(double a)
{
    return a > 0.04045 ? pow(__ddiv_rn(__dadd_rn(a, 0.055), 1.055), 2.4) : __ddiv_rn(a, 12.92);
}

__device__ __forceinline__ double lab_f(double a) { return a > 0.008856 ? cbrt(a) : __dadd_rn(__dmul_rn(7.787, a), 16. / 116.); }

__global__ void __launch_bounds__(256) k_color_convert(const void* __restrict__ img, int dtype, long long n, int space, double* __restrict__ out)
{
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const double r = as_float(img, dtype, 3 * (size_t)p), g = as_float(img, dtype, 3 * (size_t)p + 1), b = as_float(img, dtype, 3 * (size_t)p + 2);
    double o0, o1, o2;
    if (space == ISB_COLOR_HSV) {
        if (isnan(r) || isnan(g) || isnan(b)) {
            o0 = o1 = o2 = 0.;   // the host leaves the hue of such a pixel unset (np.empty_like); every channel is NaN -> 0 here
        } else {
            const double v = fmax(r, fmax(g, b)), delta = __dsub_rn(v, fmin(r, fmin(g, b)));
            double s = __ddiv_rn(delta, v);
            if (delta == 0.) s = 0.;
            double h = 0.;       // later channels override earlier ones when two of them equal the maximum (rgb2hsv)
            if (r == v) h = __ddiv_rn(__dsub_rn(g, b), delta);
            if (g == v) h = __dadd_rn(2., __ddiv_rn(__dsub_rn(b, r), delta));
            if (b == v) h = __dadd_rn(4., __ddiv_rn(__dsub_rn(r, g), delta));
            h = np_mod1(__ddiv_rn(h, 6.));
            if (delta == 0.) h = 0.;
            o0 = nan0(h); o1 = nan0(s); o2 = nan0(v);
        }
    } else if (space == ISB_COLOR_HED) {
        double l[3] = {r, g, b};
        for (int c = 0; c < 3; ++c) l[c] = __ddiv_rn(log(l[c] < 1e-6 ? 1e-6 : l[c]), kLogAdjust);   // np.maximum keeps a NaN
        double st[3];
        for (int j = 0; j < 3; ++j) {
            const double s = __dadd_rn(__dadd_rn(__dmul_rn(l[0], c_hed_from_rgb[j]), __dmul_rn(l[1], c_hed_from_rgb[3 + j])),
                                       __dmul_rn(l[2], c_hed_from_rgb[6 + j]));
            st[j] = s < 0. ? 0. : s;
        }
        o0 = st[0]; o1 = st[1]; o2 = st[2];
    } else {
        const double lin[3] = {srgb_linear(r), srgb_linear(g), srgb_linear(b)};
        double xyz[3];
        for (int i = 0; i < 3; ++i)
            xyz[i] = __dadd_rn(__dadd_rn(__dmul_rn(lin[0], c_xyz_from_rgb[3 * i]), __dmul_rn(lin[1], c_xyz_from_rgb[3 * i + 1])),
                               __dmul_rn(lin[2], c_xyz_from_rgb[3 * i + 2]));
        if (space == ISB_COLOR_XYZ) {
            o0 = xyz[0]; o1 = xyz[1]; o2 = xyz[2];
        } else if (space == ISB_COLOR_LAB) {
            const double fx = lab_f(__ddiv_rn(xyz[0], kD65x)), fy = lab_f(__ddiv_rn(xyz[1], kD65y)), fz = lab_f(__ddiv_rn(xyz[2], kD65z));
            o0 = __dsub_rn(__dmul_rn(116., fy), 16.);
            o1 = __dmul_rn(500., __dsub_rn(fx, fy));
            o2 = __dmul_rn(200., __dsub_rn(fy, fz));
        } else {   // luv
            const double x = xyz[0], y = xyz[1], z = xyz[2];
            double L = __ddiv_rn(y, kD65y);
            L = L > 0.008856 ? __dsub_rn(__dmul_rn(116., cbrt(L)), 16.) : __dmul_rn(903.3, L);
            const double d = __dadd_rn(__dadd_rn(__dadd_rn(x, __dmul_rn(15., y)), __dmul_rn(3., z)), kEps);
            const double l13 = __dmul_rn(13., L);
            o0 = L;
            o1 = __dmul_rn(l13, __dsub_rn(__ddiv_rn(__dmul_rn(4., x), d), kU0));
            o2 = __dmul_rn(l13, __dsub_rn(__ddiv_rn(__dmul_rn(9., y), d), kV0));
        }
    }
    out[3 * (size_t)p] = o0; out[3 * (size_t)p + 1] = o1; out[3 * (size_t)p + 2] = o2;
}

// ---- summed gradient -------------------------------------------------------------------------------------------------------

__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double fsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double fadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float fhalf(float a) { return __fdiv_rn(a, 2.f); }
__device__ __forceinline__ double fhalf(double a) { return __ddiv_rn(a, 2.); }

// np.nan_to_num in the pixel's own type (integers pass unchanged), then the type np.gradient computes in
template <typename T> __device__ __forceinline__ T load_clean(const void* p, int dtype, size_t i);
template <> __device__ __forceinline__ float load_clean<float>(const void* p, int, size_t i)
{
    const float v = ((const float*)p)[i];
    return isnan(v) ? 0.f : (isinf(v) ? (v > 0.f ? FLT_MAX : -FLT_MAX) : v);
}
template <> __device__ __forceinline__ double load_clean<double>(const void* p, int dtype, size_t i)
{
    const double v = load_as_f64(p, dtype, i);
    if (dtype != ISB_F64) return v;
    return isnan(v) ? 0. : (isinf(v) ? (v > 0. ? DBL_MAX : -DBL_MAX) : v);
}

// np.gradient along one axis, spacing 1, edge_order 1: one-sided at the borders, central halves inside
template <typename T> __device__ __forceinline__ T grad1(const void* img, int dtype, size_t base, int i, int n, size_t stride)
{
    if (i == 0) return fsub(load_clean<T>(img, dtype, base + stride), load_clean<T>(img, dtype, base));
    if (i == n - 1) return fsub(load_clean<T>(img, dtype, base), load_clean<T>(img, dtype, base - stride));
    return fhalf(fsub(load_clean<T>(img, dtype, base + stride), load_clean<T>(img, dtype, base - stride)));
}

template <typename T>
__global__ void __launch_bounds__(256) k_gradient_sum(const void* __restrict__ img, int dtype, int H, int W, int C, T* __restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)H * W * C) return;
    const int x = (int)((i / C) % W), y = (int)(i / ((size_t)C * W));
    out[i] = fadd(grad1<T>(img, dtype, i, y, H, (size_t)W * C), grad1<T>(img, dtype, i, x, W, (size_t)C));
}

// ---- materialised Leung-Malik responses -------------------------------------------------------------------------------------

struct Mix { double m[9]; };

// interleaved [H*W, 3] of any dtype -> planar f64 [3, H*W]
__global__ void __launch_bounds__(256) k_to_planar(const void* __restrict__ img, int dtype, size_t hw, double* __restrict__ planar)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 3 * hw) return;
    const size_t c = i / hw, p = i % hw;
    planar[i] = load_as_f64(img, dtype, 3 * p + c);
}

// roll - np.tensordot(mix, smooth, axes=(1, 0)): the background blur folded onto the reflected length-3 channel axis
__global__ void __launch_bounds__(256) k_sub_mix(double* __restrict__ planar, const double* __restrict__ smooth, size_t hw, Mix mix)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 3 * hw) return;
    const size_t c = i / hw, p = i % hw;
    double w[3];   // the row of mix, picked without indexing the parameter (which would copy it to the stack)
#pragma unroll
    for (int j = 0; j < 3; ++j) w[j] = c == 0 ? mix.m[j] : (c == 1 ? mix.m[3 + j] : mix.m[6 + j]);
    const double bg = __dadd_rn(__dadd_rn(__dmul_rn(w[0], smooth[p]), __dmul_rn(w[1], smooth[hw + p])), __dmul_rn(w[2], smooth[2 * hw + p]));
    planar[i] = __dsub_rn(planar[i], bg);
}

constexpr int NORM_BLOCKS = 512;   // fixed, so the summation order does not depend on the device
constexpr int NORM_THREADS = 256;

__device__ __forceinline__ double clip_resp(double v, double vmax) { return v > vmax ? vmax : v; }

// the fixed-order tree sum of one value per thread; every thread gets the total
__device__ __forceinline__ double block_sum(double v, double* s)
{
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = NORM_THREADS / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) s[threadIdx.x] = __dadd_rn(s[threadIdx.x], s[threadIdx.x + o]);
        __syncthreads();
    }
    const double t = s[0];
    __syncthreads();
    return t;
}

// NORM_BLOCKS partial sums of the squared clipped responses resp [3][hw]: of every element (kWhole), or of the pixels [p0, p0 + np)
// of each plane -- the owned rows of a slab.  Both visit the elements in the same order, so a slab that owns all its rows gets the
// whole-image partials.
template <bool kWhole>
__global__ void __launch_bounds__(NORM_THREADS) k_resp_sumsq(const double* __restrict__ resp, size_t n, size_t hw, size_t p0, size_t np,
                                                             double vmax, double* __restrict__ partial)
{
    __shared__ double s[NORM_THREADS];
    double acc = 0.;
    for (size_t i = (size_t)blockIdx.x * NORM_THREADS + threadIdx.x; i < n; i += (size_t)NORM_BLOCKS * NORM_THREADS) {
        const double v = clip_resp(resp[kWhole ? i : (i / np) * hw + p0 + i % np], vmax);
        acc = __dadd_rn(acc, __dmul_rn(v, v));
    }
    const double t = block_sum(acc, s);
    if (threadIdx.x == 0) partial[blockIdx.x] = t;
}

// the sum of the NORM_BLOCKS partials, in one fixed order; every thread gets it
__device__ __forceinline__ double partials_total(const double* __restrict__ partial, double* s)
{
    double acc = 0.;
    for (int j = threadIdx.x; j < NORM_BLOCKS; j += NORM_THREADS) acc = __dadd_rn(acc, partial[j]);
    return block_sum(acc, s);
}

__global__ void __launch_bounds__(NORM_THREADS) k_partials_total(const double* __restrict__ partial, double* __restrict__ total)
{
    __shared__ double s[NORM_THREADS];
    const double t = partials_total(partial, s);
    if (threadIdx.x == 0) *total = t;
}

// (clip(r) * scale) / |r| with scale = log(1 + |r|) / 0.03, or 0 when |r| is 0 or infinite
__device__ __forceinline__ double scaled_resp(double r, double vmax, double scale, double norm, bool zero)
{
    return zero ? 0. : __ddiv_rn(__dmul_rn(clip_resp(r, vmax), scale), norm);
}

// (clip(r) * (log(1 + |r|) / 0.03)) / |r|, or 0 everywhere when |r| is 0 or infinite; planar [3, hw] -> interleaved [hw, 3]
__global__ void __launch_bounds__(NORM_THREADS) k_resp_scale(const double* __restrict__ resp, size_t hw, double vmax,
                                                             const double* __restrict__ partial, double* __restrict__ out)
{
    __shared__ double s[NORM_THREADS];
    const double norm = sqrt(partials_total(partial, s));
    const bool zero = norm == 0. || isinf(norm);
    const double scale = __ddiv_rn(log(__dadd_rn(1., norm)), 0.03);
    for (size_t i = (size_t)blockIdx.x * NORM_THREADS + threadIdx.x; i < 3 * hw; i += (size_t)gridDim.x * NORM_THREADS) {
        const size_t c = i / hw, p = i % hw;
        out[3 * p + c] = scaled_resp(resp[i], vmax, scale, norm, zero);
    }
}

// the same scaling with the norm's square given (summed over the bands of an image): the pixels [p0, p0 + np) of every plane of
// resp [3, hw] -> interleaved out [np, 3]
__global__ void __launch_bounds__(NORM_THREADS) k_resp_scale_rows(const double* __restrict__ resp, size_t hw, size_t p0, size_t np,
                                                                  double vmax, const double* __restrict__ sumsq, double* __restrict__ out)
{
    const double norm = sqrt(*sumsq);
    const bool zero = norm == 0. || isinf(norm);
    const double scale = __ddiv_rn(log(__dadd_rn(1., norm)), 0.03);
    for (size_t i = (size_t)blockIdx.x * NORM_THREADS + threadIdx.x; i < 3 * np; i += (size_t)gridDim.x * NORM_THREADS) {
        const size_t c = i / np, q = i % np;
        out[3 * q + c] = scaled_resp(resp[c * hw + p0 + q], vmax, scale, norm, zero);
    }
}

static unsigned blocks_for(size_t n) { return (unsigned)((n + 255) / 256); }

} // namespace

extern "C" int isb_color_convert(const void* img, int dtype, long long n_px, int space, double* out, isb_stream_t stream)
{
    ISB_REQUIRE(img && out, "null pointer");
    ISB_REQUIRE(n_px > 0, "bad sizes");
    ISB_REQUIRE(dtype >= ISB_U8 && dtype <= ISB_F64, "bad dtype");
    ISB_REQUIRE(space >= ISB_COLOR_HSV && space <= ISB_COLOR_XYZ, "bad colour space");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_STATS, st);
    k_color_convert<<<blocks_for((size_t)n_px), 256, 0, st>>>(img, dtype, n_px, space, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_gradient_sum_2d(const void* img, int dtype, int H, int W, int channels, void* out, isb_stream_t stream)
{
    ISB_REQUIRE(img && out, "null pointer");
    ISB_REQUIRE(H >= 2 && W >= 2, "Shape of array too small to calculate a numerical gradient, at least (edge_order + 1) elements are required.");
    ISB_REQUIRE(channels > 0, "bad sizes");
    ISB_REQUIRE(dtype >= ISB_U8 && dtype <= ISB_F64, "bad dtype");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_STATS, st);
    const size_t n = (size_t)H * W * channels;
    if (dtype == ISB_F32) k_gradient_sum<float><<<blocks_for(n), 256, 0, st>>>(img, dtype, H, W, channels, (float*)out);
    else k_gradient_sum<double><<<blocks_for(n), 256, 0, st>>>(img, dtype, H, W, channels, (double*)out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_lm_background(const void* img, int dtype, int H, int W, const double* w_half, int radius, const double* mix, double* planar,
                                 double* tmp, double* smooth, isb_stream_t stream)
{
    ISB_REQUIRE(img && w_half && mix && planar && tmp && smooth, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && radius >= 0, "bad sizes");
    ISB_REQUIRE(dtype >= ISB_U8 && dtype <= ISB_F64, "bad dtype");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_LM, st);
    const size_t hw = (size_t)H * W;
    Mix m;
    for (int i = 0; i < 9; ++i) m.m[i] = mix[i];
    k_to_planar<<<blocks_for(3 * hw), 256, 0, st>>>(img, dtype, hw, planar);
    ISB_LAUNCH_CHECK();
    const int rc = isb_gaussian_filter_2d(planar, 3, H, W, w_half, radius, tmp, smooth, stream);
    if (rc != ISB_OK) return rc;
    k_sub_mix<<<blocks_for(3 * hw), 256, 0, st>>>(planar, smooth, hw, m);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" size_t isb_lm_battery_workspace_bytes(void) { return isb_align(sizeof(double) * NORM_BLOCKS); }

extern "C" int isb_lm_battery_response(const double* planar, int H, int W, const double* kernels, int n_kernels, int kh, int kw,
                                       double max_signal, double* resp, double* out, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(planar && kernels && resp && out && ws, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0, "bad sizes");
    ISB_REQUIRE(ws_bytes >= isb_lm_battery_workspace_bytes(), "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_LM, st);
    const int rc = isb_filter_response_2d(planar, 3, H, W, kernels, n_kernels, kh, kw, resp, stream);
    if (rc != ISB_OK) return rc;
    const size_t hw = (size_t)H * W;
    k_resp_sumsq<true><<<NORM_BLOCKS, NORM_THREADS, 0, st>>>(resp, 3 * hw, hw, 0, hw, max_signal, (double*)ws);
    ISB_LAUNCH_CHECK();
    const unsigned grid = (unsigned)std::min<size_t>((3 * hw + NORM_THREADS - 1) / NORM_THREADS, 4096);
    k_resp_scale<<<grid, NORM_THREADS, 0, st>>>(resp, hw, max_signal, (const double*)ws, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// ---- the same battery step split for row bands: the norm is summed over the bands between the two calls ------------------------

extern "C" int isb_lm_battery_partial(const double* planar, int H, int W, const double* kernels, int n_kernels, int kh, int kw,
                                      double max_signal, int row_lo, int row_hi, double* resp, double* sumsq, void* ws, size_t ws_bytes,
                                      isb_stream_t stream)
{
    ISB_REQUIRE(planar && kernels && resp && sumsq && ws, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && row_lo >= 0 && row_lo < row_hi && row_hi <= H, "bad sizes");
    ISB_REQUIRE(ws_bytes >= isb_lm_battery_workspace_bytes(), "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_LM, st);
    const int rc = isb_filter_response_2d(planar, 3, H, W, kernels, n_kernels, kh, kw, resp, stream);
    if (rc != ISB_OK) return rc;
    const size_t hw = (size_t)H * W, np = (size_t)(row_hi - row_lo) * W;
    k_resp_sumsq<false><<<NORM_BLOCKS, NORM_THREADS, 0, st>>>(resp, 3 * np, hw, (size_t)row_lo * W, np, max_signal, (double*)ws);
    ISB_LAUNCH_CHECK();
    k_partials_total<<<1, NORM_THREADS, 0, st>>>((const double*)ws, sumsq);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_lm_battery_scale(const double* resp, int H, int W, int row_lo, int row_hi, double max_signal, const double* sumsq,
                                    double* out, isb_stream_t stream)
{
    ISB_REQUIRE(resp && sumsq && out, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && row_lo >= 0 && row_lo < row_hi && row_hi <= H, "bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_LM, st);
    const size_t np = (size_t)(row_hi - row_lo) * W;
    const unsigned grid = (unsigned)std::min<size_t>((3 * np + NORM_THREADS - 1) / NORM_THREADS, 4096);
    k_resp_scale_rows<<<grid, NORM_THREADS, 0, st>>>(resp, (size_t)H * W, (size_t)row_lo * W, np, max_signal, sumsq, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
