// segment_stats.cu -- per-superpixel colour statistics + centroids.
//
// Replaces the reference's native module imsegm/features_cython.pyx:
//   computeColorImage2dMean :81, computeColorImage2dEnergy :101, computeColorImage2dVariance :122,
//   normColorFeatures :59 (count + divide), and regionprops centroids of imsegm/superpixels.py:205-224.
// The reference makes 4 passes over the labels and 3 strided passes over the image PER statistic; here one
// pass produces sum, sum of squares, count and coordinate sums, a second pass the squared deviations from the
// f32 mean (the reference's two-pass variance, descriptors.py:291-295).  Pixels are converted to f32 and the
// products are formed in f32 exactly as the Cython code does (float val; val * val), accumulation is f64.
//
// Mapping: a thread owns one image column inside a strip of SROWS rows, so warp loads are coalesced along x and
// label runs along y (~ one superpixel height) are accumulated in registers; the runs that end in the same row on neighbouring
// lanes with the same label are summed across the warp, and one lane flushes them.  The f64 sums of the flushes are added exactly
// (exact_sum.cuh) and rounded once per label, so a launch gives the same bits whatever order the warps flush in; the integer sums
// (count, rows, columns) keep plain integer atomics.
// Algorithmic HBM bytes: pass 1 = image bytes + 4 B/px labels, pass 2 the same.
#include "exact_sum.cuh"

namespace {

constexpr int SROWS = 16;

struct StatWs {
    double* acc;      // [nb][6]  sum c0..c2, sumsq c0..c2
    double* var;      // [nb][3]
    long long* iacc;  // [nb][3]  count, sum row, sum col
    float* meanf;     // [nb][3]
    long long* xacc;  // [nb][6][XS_DIGITS]  exact sums of pass 1, rounded into acc
    unsigned* xflag1; // [nb]
    long long* xvar;  // [nb][3][XS_DIGITS]  exact sums of pass 2, rounded into var
    unsigned* xflag2; // [nb]
};

__device__ __forceinline__ float clean(float v) { return isnan(v) ? 0.0f : v; } // np.nan_to_num (descriptors.py:824)

// Runs that end in the same row on neighbouring lanes of a warp with the same label (a boundary across the columns, or the end of the
// strip) are summed across those lanes before one lane flushes them.  A segment is a maximal group of consecutive flushing lanes with
// one key; every lane of the warp calls this.  Returns the lane one past the segment that starts at or spans this lane (use it with
// seg_sum); *head tells whether this lane is the segment's first, the one that holds its sum.
__device__ __forceinline__ int run_segment_end(bool flush, int key, bool* head)
{
    const int lane = threadIdx.x & 31;
    const unsigned fl = __ballot_sync(0xffffffffu, flush);
    const int prev = __shfl_up_sync(0xffffffffu, key, 1);
    *head = flush && !(lane > 0 && ((fl >> (lane - 1)) & 1) && prev == key);
    const unsigned starts = __ballot_sync(0xffffffffu, !flush || *head) & ~((2u << lane) - 1u); // segment starts above this lane
    return starts ? __ffs(starts) - 1 : 32;
}

// after log2(32) steps lane i holds the sum of lanes [i, end): each step adds the partial of lane i + o when that lane is in the segment
template <typename T> __device__ __forceinline__ T seg_sum(T v, int end)
{
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T u = __shfl_down_sync(0xffffffffu, v, o);
        if (lane + o < end) v += u;
    }
    return v;
}

// Every lane of a warp walks the y loop to its end (the shuffles of the flush need all 32), lanes beyond W with no label.  The next
// row's label and pixel are loaded before the current row's flush, so two rows of loads are in flight per thread.
__global__ void __launch_bounds__(256) k_stats_pass1(const void* __restrict__ img, int dtype, const int* __restrict__ seg, int H, int W,
                                                     int y_off, StatWs ws)
{
    const int x = blockIdx.x * 256 + threadIdx.x;
    const bool live = x < W;
    const int y0 = blockIdx.y * SROWS, y1 = min(y0 + SROWS, H);
    int cur = -1;
    double s0 = 0, s1 = 0, s2 = 0, e0 = 0, e1 = 0, e2 = 0;
    int cnt = 0;
    long long sy = 0;
    int nl = -1;
    float n0 = 0, n1 = 0, n2 = 0;
    auto load = [&](int y) {
        nl = -1;
        if (live && y < y1) {
            const size_t p = (size_t)y * W + x;
            nl = seg[p];
            if (img) { n0 = clean(load_as_f32(img, dtype, 3 * p)); n1 = clean(load_as_f32(img, dtype, 3 * p + 1)); n2 = clean(load_as_f32(img, dtype, 3 * p + 2)); }
        }
    };
    load(y0);
    for (int y = y0; y <= y1; ++y) {
        const int l = nl;
        const float v0 = n0, v1 = n1, v2 = n2;
        load(y + 1);
        const bool flush = cur >= 0 && l != cur;
        if (__any_sync(0xffffffffu, flush)) {
            bool head;
            const int end = run_segment_end(flush, cur, &head);
            const double t0 = seg_sum(s0, end), t1 = seg_sum(s1, end), t2 = seg_sum(s2, end);
            const double u0 = seg_sum(e0, end), u1 = seg_sum(e1, end), u2 = seg_sum(e2, end);
            const int tc = seg_sum(cnt, end);
            const long long ty = seg_sum(sy, end), tx = seg_sum((long long)cnt * x, end);
            if (head) {
                long long* xa = ws.xacc + 6 * XS_DIGITS * (size_t)cur;
                unsigned* fl = ws.xflag1 + cur;
                xs_add(xa, fl, 0, t0); xs_add(xa + XS_DIGITS, fl, 1, t1); xs_add(xa + 2 * XS_DIGITS, fl, 2, t2);
                xs_add(xa + 3 * XS_DIGITS, fl, 3, u0); xs_add(xa + 4 * XS_DIGITS, fl, 4, u1); xs_add(xa + 5 * XS_DIGITS, fl, 5, u2);
                unsigned long long* ia = (unsigned long long*)(ws.iacc + 3 * (size_t)cur);
                atomicAdd(ia, (unsigned long long)tc);
                atomicAdd(ia + 1, (unsigned long long)ty);
                atomicAdd(ia + 2, (unsigned long long)tx);
            }
        }
        if (l != cur) {
            cur = l;
            s0 = s1 = s2 = e0 = e1 = e2 = 0;
            cnt = 0; sy = 0;
        }
        if (l >= 0) {
            s0 += (double)v0; s1 += (double)v1; s2 += (double)v2;
            e0 += (double)__fmul_rn(v0, v0); e1 += (double)__fmul_rn(v1, v1); e2 += (double)__fmul_rn(v2, v2);
            cnt += 1; sy += y + y_off;
        }
    }
}

__global__ void k_stats_means(int nb, StatWs ws)
{
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nb) return;
    long long c = ws.iacc[3 * (size_t)k];
    for (int z = 0; z < 3; ++z) {
        double m = ws.acc[6 * (size_t)k + z];
        if (c > 0) m = m / (double)c;
        ws.meanf[3 * (size_t)k + z] = (float)m; // np.array(means, dtype=np.float32), descriptors.py:293
    }
}

// the same walk as pass 1 over the squared deviations from the f32 mean
__global__ void __launch_bounds__(256) k_stats_pass2(const void* __restrict__ img, int dtype, const int* __restrict__ seg, int H, int W,
                                                     StatWs ws)
{
    const int x = blockIdx.x * 256 + threadIdx.x;
    const bool live = x < W;
    const int y0 = blockIdx.y * SROWS, y1 = min(y0 + SROWS, H);
    int cur = -1;
    double a0 = 0, a1 = 0, a2 = 0;
    float m0 = 0, m1 = 0, m2 = 0;
    int nl = -1;
    float n0 = 0, n1 = 0, n2 = 0;
    auto load = [&](int y) {
        nl = -1;
        if (live && y < y1) {
            const size_t p = (size_t)y * W + x;
            nl = seg[p];
            n0 = clean(load_as_f32(img, dtype, 3 * p)); n1 = clean(load_as_f32(img, dtype, 3 * p + 1)); n2 = clean(load_as_f32(img, dtype, 3 * p + 2));
        }
    };
    load(y0);
    for (int y = y0; y <= y1; ++y) {
        const int l = nl;
        const float v0 = n0, v1 = n1, v2 = n2;
        load(y + 1);
        const bool flush = cur >= 0 && l != cur;
        if (__any_sync(0xffffffffu, flush)) {
            bool head;
            const int end = run_segment_end(flush, cur, &head);
            const double t0 = seg_sum(a0, end), t1 = seg_sum(a1, end), t2 = seg_sum(a2, end);
            if (head) {
                long long* xv = ws.xvar + 3 * XS_DIGITS * (size_t)cur;
                unsigned* fl = ws.xflag2 + cur;
                xs_add(xv, fl, 0, t0); xs_add(xv + XS_DIGITS, fl, 1, t1); xs_add(xv + 2 * XS_DIGITS, fl, 2, t2);
            }
        }
        if (l != cur) {
            cur = l;
            a0 = a1 = a2 = 0;
            if (l >= 0) { m0 = ws.meanf[3 * (size_t)l]; m1 = ws.meanf[3 * (size_t)l + 1]; m2 = ws.meanf[3 * (size_t)l + 2]; }
        }
        if (l >= 0) {
            const float d0 = __fsub_rn(v0, m0), d1 = __fsub_rn(v1, m1), d2 = __fsub_rn(v2, m2);
            a0 += (double)__fmul_rn(d0, d0); a1 += (double)__fmul_rn(d1, d1); a2 += (double)__fmul_rn(d2, d2);
        }
    }
}

__device__ __forceinline__ double tidy(double v)
{
    if (isnan(v)) return 0.0;          // np.nan_to_num (descriptors.py:857)
    if (isinf(v)) return v > 0 ? 1.7976931348623157e308 : -1.7976931348623157e308;
    return v == 0.0 ? 0.0 : v;         // features[features == 0] = 0  (-0 -> +0)
}

__global__ void k_stats_finalize(int nb, int flags, StatWs ws, double* feat, int ld, int col0, double* centres, int* counts)
{
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nb) return;
    long long c = ws.iacc[3 * (size_t)k];
    double dn = (double)c;
    int col = col0;
    double* row = feat ? feat + (size_t)k * ld : nullptr;
    if (row) {
        if (flags & 1) { for (int z = 0; z < 3; ++z) { double v = ws.acc[6 * (size_t)k + z]; if (c > 0) v = v / dn; row[col++] = tidy(v); } }
        if (flags & 2) { for (int z = 0; z < 3; ++z) { double v = ws.var[3 * (size_t)k + z]; if (c > 0) v = v / dn; row[col++] = tidy(sqrt(v)); } }
        if (flags & 4) { for (int z = 0; z < 3; ++z) { double v = ws.acc[6 * (size_t)k + 3 + z]; if (c > 0) v = v / dn; row[col++] = tidy(v); } }
    }
    if (centres) {
        if (c > 0) { centres[2 * (size_t)k] = (double)ws.iacc[3 * (size_t)k + 1] / dn; centres[2 * (size_t)k + 1] = (double)ws.iacc[3 * (size_t)k + 2] / dn; }
        else { centres[2 * (size_t)k] = -1.0; centres[2 * (size_t)k + 1] = -1.0; }
    }
    if (counts) counts[k] = (int)c;
}

// dense tables first, then the exact sums of pass 1 (from *x1) and of pass 2 (from *x2), each a contiguous range that its pass zeroes
static size_t carve(StatWs& w, void* ws, size_t bytes, int nb, size_t* x1 = nullptr, size_t* x2 = nullptr)
{
    WsCarver c(ws, bytes);
    w.acc = c.take<double>(6 * (size_t)nb);
    w.var = c.take<double>(3 * (size_t)nb);
    w.iacc = c.take<long long>(3 * (size_t)nb);
    w.meanf = c.take<float>(3 * (size_t)nb);
    const size_t o1 = isb_align(c.off);
    const size_t o2 = o1 + xs_carve((char*)ws + o1, nb, 6, &w.xacc, &w.xflag1);
    const size_t end = o2 + xs_carve((char*)ws + o2, nb, 3, &w.xvar, &w.xflag2);
    if (x1) *x1 = o1;
    if (x2) *x2 = o2;
    return end;
}

// pass 1 into the exact sums w.xacc / w.xflag1 (the xbytes from x, zeroed here), rounded and added into w.acc; the integer sums
// go straight into w.iacc
static int stats_pass1(const void* img, int dtype, const int32_t* seg, int H, int W, int y_off, int nb, const StatWs& w, void* x,
                       size_t xbytes, cudaStream_t st)
{
    ISB_CUDA_CHECK(cudaMemsetAsync(x, 0, xbytes, st));
    k_stats_pass1<<<dim3((W + 255) / 256, (H + SROWS - 1) / SROWS), 256, 0, st>>>(img, dtype, seg, H, W, y_off, w);
    ISB_LAUNCH_CHECK();
    k_exact_fold<<<(unsigned)((6 * (long long)nb + 255) / 256), 256, 0, st>>>(nb, 6, w.xacc, w.xflag1, w.acc);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// the f32 means from w.acc / w.iacc into w.meanf, pass 2 into the exact sums w.xvar / w.xflag2 (the xbytes from x, zeroed here),
// rounded and added into w.var
static int stats_pass2(const void* img, int dtype, const int32_t* seg, int H, int W, int nb, const StatWs& w, void* x, size_t xbytes,
                       cudaStream_t st)
{
    ISB_CUDA_CHECK(cudaMemsetAsync(x, 0, xbytes, st));
    k_stats_means<<<(nb + 255) / 256, 256, 0, st>>>(nb, w);
    ISB_LAUNCH_CHECK();
    k_stats_pass2<<<dim3((W + 255) / 256, (H + SROWS - 1) / SROWS), 256, 0, st>>>(img, dtype, seg, H, W, w);
    ISB_LAUNCH_CHECK();
    k_exact_fold<<<(unsigned)((3 * (long long)nb + 255) / 256), 256, 0, st>>>(nb, 3, w.xvar, w.xflag2, w.var);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

} // namespace

// a label's exact sums take one partial per flush, at most one per pixel: 2^31 of them fit (exact_sum.cuh)
#define ISB_REQUIRE_FLUSHES(npx) ISB_REQUIRE((npx) <= (1ll << 31), "more than 2^31 pixels in one call")

extern "C" size_t isb_segment_stats_workspace_bytes(int nb)
{
    StatWs w;
    return carve(w, nullptr, 0, nb);
}

extern "C" int isb_segment_stats_2d(const void* img, int dtype, const int32_t* seg, int H, int W, int nb, int flags, double* feat,
                                    int ld, int col0, double* centres, int32_t* counts, void* ws, size_t ws_bytes,
                                    isb_stream_t stream)
{
    ISB_REQUIRE(seg && ws && (img || (flags & 7) == 0), "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && nb > 0, "bad sizes");
    ISB_REQUIRE_FLUSHES((long long)H * W);
    ISB_REQUIRE(dtype >= ISB_U8 && dtype <= ISB_F64, "bad dtype");
    StatWs w;
    size_t x1, x2;
    const size_t need = carve(w, ws, ws_bytes, nb, &x1, &x2);
    ISB_REQUIRE(need <= ws_bytes, "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_STATS, st);
    ISB_CUDA_CHECK(cudaMemsetAsync(ws, 0, x1, st));
    if (int rc = stats_pass1(img, dtype, seg, H, W, 0, nb, w, (char*)ws + x1, x2 - x1, st)) return rc;
    if (flags & 2)
        if (int rc = stats_pass2(img, dtype, seg, H, W, nb, w, (char*)ws + x2, need - x2, st)) return rc;
    k_stats_finalize<<<(nb + 255) / 256, 256, 0, st>>>(nb, flags, w, feat, ld, col0, centres, counts);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// ---- caller-owned accumulators (row bands of one image merged by a collective between the calls) -------------------------
// The band's exact sums live in memory allocated on the caller's stream for the call.

extern "C" int isb_segment_stats_accumulate(const void* img, int dtype, const int32_t* seg, int H, int W, int y_off, int nb, double* acc,
                                            int64_t* iacc, isb_stream_t stream)
{
    ISB_REQUIRE(seg && acc && iacc, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && nb > 0 && y_off >= 0, "bad sizes");
    ISB_REQUIRE_FLUSHES((long long)H * W);
    ISB_REQUIRE(dtype >= ISB_U8 && dtype <= ISB_F64, "bad dtype");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_STATS, st);
    StatWs w;
    w.acc = acc; w.iacc = (long long*)iacc; w.var = nullptr; w.meanf = nullptr; w.xvar = nullptr; w.xflag2 = nullptr;
    const size_t xb = xs_carve(nullptr, nb, 6, &w.xacc, &w.xflag1);
    StreamScratch x(st);
    ISB_CUDA_CHECK(cudaMallocAsync(&x.p, xb, st));
    xs_carve(x.p, nb, 6, &w.xacc, &w.xflag1);
    return stats_pass1(img, dtype, seg, H, W, y_off, nb, w, x.p, xb, st);
}

extern "C" int isb_segment_stats_deviation(const void* img, int dtype, const int32_t* seg, int H, int W, int nb, const double* acc,
                                           const int64_t* iacc, float* meanf_scratch, double* var, isb_stream_t stream)
{
    ISB_REQUIRE(img && seg && acc && iacc && meanf_scratch && var, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && nb > 0, "bad sizes");
    ISB_REQUIRE_FLUSHES((long long)H * W);
    ISB_REQUIRE(dtype >= ISB_U8 && dtype <= ISB_F64, "bad dtype");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_STATS, st);
    StatWs w;
    w.acc = (double*)acc; w.iacc = (long long*)iacc; w.var = var; w.meanf = meanf_scratch; w.xacc = nullptr; w.xflag1 = nullptr;
    const size_t xb = xs_carve(nullptr, nb, 3, &w.xvar, &w.xflag2);
    StreamScratch x(st);
    ISB_CUDA_CHECK(cudaMallocAsync(&x.p, xb, st));
    xs_carve(x.p, nb, 3, &w.xvar, &w.xflag2);
    return stats_pass2(img, dtype, seg, H, W, nb, w, x.p, xb, st);
}

extern "C" int isb_segment_stats_finish(int nb, int flags, const double* acc, const double* var, const int64_t* iacc, double* feat, int ld,
                                        int col0, double* centres, int32_t* counts, isb_stream_t stream)
{
    ISB_REQUIRE(acc && iacc && (var || !(flags & 2)), "null pointer");
    ISB_REQUIRE(nb > 0, "bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    StatWs w;
    w.acc = (double*)acc; w.iacc = (long long*)iacc; w.var = (double*)var; w.meanf = nullptr;
    k_stats_finalize<<<(nb + 255) / 256, 256, 0, st>>>(nb, flags, w, feat, ld, col0, centres, counts);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
