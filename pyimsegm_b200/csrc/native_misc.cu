// native_misc.cu -- the remaining functions of the reference's native module imsegm/features_cython.pyx:
//   computeGrayImage3dMean :144, ...Energy :169, ...Variance :194   (f32 voxels, f64 accumulators; one channel, any rank)
//   computeLabelHistogram2d :222                                     (labels under a structuring element)
//   computeRayFeaturesBinary2d :239                                  (distance to the first boundary along rays, f32 marching)
// They sit beside the hot path (3-D gray pipeline, RG2SP / centre detection: SURVEY.md section 8f) and are provided so that
// the whole native surface of the reference has a device entry point.
#include "exact_sum.cuh"

namespace {

constexpr int GSTRIP = 16;

__device__ __forceinline__ float clean(float v) { return isnan(v) ? 0.0f : v; }

// pass 0: sum, sum of squares (f32 product) -> exact sums x [nb][2][XS_DIGITS], count -> cnt.  pass 1: sum (v - mean_f32)^2 -> x [nb][1][..]
// (the variance sums).  Every run a thread ends flushes its partials into the label's exact sums (exact_sum.cuh), so the totals do
// not depend on the order of the flushes.
__global__ void __launch_bounds__(256) k_gray_stats(const void* __restrict__ img, int dtype, const int* __restrict__ seg, long long n, int pass,
                                                    long long* x, unsigned* xflag, long long* cnt, const float* meanf)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long beg = t * GSTRIP, end = min(beg + GSTRIP, n);
    if (beg >= n) return;
    int cur = -1;
    double s = 0, e = 0;
    long long c = 0;
    float m = 0.f;
    for (long long i = beg; i <= end; ++i) {
        const int l = i < end ? seg[i] : -1;
        if (l != cur) {
            if (cur >= 0) {
                if (pass == 0) {
                    long long* xa = x + 2 * XS_DIGITS * (size_t)cur;
                    xs_add(xa, xflag + cur, 0, s); xs_add(xa + XS_DIGITS, xflag + cur, 1, e);
                    atomicAdd((unsigned long long*)&cnt[cur], (unsigned long long)c);
                } else xs_add(x + XS_DIGITS * (size_t)cur, xflag + cur, 0, s);
            }
            cur = l; s = 0; e = 0; c = 0;
            if (pass == 1 && l >= 0) m = meanf[l];
        }
        if (i < end) {
            const float v = clean(load_as_f32(img, dtype, (size_t)i));
            if (pass == 0) { s += (double)v; e += (double)__fmul_rn(v, v); c += 1; }
            else { const float d = __fsub_rn(v, m); s += (double)__fmul_rn(d, d); }
        }
    }
}

__global__ void k_gray_means(int nb, const double* acc, const long long* cnt, float* meanf)
{
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nb) return;
    double m = acc[2 * (size_t)k];
    if (cnt[k] > 0) m = m / (double)cnt[k];
    meanf[k] = (float)m;
}

__global__ void k_gray_finalize(int nb, int flags, const double* acc, const double* var, const long long* cnt, double* feat, int ld, int col0)
{
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nb) return;
    const long long c = cnt[k];
    int col = col0;
    double* row = feat + (size_t)k * ld;
    for (int st = 0; st < 3; ++st) {
        if (!(flags & (1 << st))) continue;
        double v = st == 0 ? acc[2 * (size_t)k] : (st == 1 ? var[k] : acc[2 * (size_t)k + 1]);
        if (c > 0) v = v / (double)c;
        if (st == 1) v = sqrt(v);
        row[col++] = isnan(v) ? 0.0 : (v == 0.0 ? 0.0 : v);
    }
}

__global__ void k_label_hist(const short* __restrict__ segm, const short* __restrict__ selem, long long n, int nb_labels, unsigned* hist)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int l = segm[i];
    if (l >= 0 && l < nb_labels && selem[i] == 1) atomicAdd(&hist[l], 1u);
}

// one thread per (position, angle).  Positions lie in [-H, H) x [-W, W) (checked by the caller): like the reference's
// wraparound memoryview, a negative start reads pixel (H + pr, W + pc) while the march starts from (pr, pc).  The reference
// rounds the marching position with Python's round(), half to even, which is rintf on these non-negative values.
__global__ void k_ray_features(const signed char* __restrict__ seg, int H, int W, const int* __restrict__ pos, int n_pos, const float* __restrict__ sin_a,
                               const float* __restrict__ cos_a, int n_ang, int edge, float* __restrict__ out)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_pos * n_ang) return;
    const int p = t / n_ang, i = t - p * n_ang;
    const int pr = pos[2 * p], pc = pos[2 * p + 1];
    const signed char start = seg[(size_t)(pr < 0 ? pr + H : pr) * W + (pc < 0 ? pc + W : pc)];
    if (start && edge == 1) { out[t] = 0.0f; return; } // the position sits inside the border label
    float dist = -1.0f;
    const int diag = (int)sqrt((double)W * W + (double)H * H);
    float pos0 = (float)pr, pos1 = (float)pc;
    float g0 = sin_a[i], g1 = cos_a[i];
    const float gmax = fmaxf(fabsf(g0), fabsf(g1));
    g0 = __fdiv_rn(g0, gmax); g1 = __fdiv_rn(g1, gmax);
    signed char last = start;
    for (int s = 0; s < diag; ++s) {
        pos0 = __fadd_rn(pos0, g0); pos1 = __fadd_rn(pos1, g1);
        if (pos0 < 0 || rintf(pos0) >= H || pos1 < 0 || rintf(pos1) >= W) break;
        const signed char actual = seg[(size_t)((int)rintf(pos0)) * W + (int)rintf(pos1)];
        if ((edge == 1 && actual) || (edge == -1 && last && !actual)) {
            const float dx = __fsub_rn(pos0, (float)pr), dy = __fsub_rn(pos1, (float)pc);
            dist = (float)sqrt((double)__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
            break;
        }
        last = actual;
    }
    out[t] = dist;
}

// joint histogram of two label maps: hist[a][b] = #{p : slic[p] == a, annot[p] == b}; a thread walks a short column strip so
// that runs of equal (a, b) cost one atomic.  A pixel with a negative label in either map is not counted
// (compute_labels_overlap_matrix, imsegm/labeling.py:519-521).
__global__ void __launch_bounds__(256) k_region_label_hist(const int* __restrict__ slic, const int* __restrict__ annot, int H, int W, int nb_annot,
                                                           unsigned* hist)
{
    const int x = blockIdx.x * 256 + threadIdx.x;
    if (x >= W) return;
    const int y0 = blockIdx.y * GSTRIP, y1 = min(y0 + GSTRIP, H);
    int ca = -1, cb = -1;
    unsigned run = 0;
    for (int y = y0; y <= y1; ++y) {
        int a = -1, b = -1;
        if (y < y1) { a = slic[(size_t)y * W + x]; b = annot[(size_t)y * W + x]; }
        if (a != ca || b != cb) {
            if (run && ca >= 0 && cb >= 0) atomicAdd(&hist[(size_t)ca * nb_annot + cb], run);
            ca = a; cb = b; run = 0;
        }
        if (y < y1) ++run;
    }
}

} // namespace

extern "C" int isb_region_label_hist(const int32_t* slic, const int32_t* annot, int H, int W, int nb_slic, int nb_annot, uint32_t* hist,
                                     isb_stream_t stream)
{
    ISB_REQUIRE(slic && annot && hist && H > 0 && W > 0 && nb_slic > 0 && nb_annot > 0, "bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    ISB_CUDA_CHECK(cudaMemsetAsync(hist, 0, sizeof(uint32_t) * (size_t)nb_slic * nb_annot, st));
    k_region_label_hist<<<dim3((W + 255) / 256, (H + GSTRIP - 1) / GSTRIP), 256, 0, st>>>(slic, annot, H, W, nb_annot, hist);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

namespace {

struct GrayWs {
    double* acc;      // [nb][2] sum, sum of squares
    long long* cnt;   // [nb]
    float* meanf;     // [nb]
    double* var;      // [nb]
    long long* xacc;  // [nb][2][XS_DIGITS]  exact sums of pass 0, rounded into acc
    unsigned* xflag0; // [nb]
    long long* xvar;  // [nb][XS_DIGITS]     exact sums of pass 1, rounded into var
    unsigned* xflag1; // [nb]
};

// dense tables first, then the exact sums of pass 0 (from *x0) and of pass 1 (from *x1), each a contiguous range that its pass zeroes
static size_t carve_gray(GrayWs& w, void* ws, size_t bytes, int nb, size_t* x0 = nullptr, size_t* x1 = nullptr)
{
    WsCarver c(ws, bytes);
    w.acc = c.take<double>(2 * (size_t)nb);
    w.cnt = c.take<long long>(nb);
    w.meanf = c.take<float>(nb);
    w.var = c.take<double>(nb);
    const size_t o0 = isb_align(c.off);
    const size_t o1 = o0 + xs_carve((char*)ws + o0, nb, 2, &w.xacc, &w.xflag0);
    const size_t end = o1 + xs_carve((char*)ws + o1, nb, 1, &w.xvar, &w.xflag1);
    if (x0) *x0 = o0;
    if (x1) *x1 = o1;
    return end;
}

static unsigned gray_blocks(long long n) { return (unsigned)(((n + GSTRIP - 1) / GSTRIP + 255) / 256); }

// pass 0 into the exact sums (xbytes from x, zeroed here: digits xacc, flags xflag), rounded and added into acc; counts into cnt
static int gray_pass0(const void* img, int dtype, const int32_t* seg, long long n, int nb, double* acc, int64_t* cnt, long long* xacc,
                      unsigned* xflag, void* x, size_t xbytes, cudaStream_t st)
{
    ISB_CUDA_CHECK(cudaMemsetAsync(x, 0, xbytes, st));
    k_gray_stats<<<gray_blocks(n), 256, 0, st>>>(img, dtype, seg, n, 0, xacc, xflag, (long long*)cnt, nullptr);
    ISB_LAUNCH_CHECK();
    k_exact_fold<<<(unsigned)((2 * (long long)nb + 255) / 256), 256, 0, st>>>(nb, 2, xacc, xflag, acc);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// the f32 means into meanf, pass 1 into the exact sums (as pass 0), rounded and added into var
static int gray_pass1(const void* img, int dtype, const int32_t* seg, long long n, int nb, const double* acc, const int64_t* cnt,
                      float* meanf, double* var, long long* xvar, unsigned* xflag, void* x, size_t xbytes, cudaStream_t st)
{
    ISB_CUDA_CHECK(cudaMemsetAsync(x, 0, xbytes, st));
    k_gray_means<<<(nb + 255) / 256, 256, 0, st>>>(nb, acc, (const long long*)cnt, meanf);
    ISB_LAUNCH_CHECK();
    k_gray_stats<<<gray_blocks(n), 256, 0, st>>>(img, dtype, seg, n, 1, xvar, xflag, nullptr, meanf);
    ISB_LAUNCH_CHECK();
    k_exact_fold<<<(unsigned)((nb + 255) / 256), 256, 0, st>>>(nb, 1, xvar, xflag, var);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

} // namespace

// a label's exact sums take one partial per flushed run, at most one per voxel: 2^31 of them fit (exact_sum.cuh)
#define ISB_REQUIRE_FLUSHES(n) ISB_REQUIRE((n) <= (1ll << 31), "more than 2^31 voxels in one call")

extern "C" size_t isb_gray_stats_workspace_bytes(int nb)
{
    GrayWs w;
    return carve_gray(w, nullptr, 0, nb);
}

// the slab's exact sums live in memory allocated on the caller's stream for the call
extern "C" int isb_gray_stats_accumulate(const void* img, int dtype, const int32_t* seg, long long n, int nb, double* acc, int64_t* cnt,
                                         isb_stream_t stream)
{
    ISB_REQUIRE(img && seg && acc && cnt, "null pointer");
    ISB_REQUIRE(n > 0 && nb > 0 && dtype >= ISB_U8 && dtype <= ISB_F64, "bad arguments");
    ISB_REQUIRE_FLUSHES(n);
    cudaStream_t st = (cudaStream_t)stream;
    long long* xacc;
    unsigned* xflag;
    const size_t xb = xs_carve(nullptr, nb, 2, &xacc, &xflag);
    StreamScratch x(st);
    ISB_CUDA_CHECK(cudaMallocAsync(&x.p, xb, st));
    xs_carve(x.p, nb, 2, &xacc, &xflag);
    return gray_pass0(img, dtype, seg, n, nb, acc, cnt, xacc, xflag, x.p, xb, st);
}

extern "C" int isb_gray_stats_deviation(const void* img, int dtype, const int32_t* seg, long long n, int nb, const double* acc,
                                        const int64_t* cnt, float* meanf_scratch, double* var, isb_stream_t stream)
{
    ISB_REQUIRE(img && seg && acc && cnt && meanf_scratch && var, "null pointer");
    ISB_REQUIRE(n > 0 && nb > 0 && dtype >= ISB_U8 && dtype <= ISB_F64, "bad arguments");
    ISB_REQUIRE_FLUSHES(n);
    cudaStream_t st = (cudaStream_t)stream;
    long long* xvar;
    unsigned* xflag;
    const size_t xb = xs_carve(nullptr, nb, 1, &xvar, &xflag);
    StreamScratch x(st);
    ISB_CUDA_CHECK(cudaMallocAsync(&x.p, xb, st));
    xs_carve(x.p, nb, 1, &xvar, &xflag);
    return gray_pass1(img, dtype, seg, n, nb, acc, cnt, meanf_scratch, var, xvar, xflag, x.p, xb, st);
}

extern "C" int isb_gray_stats_finish(int nb, int flags, const double* acc, const double* var, const int64_t* cnt, double* feat, int ld,
                                     int col0, isb_stream_t stream)
{
    ISB_REQUIRE(acc && cnt && feat && (var || !(flags & 2)), "null pointer");
    ISB_REQUIRE(nb > 0, "bad sizes");
    k_gray_finalize<<<(nb + 255) / 256, 256, 0, (cudaStream_t)stream>>>(nb, flags, acc, var, (const long long*)cnt, feat, ld, col0);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_gray_stats(const void* img, int dtype, const int32_t* seg, long long n, int nb, int flags, double* feat, int ld, int col0,
                              void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(img && seg && feat && ws, "null pointer");
    ISB_REQUIRE(n > 0 && nb > 0 && dtype >= ISB_U8 && dtype <= ISB_F64, "bad arguments");
    ISB_REQUIRE_FLUSHES(n);
    GrayWs w;
    size_t x0, x1;
    const size_t need = carve_gray(w, ws, ws_bytes, nb, &x0, &x1);
    ISB_REQUIRE(need <= ws_bytes, "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    ISB_CUDA_CHECK(cudaMemsetAsync(ws, 0, x0, st));
    if (int rc = gray_pass0(img, dtype, seg, n, nb, w.acc, (int64_t*)w.cnt, w.xacc, w.xflag0, (char*)ws + x0, x1 - x0, st)) return rc;
    if (flags & 2)
        if (int rc = gray_pass1(img, dtype, seg, n, nb, w.acc, (const int64_t*)w.cnt, w.meanf, w.var, w.xvar, w.xflag1, (char*)ws + x1,
                                need - x1, st)) return rc;
    return isb_gray_stats_finish(nb, flags, w.acc, w.var, (const int64_t*)w.cnt, feat, ld, col0, stream);
}

extern "C" int isb_label_hist_2d(const int16_t* segm_select, const int16_t* struc_elem, int H, int W, int nb_labels, uint32_t* hist,
                                 isb_stream_t stream)
{
    ISB_REQUIRE(segm_select && struc_elem && hist && H > 0 && W > 0 && nb_labels > 0, "bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    ISB_CUDA_CHECK(cudaMemsetAsync(hist, 0, sizeof(uint32_t) * (size_t)nb_labels, st));
    const long long n = (long long)H * W;
    k_label_hist<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(segm_select, struc_elem, n, nb_labels, hist);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_ray_features_2d(const int8_t* seg_binary, int H, int W, const int32_t* positions, int n_pos, const float* sin_a,
                                   const float* cos_a, int n_ang, int edge, float* out, isb_stream_t stream)
{
    ISB_REQUIRE(seg_binary && positions && sin_a && cos_a && out, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && n_pos > 0 && n_ang > 0 && (edge == 1 || edge == -1), "bad arguments");
    const int n = n_pos * n_ang;
    k_ray_features<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(seg_binary, H, W, positions, n_pos, sin_a, cos_a, n_ang, edge, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// compute_label_histograms_positions (imsegm/descriptors.py:1288-1352): label histograms under discs of growing diameter
// about a list of positions.  The reference crops the segmentation and a skimage.morphology.disk(d) mask per (position,
// diameter) and calls computeLabelHistogram2d on the crop; here ONE launch covers every (position, diameter): a CTA per pair
// walks the disc {(dy, dx): dy^2 + dx^2 <= d^2} clipped to the image (= adjust_bounding_box_crop, descriptors.py:1355-1393).
//   segm   : [H, W] int32 labels (entries outside [0, nb_labels) are ignored), or -- when proba != nullptr -- unused
//   proba  : optional [H, W, nb_labels] f64 (compute_label_hist_proba :1501-1528): hist[l] = sum of proba[..., l] under the disc
//   hist   : out [n_pos, n_diam, nb_labels] f64;  sizes: out [n_pos, n_diam] f64 = pixels of the (clipped) disc
//   selem  : optional explicit structuring element [mh, mw] u8 instead of the discs (then n_diam == 1): compute_label_hist_segm /
//            compute_label_hist_proba with any mask; mask pixel (iy, ix) sits on image pixel (row - mh/2 + iy, col - mw/2 + ix)
// ---------------------------------------------------------------------------------------------------------------------
namespace {

__global__ void __launch_bounds__(256) k_disc_hist(const int* __restrict__ segm, const double* __restrict__ proba, int H, int W,
                                                   const int* __restrict__ positions, const int* __restrict__ diameters, int n_diam,
                                                   const unsigned char* __restrict__ selem, int mh, int mw, int nb_labels,
                                                   double* __restrict__ hist, double* __restrict__ sizes)
{
    extern __shared__ double s_hist[];   // [nb_labels] + 1 (size)
    const int ip = blockIdx.x / n_diam, id = blockIdx.x % n_diam;
    const int py = positions[2 * ip], px = positions[2 * ip + 1], d = selem ? 0 : diameters[id];
    for (int i = threadIdx.x; i <= nb_labels; i += blockDim.x) s_hist[i] = 0.0;
    __syncthreads();
    const int sh = selem ? mh : 2 * d + 1, sw = selem ? mw : 2 * d + 1;
    const int oy = selem ? mh / 2 : d, ox = selem ? mw / 2 : d;
    double cnt = 0;
    for (int i = threadIdx.x; i < sh * sw; i += blockDim.x) {
        const int dy = i / sw - oy, dx = i % sw - ox;
        if (selem ? selem[i] != 1 : dy * dy + dx * dx > d * d) continue;
        const int y = py + dy, x = px + dx;
        if (y < 0 || y >= H || x < 0 || x >= W) continue;
        cnt += 1.0;
        if (proba) {
            const double* p = proba + ((size_t)y * W + x) * nb_labels;
            for (int l = 0; l < nb_labels; ++l) atomicAdd(&s_hist[l], p[l]);
        } else {
            const int l = segm[(size_t)y * W + x];
            if (l >= 0 && l < nb_labels) atomicAdd(&s_hist[l], 1.0);
        }
    }
    atomicAdd(&s_hist[nb_labels], cnt);
    __syncthreads();
    double* out = hist + ((size_t)ip * n_diam + id) * nb_labels;
    for (int i = threadIdx.x; i < nb_labels; i += blockDim.x) out[i] = s_hist[i];
    if (threadIdx.x == 0) sizes[(size_t)ip * n_diam + id] = s_hist[nb_labels];
}

} // namespace

extern "C" int isb_disc_label_hist(const int32_t* segm, const double* proba, int H, int W, const int32_t* positions, int n_pos,
                                   const int32_t* diameters, int n_diam, const uint8_t* selem, int mh, int mw, int nb_labels,
                                   double* hist, double* sizes, isb_stream_t stream)
{
    ISB_REQUIRE((segm || proba) && positions && (diameters || selem) && hist && sizes, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && n_pos > 0 && n_diam > 0 && nb_labels > 0 && nb_labels <= 4096, "bad sizes");
    ISB_REQUIRE(!selem || (n_diam == 1 && mh > 0 && mw > 0), "an explicit structuring element replaces the list of diameters");
    k_disc_hist<<<n_pos * n_diam, 256, sizeof(double) * (nb_labels + 1), (cudaStream_t)stream>>>(segm, proba, H, W, positions, diameters, n_diam,
                                                                                           selem, mh, mw, nb_labels, hist, sizes);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Generic (any image, any odd kernels) FP64 versions of two host helpers of imsegm/descriptors.py that the gray-volume
// texture path is built from -- the colour path has its own fused tensor-core kernel (lm_texture.cu):
//   compute_img_filter_response2d :951-966  : max over a battery of ndimage.convolve(img, kernel) (true convolution, 'reflect')
//   image_subtract_gauss_smooth   :986-1000 : per-slice scipy gaussian_filter (rows then columns, symmetric 1-D correlate, 'reflect')
// Plain direct sums in IEEE double in scipy's order; these are utilities, not hot-path kernels.
// ---------------------------------------------------------------------------------------------------------------------
namespace {

// out[s][y][x] = max_f sum_{a,b} K[f][a][b] img[s][reflect(y + kh/2 - a)][reflect(x + kw/2 - b)]
__global__ void __launch_bounds__(256) k_conv_battery_max(const double* __restrict__ img, int S, int H, int W, const double* __restrict__ kern,
                                                          int nf, int kh, int kw, double* __restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)S * H * W) return;
    const int x = (int)(i % W), y = (int)((i / W) % H);
    const double* im = img + (i / ((size_t)H * W)) * (size_t)H * W;
    double best = 0.0;
    for (int f = 0; f < nf; ++f) {
        const double* k = kern + (size_t)f * kh * kw;
        double acc = 0.0;
        // ndimage.convolve == correlate with the flipped kernel: walk the flipped kernel in C order
        for (int a = kh - 1; a >= 0; --a) {
            const int yy = reflect_index(y + kh / 2 - a, H);
            for (int b = kw - 1; b >= 0; --b) acc = __dadd_rn(acc, __dmul_rn(k[a * kw + b], im[(size_t)yy * W + reflect_index(x + kw / 2 - b, W)]));
        }
        // np.max over the battery, which returns NaN when any kernel's response is NaN: the Leung-Malik route feeds this kernel an
        // image minus its background, NaN wherever the image has a NaN or an infinity within the background's reach
        best = (f == 0 || acc > best || isnan(acc)) ? acc : best;
    }
    out[i] = best;
}

// one axis of scipy's gaussian_filter on [S, H, W]: axis 0 = rows (y), 1 = columns (x)
__global__ void __launch_bounds__(256) k_gauss_axis(const double* __restrict__ in, int S, int H, int W, int axis, const double* __restrict__ w_half,
                                                    int r, double* __restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)S * H * W) return;
    const int x = (int)(i % W), y = (int)((i / W) % H);
    const double* im = in + (i / ((size_t)H * W)) * (size_t)H * W;
    double t = __dmul_rn(im[(size_t)y * W + x], w_half[0]);
    for (int j = r; j >= 1; --j) {
        double a, b;
        if (axis == 0) { a = im[(size_t)reflect_index(y - j, H) * W + x]; b = im[(size_t)reflect_index(y + j, H) * W + x]; }
        else { a = im[(size_t)y * W + reflect_index(x - j, W)]; b = im[(size_t)y * W + reflect_index(x + j, W)]; }
        t = __dadd_rn(t, __dmul_rn(__dadd_rn(a, b), w_half[j]));
    }
    out[i] = t;
}

} // namespace

extern "C" int isb_filter_response_2d(const double* img, int n_slices, int H, int W, const double* kernels, int n_kernels, int kh, int kw,
                                      double* out, isb_stream_t stream)
{
    ISB_REQUIRE(img && kernels && out, "null pointer");
    ISB_REQUIRE(n_slices > 0 && H > 0 && W > 0 && n_kernels > 0 && kh > 0 && kw > 0, "bad sizes");
    ISB_REQUIRE((kh & 1) && (kw & 1), "kernels must have odd sizes");
    const size_t n = (size_t)n_slices * H * W;
    k_conv_battery_max<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(img, n_slices, H, W, kernels, n_kernels, kh, kw, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_gaussian_filter_2d(const double* img, int n_slices, int H, int W, const double* w_half, int radius, double* tmp, double* out,
                                      isb_stream_t stream)
{
    ISB_REQUIRE(img && w_half && tmp && out, "null pointer");
    ISB_REQUIRE(n_slices > 0 && H > 0 && W > 0 && radius >= 0, "bad sizes");
    const size_t n = (size_t)n_slices * H * W;
    k_gauss_axis<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(img, n_slices, H, W, 0, w_half, radius, tmp);
    ISB_LAUNCH_CHECK();
    k_gauss_axis<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(tmp, n_slices, H, W, 1, w_half, radius, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
