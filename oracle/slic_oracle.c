/*
 * oracle/slic_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement (plain C, single thread, IEEE double, no FMA contraction) of the
 * SLIC superpixel algorithm the reference calls at
 *     imsegm/superpixels.py:61-63   ski_segm.slic(img, n_segments, compactness, sigma=1,
 *                                                 enforce_connectivity=True, slic_zero=slico)
 * The arithmetic lives in a third-party dependency that is NOT vendored in the reference and not
 * installed in this image: scikit-image (requirements.txt:9 "scikit-image >= 0.14.0"; effective < 0.19
 * because superpixels.py:105 passes `multichannel=`).  This file restates the published algorithm of
 * skimage.segmentation.slic / _slic_cython / _enforce_label_connectivity_cython for 2-D multichannel
 * images as of 0.14-0.18 (label base 0):
 *   1. Gaussian pre-blur, scipy.ndimage.gaussian_filter semantics (symmetric correlate1d, mode reflect),
 *      axes in order depth(len 1) -> rows -> cols           [pinned bit-exact against scipy in tests]
 *   2. rgb2lab (sRGB companding, XYZ matrix, D65/2deg white, cbrt)  [pinned to 1e-12 against a numpy formula]
 *   3. image * (1/compactness); seeds on a regular grid with colour part 0
 *   4. max_iter cluster-centric k-means sweeps: window +-2*step around the centroid, strict '>' so the
 *      lowest cluster index wins ties; centroid = sequential raster-order double sums / count
 *   5. enforce connectivity: raster-order BFS relabel (neighbour order +x,-x,+y,-y), BFS truncated at
 *      max_size, components < min_size take the label of the last already-labelled neighbour seen.
 *
 * PARITY UNPINNED for label maps: the reference's own tests pin only the output SHAPE of SLIC
 * (superpixels.py:32-40) and the real library cannot be run here.  Two deliberate definitions make the
 * result reproducible bit-for-bit on any IEEE machine (CPU or GPU):
 *   - pow(t, 2.4) and cbrt(t) are computed by det_pow24()/det_cbrt() below: fixed sequences of
 *     + - * on doubles (division-free Newton iterations on the inverse root from an integer-bit seed).
 *     They agree with libm to a few ulp; libm itself differs between platforms at that level.
 *   - the 3x3 colour matrix product is evaluated as (r*m0 + g*m1) + b*m2 without fused multiply-add.
 *   - a cluster that loses all its pixels gets a 0/0 centroid in the original; on x86 the NaN window
 *     bounds cast to INT64_MIN and the cluster is never assigned again.  Here: count==0 => dead forever.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may use this file.
 * Build: see oracle/Makefile (-O2 -ffp-contract=off, no -ffast-math, no -march=native).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>

/* ---------- deterministic math (pure IEEE + - * /) ---------- */

static double det_cbrt(double x) /* x in (0.008, 1.3) */
{
    /* division-free: Newton on y = x^(-1/3)  (y <- y (4 - x y^3) / 3, seed from the exponent bits, 3.4 % off),
     * then cbrt = x y^2 and one correction step c <- c - (c^3 - x) y^2 / 3 */
    union { double d; uint64_t u; } v;
    v.d = x;
    v.u = 0x553EF00000000000ull - v.u / 3u;
    double y = v.d;
    for (int i = 0; i < 4; ++i) {
        double y2 = y * y;
        double y3 = y2 * y;
        double t = x * y3;
        double u = 4.0 - t;
        y = (y * u) * (1.0 / 3.0);
    }
    double y2 = y * y;
    double c = x * y2;
    double c3 = (c * c) * c;
    c = c - ((c3 - x) * y2) * (1.0 / 3.0);
    return c;
}

static double det_root5(double x) /* x in (0.05, 1.1) */
{
    /* division-free: Newton on y = x^(-1/5)  (y <- y (6 - x y^5) / 5), then x^(1/5) = x y^4 and one correction step */
    union { double d; uint64_t u; } v;
    v.d = x;
    v.u = 0x4CB8A99999999800ull - v.u / 5u;
    double y = v.d;
    for (int i = 0; i < 4; ++i) {
        double y2 = y * y;
        double y4 = y2 * y2;
        double y5 = y4 * y;
        double t = x * y5;
        double u = 6.0 - t;
        y = (y * u) * 0.2;
    }
    double y2 = y * y;
    double y4 = y2 * y2;
    double r = x * y4;
    double r2 = r * r;
    double r5 = (r2 * r2) * r;
    r = r - ((r5 - x) * y4) * 0.2;
    return r;
}

static double det_pow24(double t) /* t^2.4 = t^2 * (t^(1/5))^2 */
{
    double r = det_root5(t);
    return (t * t) * (r * r);
}

double oracle_det_cbrt(double x) { return det_cbrt(x); }
double oracle_det_pow24(double x) { return det_pow24(x); }

/* ---------- 1. gaussian blur (scipy.ndimage.gaussian_filter restatement) ---------- */

static inline int reflect_idx(int i, int n)
{
    /* scipy mode='reflect': (d c b a | a b c d | d c b a); period 2n */
    if (n == 1) return 0;
    int p = 2 * n;
    i %= p;
    if (i < 0) i += p;
    return (i < n) ? i : (p - 1 - i);
}

/* one symmetric correlate1d along a line of `n` samples with stride `st` (in doubles).
 * scipy's symmetric branch: tmp = x[l]*w[0]; for j = r..1: tmp += (x[l-j] + x[l+j]) * w[-j]
 * `w` points at the centre weight, w[-j] == w[j]. */
static void blur_line(const double* in, double* out, int n, long st, const double* w, int r, double* buf)
{
    for (int i = -r; i < n + r; ++i) buf[i + r] = in[(long)reflect_idx(i, n) * st];
    for (int l = 0; l < n; ++l) {
        const double* c = buf + r + l;
        double tmp = c[0] * w[0];
        for (int j = r; j >= 1; --j) tmp += (c[-j] + c[j]) * w[j];
        out[(long)l * st] = tmp;
    }
}

/* img: H*W*C interleaved doubles.  w_half: r+1 weights, w_half[0] = centre, w_half[j] = weight at +-j.
 * Applies the length-1 depth axis first (as skimage's [1,H,W,C] array sees it), then rows, then cols. */
int oracle_gaussian_blur(const double* img, int H, int W, int C, const double* w_half, int r, double* out)
{
    long n = (long)H * W * C;
    double* tmp = (double*)malloc(sizeof(double) * (size_t)n);
    int maxn = (H > W ? H : W) + 2 * r + 2;
    double* buf = (double*)malloc(sizeof(double) * (size_t)maxn);
    if (!tmp || !buf) { free(tmp); free(buf); return -1; }
    /* axis 0 (depth, length 1): every tap reflects onto the same sample */
    for (long i = 0; i < n; ++i) {
        double x = img[i];
        double t = x * w_half[0];
        for (int j = r; j >= 1; --j) t += (x + x) * w_half[j];
        tmp[i] = t;
    }
    /* axis 1 (rows): lines along y for each (x, c) */
    for (int x = 0; x < W; ++x)
        for (int c = 0; c < C; ++c)
            blur_line(tmp + (long)x * C + c, out + (long)x * C + c, H, (long)W * C, w_half, r, buf);
    /* axis 2 (cols): lines along x for each (y, c) */
    for (int y = 0; y < H; ++y)
        for (int c = 0; c < C; ++c)
            blur_line(out + (long)y * W * C + c, tmp + (long)y * W * C + c, W, (long)C, w_half, r, buf);
    memcpy(out, tmp, sizeof(double) * (size_t)n);
    free(tmp);
    free(buf);
    return 0;
}

/* ---------- 2. rgb2lab ---------- */

void oracle_rgb2lab_px(double r, double g, double b, double* L, double* A, double* B)
{
    double c[3] = { r, g, b };
    for (int i = 0; i < 3; ++i) {
        if (c[i] > 0.04045) c[i] = det_pow24((c[i] + 0.055) / 1.055);
        else c[i] = c[i] / 12.92;
    }
    double X = (c[0] * 0.412453 + c[1] * 0.357580) + c[2] * 0.180423;
    double Y = (c[0] * 0.212671 + c[1] * 0.715160) + c[2] * 0.072169;
    double Z = (c[0] * 0.019334 + c[1] * 0.119193) + c[2] * 0.950227;
    double f[3] = { X / 0.95047, Y / 1.0, Z / 1.08883 };
    for (int i = 0; i < 3; ++i) {
        if (f[i] > 0.008856) f[i] = det_cbrt(f[i]);
        else f[i] = 7.787 * f[i] + 16.0 / 116.0;
    }
    *L = 116.0 * f[1] - 16.0;
    *A = 500.0 * (f[0] - f[1]);
    *B = 200.0 * (f[1] - f[2]);
}

/* img,out: H*W*3 interleaved; out = rgb2lab(img) * ratio */
void oracle_rgb2lab_scaled(const double* img, long npx, double ratio, double* out)
{
    for (long i = 0; i < npx; ++i) {
        double L, A, B;
        oracle_rgb2lab_px(img[3 * i], img[3 * i + 1], img[3 * i + 2], &L, &A, &B);
        out[3 * i] = L * ratio;
        out[3 * i + 1] = A * ratio;
        out[3 * i + 2] = B * ratio;
    }
}

/* ---------- 3/4. k-means sweeps (restates skimage _slic_cython, depth == 1) ---------- */

/* lab: H*W*3 interleaved, already multiplied by 1/compactness.
 * seeds_yx: n_seg * 2 doubles (row, col) -- the regular grid, colour part starts at 0.
 * step_y, step_x: integer grid steps (window half-size is 2*step); step = max of the steps (spatial weight).
 * labels_out: H*W int64.  centroids_out (optional): n_seg*5 (y, x, L, a, b) after the last update.
 * Returns number of sweeps executed. */
int oracle_slic_kmeans(const double* lab, int H, int W, const double* seeds_yx, int n_seg, int step_y, int step_x,
                       double step, int max_iter, int slic_zero, int64_t* labels_out, double* centroids_out)
{
    long npx = (long)H * W;
    double* seg = (double*)calloc((size_t)n_seg * 5, sizeof(double));
    double* dist = (double*)malloc(sizeof(double) * (size_t)npx);
    int64_t* cnt = (int64_t*)calloc((size_t)n_seg, sizeof(int64_t));
    char* dead = (char*)calloc((size_t)n_seg, 1);
    double* maxdc = (double*)malloc(sizeof(double) * (size_t)n_seg);
    if (!seg || !dist || !cnt || !dead || !maxdc) return -1;
    for (int k = 0; k < n_seg; ++k) {
        seg[5 * k] = seeds_yx[2 * k];
        seg[5 * k + 1] = seeds_yx[2 * k + 1];
        maxdc[k] = 1.0;
    }
    for (long i = 0; i < npx; ++i) labels_out[i] = 0; /* np.empty in the original; every pixel is covered */
    const double spatial_weight = 1.0 / (step * step);
    int it;
    for (it = 0; it < max_iter; ++it) {
        int change = 0;
        for (long i = 0; i < npx; ++i) dist[i] = DBL_MAX;
        for (int k = 0; k < n_seg; ++k) {
            if (dead[k]) continue;
            const double cy = seg[5 * k], cx = seg[5 * k + 1];
            const double c0 = seg[5 * k + 2], c1 = seg[5 * k + 3], c2 = seg[5 * k + 4];
            double lo, hi;
            lo = cy - 2 * step_y; if (0 > lo) lo = 0;
            hi = cy + 2 * step_y + 1; if (H < hi) hi = H;
            long y_min = (long)lo, y_max = (long)hi;
            lo = cx - 2 * step_x; if (0 > lo) lo = 0;
            hi = cx + 2 * step_x + 1; if (W < hi) hi = W;
            long x_min = (long)lo, x_max = (long)hi;
            for (long y = y_min; y < y_max; ++y) {
                double ty = cy - (double)y;
                double dy = ty * ty;
                for (long x = x_min; x < x_max; ++x) {
                    double tx = cx - (double)x;
                    double dc = (dy + tx * tx) * spatial_weight; /* dz == 0: (0 + dy) + dx^2 */
                    const double* p = lab + 3 * (y * W + x);
                    double d0 = p[0] - c0, d1 = p[1] - c1, d2 = p[2] - c2;
                    double dcol = d0 * d0;
                    dcol += d1 * d1;
                    dcol += d2 * d2;
                    if (slic_zero) dc += dcol / maxdc[k];
                    else dc += dcol;
                    if (dist[y * W + x] > dc) {
                        labels_out[y * W + x] = k;
                        dist[y * W + x] = dc;
                        change = 1;
                    }
                }
            }
        }
        if (!change) break;
        /* recompute centres: sequential raster-order sums */
        memset(cnt, 0, sizeof(int64_t) * (size_t)n_seg);
        memset(seg, 0, sizeof(double) * (size_t)n_seg * 5);
        for (long y = 0; y < H; ++y)
            for (long x = 0; x < W; ++x) {
                int64_t k = labels_out[y * W + x];
                const double* p = lab + 3 * (y * W + x);
                cnt[k] += 1;
                seg[5 * k] += (double)y;
                seg[5 * k + 1] += (double)x;
                seg[5 * k + 2] += p[0];
                seg[5 * k + 3] += p[1];
                seg[5 * k + 4] += p[2];
            }
        for (int k = 0; k < n_seg; ++k) {
            if (cnt[k] == 0) { dead[k] = 1; continue; }
            for (int c = 0; c < 5; ++c) seg[5 * k + c] /= (double)cnt[k];
        }
        if (slic_zero) {
            for (long i = 0; i < npx; ++i) {
                int64_t k = labels_out[i];
                const double* p = lab + 3 * i;
                double d0 = p[0] - seg[5 * k + 2], d1 = p[1] - seg[5 * k + 3], d2 = p[2] - seg[5 * k + 4];
                double dcol = d0 * d0;
                dcol += d1 * d1;
                dcol += d2 * d2;
                if (maxdc[k] < dcol) maxdc[k] = dcol;
            }
        }
    }
    if (centroids_out) memcpy(centroids_out, seg, sizeof(double) * (size_t)n_seg * 5);
    free(seg); free(dist); free(cnt); free(dead); free(maxdc);
    return it;
}

/* ---------- 5. enforce connectivity (restates skimage _enforce_label_connectivity_cython, depth == 1) ---------- */

int64_t oracle_enforce_connectivity(const int64_t* seg, int H, int W, long min_size, long max_size, int64_t* out)
{
    static const int ddx[4] = { 1, -1, 0, 0 };
    static const int ddy[4] = { 0, 0, 1, -1 };
    long npx = (long)H * W;
    if (max_size < 1) max_size = 1;
    long* qy = (long*)malloc(sizeof(long) * (size_t)max_size);
    long* qx = (long*)malloc(sizeof(long) * (size_t)max_size);
    if (!qy || !qx) return -1;
    for (long i = 0; i < npx; ++i) out[i] = -1;
    int64_t cur = 0;
    for (long y = 0; y < H; ++y)
        for (long x = 0; x < W; ++x) {
            if (out[y * W + x] >= 0) continue;
            int64_t adjacent = 0;
            int64_t label = seg[y * W + x];
            out[y * W + x] = cur;
            long size = 1, visited = 0;
            qy[0] = y; qx[0] = x;
            while (visited < size && size < max_size) {
                for (int i = 0; i < 4; ++i) {
                    long yy = qy[visited] + ddy[i], xx = qx[visited] + ddx[i];
                    if (xx >= 0 && xx < W && yy >= 0 && yy < H) {
                        long q = yy * W + xx;
                        if (seg[q] == label && out[q] == -1) {
                            out[q] = cur;
                            qy[size] = yy; qx[size] = xx;
                            size += 1;
                            if (size >= max_size) break;
                        } else if (out[q] >= 0 && out[q] != cur) {
                            adjacent = out[q];
                        }
                    }
                }
                visited += 1;
            }
            if (size < min_size) {
                for (long i = 0; i < size; ++i) out[qy[i] * W + qx[i]] = adjacent;
            } else {
                cur += 1;
            }
        }
    free(qy); free(qx);
    return cur;
}
