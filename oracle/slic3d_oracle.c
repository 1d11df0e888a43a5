/*
 * oracle/slic3d_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of skimage.segmentation.slic for a single-channel VOLUME, as imsegm/superpixels.py:104-106 calls it
 *     slic(np.array(im), n_segments, compactness, multichannel=False, spacing=space, sigma=1)
 * (scikit-image 0.14-0.18, absent from the reference -- requirements.txt:9 -- PARITY UNPINNED, like the 2-D restatement in
 * slic_oracle.c whose arithmetic this file repeats with a depth axis):
 *   1. gaussian pre-blur, sigma / spacing per axis, scipy semantics (symmetric 1-D correlate, mode reflect), axes z, y, x
 *   2. k-means of _slic_cython: window +-2*step per axis about each centre, distance
 *          ((sz (cz - z))^2 + (sy (cy - y))^2 + (sx (cx - x))^2) / step^2 + (v - c)^2,   strict '<' in cluster order,
 *      centres = raster-order sequential sums / count, a cluster without voxels is dead for good
 *   3. _enforce_label_connectivity_cython with its 6 neighbours (dx +-1, dy +-1, dz +-1, in that order)
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu legs may use this file.
 */
#include <float.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static inline int reflect3(int i, int n)
{
    if (n == 1) return 0;
    int p = 2 * n;
    i %= p;
    if (i < 0) i += p;
    return (i < n) ? i : (p - 1 - i);
}

/* one axis of scipy's gaussian_filter on vol[D][H][W]; w[0] centre, w[j] weight at +-j; r == 0: copy */
static void blur_axis(const double* in, double* out, int D, int H, int W, int axis, const double* w, int r)
{
    const int n[3] = { D, H, W };
    const long st[3] = { (long)H * W, W, 1 };
    for (long z = 0; z < D; ++z)
        for (long y = 0; y < H; ++y)
            for (long x = 0; x < W; ++x) {
                const long p = z * st[0] + y * st[1] + x;
                const int c[3] = { (int)z, (int)y, (int)x };
                double t = in[p] * w[0];
                for (int j = r; j >= 1; --j) {
                    const double a = in[p + (long)(reflect3(c[axis] - j, n[axis]) - c[axis]) * st[axis]];
                    const double b = in[p + (long)(reflect3(c[axis] + j, n[axis]) - c[axis]) * st[axis]];
                    t += (a + b) * w[j];
                }
                out[p] = t;
            }
}

/* w_z / w_y / w_x: half kernels (radius + 1 weights) of the three axes; radius 0 with weight 1 = axis not blurred */
int oracle_gaussian_blur3d(const double* vol, int D, int H, int W, const double* w_z, int r_z, const double* w_y, int r_y,
                           const double* w_x, int r_x, double* out)
{
    const size_t n = (size_t)D * H * W;
    double* tmp = (double*)malloc(sizeof(double) * n);
    if (!tmp) return -1;
    blur_axis(vol, out, D, H, W, 0, w_z, r_z);
    blur_axis(out, tmp, D, H, W, 1, w_y, r_y);
    blur_axis(tmp, out, D, H, W, 2, w_x, r_x);
    free(tmp);
    return 0;
}

/* vol: D*H*W doubles already multiplied by 1/compactness.  seeds_zyx [n,3].  labels_out int64.  centroids_out [n,4] optional. */
int oracle_slic_kmeans3d(const double* vol, int D, int H, int W, const double* seeds_zyx, int n_seg, int step_z, int step_y, int step_x,
                         double step, const double* spacing, int max_iter, int64_t* labels_out, double* centroids_out)
{
    const long nvx = (long)D * H * W;
    double* seg = (double*)calloc((size_t)n_seg * 4, sizeof(double));
    double* dist = (double*)malloc(sizeof(double) * (size_t)nvx);
    int64_t* cnt = (int64_t*)calloc((size_t)n_seg, sizeof(int64_t));
    char* dead = (char*)calloc((size_t)n_seg, 1);
    if (!seg || !dist || !cnt || !dead) return -1;
    for (int k = 0; k < n_seg; ++k)
        for (int c = 0; c < 3; ++c) seg[4 * k + c] = seeds_zyx[3 * k + c];
    for (long i = 0; i < nvx; ++i) labels_out[i] = 0;
    const double sz = spacing[0], sy = spacing[1], sx = spacing[2];
    const double spatial_weight = 1.0 / (step * step);
    int it;
    for (it = 0; it < max_iter; ++it) {
        int change = 0;
        for (long i = 0; i < nvx; ++i) dist[i] = DBL_MAX;
        for (int k = 0; k < n_seg; ++k) {
            if (dead[k]) continue;
            const double cz = seg[4 * k], cy = seg[4 * k + 1], cx = seg[4 * k + 2], cv = seg[4 * k + 3];
            double lo, hi;
            lo = cz - 2 * step_z; if (0 > lo) lo = 0;
            hi = cz + 2 * step_z + 1; if (D < hi) hi = D;
            const long z_min = (long)lo, z_max = (long)hi;
            lo = cy - 2 * step_y; if (0 > lo) lo = 0;
            hi = cy + 2 * step_y + 1; if (H < hi) hi = H;
            const long y_min = (long)lo, y_max = (long)hi;
            lo = cx - 2 * step_x; if (0 > lo) lo = 0;
            hi = cx + 2 * step_x + 1; if (W < hi) hi = W;
            const long x_min = (long)lo, x_max = (long)hi;
            for (long z = z_min; z < z_max; ++z) {
                const double tz = sz * (cz - (double)z);
                const double dz = tz * tz;
                for (long y = y_min; y < y_max; ++y) {
                    const double ty = sy * (cy - (double)y);
                    const double dy = ty * ty;
                    for (long x = x_min; x < x_max; ++x) {
                        const double tx = sx * (cx - (double)x);
                        double dc = ((dz + dy) + tx * tx) * spatial_weight;
                        const long p = (z * H + y) * W + x;
                        const double d0 = vol[p] - cv;
                        dc += d0 * d0;
                        if (dist[p] > dc) { labels_out[p] = k; dist[p] = dc; change = 1; }
                    }
                }
            }
        }
        if (!change) break;
        memset(cnt, 0, sizeof(int64_t) * (size_t)n_seg);
        memset(seg, 0, sizeof(double) * (size_t)n_seg * 4);
        for (long z = 0; z < D; ++z)
            for (long y = 0; y < H; ++y)
                for (long x = 0; x < W; ++x) {
                    const long p = (z * H + y) * W + x;
                    const int64_t k = labels_out[p];
                    cnt[k] += 1;
                    seg[4 * k] += (double)z; seg[4 * k + 1] += (double)y; seg[4 * k + 2] += (double)x; seg[4 * k + 3] += vol[p];
                }
        for (int k = 0; k < n_seg; ++k) {
            if (cnt[k] == 0) { dead[k] = 1; continue; }
            for (int c = 0; c < 4; ++c) seg[4 * k + c] /= (double)cnt[k];
        }
    }
    if (centroids_out) memcpy(centroids_out, seg, sizeof(double) * (size_t)n_seg * 4);
    free(seg); free(dist); free(cnt); free(dead);
    return it;
}

int64_t oracle_enforce_connectivity3d(const int64_t* seg, int D, int H, int W, long min_size, long max_size, int64_t* out)
{
    static const int ddx[6] = { 1, -1, 0, 0, 0, 0 };
    static const int ddy[6] = { 0, 0, 1, -1, 0, 0 };
    static const int ddz[6] = { 0, 0, 0, 0, 1, -1 };
    const long nvx = (long)D * H * W;
    if (max_size < 1) max_size = 1;
    long* q = (long*)malloc(sizeof(long) * (size_t)max_size);
    if (!q) return -1;
    for (long i = 0; i < nvx; ++i) out[i] = -1;
    int64_t cur = 0;
    for (long p0 = 0; p0 < nvx; ++p0) {
        if (out[p0] >= 0) continue;
        int64_t adjacent = 0;
        const int64_t label = seg[p0];
        out[p0] = cur;
        long size = 1, visited = 0;
        q[0] = p0;
        while (visited < size && size < max_size) {
            const long v = q[visited];
            const long z = v / ((long)H * W), y = (v / W) % H, x = v % W;
            for (int i = 0; i < 6; ++i) {
                const long zz = z + ddz[i], yy = y + ddy[i], xx = x + ddx[i];
                if (xx >= 0 && xx < W && yy >= 0 && yy < H && zz >= 0 && zz < D) {
                    const long n = (zz * H + yy) * W + xx;
                    if (seg[n] == label && out[n] == -1) {
                        out[n] = cur;
                        q[size] = n;
                        size += 1;
                        if (size >= max_size) break;
                    } else if (out[n] >= 0 && out[n] != cur) {
                        adjacent = out[n];
                    }
                }
            }
            visited += 1;
        }
        if (size < min_size) {
            for (long i = 0; i < size; ++i) out[q[i]] = adjacent;
        } else {
            cur += 1;
        }
    }
    free(q);
    return cur;
}
