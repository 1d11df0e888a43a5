/*
 * oracle/stats_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the per-superpixel statistics of the reference's only native module,
 * imsegm/features_cython.pyx:
 *     normColorFeatures            :59-78    count labels, divide where count > 0
 *     computeColorImage2dMean      :81-98    f32 pixels, f64 accumulators, one pass per channel
 *     computeColorImage2dEnergy    :101-119  val*val in f32, accumulated in f64
 *     computeColorImage2dVariance  :122-141  (img - mean_f32)^2 in f32, accumulated in f64
 *     computeGrayImage3dMean/Energy/Variance :144-219  (same, one channel, depth axis)
 *     computeLabelHistogram2d      :222-236
 *     computeRayFeaturesBinary2d   :239-282
 * plus the centroid rule of imsegm/superpixels.py:205-224 (regionprops centroid = mean row / mean col).
 *
 * Pinned against the doctest goldens of imsegm/descriptors.py:218-283 and against the reference's own
 * module compiled unchanged into oracle/_ref (tests/test_oracle_stats.py).
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu legs may use this file.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

/* img: H*W*3 f32 interleaved, seg: H*W i32, nb = max(seg)+1.  mode 0 = mean, 1 = energy, 2 = variance (needs mean f32 nb*3).
 * out: nb*3 f64. */
int oracle_color2d_stat(const float* img, const int32_t* seg, int H, int W, int nb, int mode, const float* mean, double* out)
{
    long npx = (long)H * W;
    int32_t* cnt = (int32_t*)calloc((size_t)nb, sizeof(int32_t));
    if (!cnt) return -1;
    memset(out, 0, sizeof(double) * (size_t)nb * 3);
    for (int z = 0; z < 3; ++z)
        for (long i = 0; i < npx; ++i) {
            int32_t k = seg[i];
            float val = img[3 * i + z];
            if (mode == 0) out[3 * k + z] += val;
            else if (mode == 1) out[3 * k + z] += val * val;
            else { float v = val - mean[3 * k + z]; out[3 * k + z] += v * v; }
        }
    for (long i = 0; i < npx; ++i) cnt[seg[i]] += 1;
    for (int z = 0; z < 3; ++z)
        for (int k = 0; k < nb; ++k)
            if (cnt[k] > 0) out[3 * k + z] = out[3 * k + z] / cnt[k];
    free(cnt);
    return 0;
}

/* img: n voxels f32, seg: n i32; mode as above (mean is nb f32). out: nb f64 */
int oracle_gray3d_stat(const float* img, const int32_t* seg, long n, int nb, int mode, const float* mean, double* out)
{
    int32_t* cnt = (int32_t*)calloc((size_t)nb, sizeof(int32_t));
    if (!cnt) return -1;
    memset(out, 0, sizeof(double) * (size_t)nb);
    for (long i = 0; i < n; ++i) {
        int32_t k = seg[i];
        cnt[k] += 1;
        if (mode == 0) out[k] += img[i];
        else if (mode == 1) out[k] += img[i] * img[i];
        else { float v = img[i] - mean[k]; out[k] += v * v; }
    }
    for (int k = 0; k < nb; ++k)
        if (cnt[k] > 0) out[k] = out[k] / cnt[k];
    free(cnt);
    return 0;
}

/* centroids (row, col) per label; absent labels -> (-1, -1).  out: nb*2 f64, cnt_out optional nb i64 */
int oracle_centroids2d(const int32_t* seg, int H, int W, int nb, double* out, int64_t* cnt_out)
{
    int64_t* acc = (int64_t*)calloc((size_t)nb * 3, sizeof(int64_t));
    if (!acc) return -1;
    for (long y = 0; y < H; ++y)
        for (long x = 0; x < W; ++x) {
            int32_t k = seg[y * W + x];
            acc[3 * k] += 1; acc[3 * k + 1] += y; acc[3 * k + 2] += x;
        }
    for (int k = 0; k < nb; ++k) {
        if (acc[3 * k] == 0) { out[2 * k] = -1; out[2 * k + 1] = -1; }
        else { out[2 * k] = (double)acc[3 * k + 1] / (double)acc[3 * k]; out[2 * k + 1] = (double)acc[3 * k + 2] / (double)acc[3 * k]; }
        if (cnt_out) cnt_out[k] = acc[3 * k];
    }
    free(acc);
    return 0;
}

/* features_cython.pyx:222 */
int oracle_label_hist2d(const int16_t* segm, const int16_t* selem, int H, int W, int nb_labels, uint32_t* hist)
{
    memset(hist, 0, sizeof(uint32_t) * (size_t)nb_labels);
    for (long i = 0; i < (long)H * W; ++i)
        if (segm[i] >= 0 && selem[i] == 1) hist[segm[i]] += 1;
    return 0;
}

/* features_cython.pyx:239.  seg: H*W int8 (0/1), pos = (row, col) in [-H, H) x [-W, W), edge = 1 ('up') or -1 ('down').
 * sin/cos of the angle are supplied by the caller (the reference takes them from numpy in double, then stores to float).
 * The reference indexes its memoryview with wraparound, so a negative start reads row H + pr / column W + pc, while the
 * march itself starts from (pr, pc).  Its round() is Python's builtin on a non-negative value: half to even, i.e. rintf. */
int oracle_ray_features2d(const int8_t* seg, int H, int W, int pr, int pc, const float* sin_a, const float* cos_a, int n_ang, int edge,
                          float* ray_dist)
{
    if (pr < -H || pr >= H || pc < -W || pc >= W) return -1;
    const int8_t start = seg[(long)(pr < 0 ? pr + H : pr) * W + (pc < 0 ? pc + W : pc)];
    for (int i = 0; i < n_ang; ++i) ray_dist[i] = -1.0f;
    if (start && edge == 1) {
        for (int i = 0; i < n_ang; ++i) ray_dist[i] = 0.0f;
        return 0;
    }
    int diag = (int)sqrt((double)W * W + (double)H * H);
    for (int i = 0; i < n_ang; ++i) {
        float pos0 = (float)pr, pos1 = (float)pc;
        float g0 = sin_a[i], g1 = cos_a[i];
        float gmax = fmaxf(fabsf(g0), fabsf(g1));
        g0 /= gmax; g1 /= gmax;
        int8_t last = start;
        for (int s = 0; s < diag; ++s) {
            pos0 += g0; pos1 += g1;
            if (pos0 < 0 || rintf(pos0) >= H || pos1 < 0 || rintf(pos1) >= W) break;
            int8_t actual = seg[(long)((int)rintf(pos0)) * W + (int)rintf(pos1)];
            if ((edge == 1 && actual) || (edge == -1 && last && !actual)) {
                float dx = pos0 - (float)pr, dy = pos1 - (float)pc;
                /* the products and the sum are C floats, np.sqrt then works on the Python float (double), the store rounds to f32 */
                ray_dist[i] = (float)sqrt((double)(dx * dx + dy * dy));
                break;
            }
            last = actual;
        }
    }
    return 0;
}
