// slic_kmeans.cu -- the k-means sweeps of SLIC, pixel-centric and bit-exact with oracle/slic_oracle.c.
//
// Replaces skimage.segmentation._slic._slic_cython as called through imsegm/superpixels.py:61-63.
//
// The original is cluster-centric: for k ascending, scan the +-2*step window and take the pixel when
// `distance > d` (strict) -- i.e. every pixel ends with argmin over {clusters whose window holds it} of
// (d, k) in lexicographic order.  That per-pixel minimum is order-independent, so it is evaluated here
// pixel-centric: one CTA per 32x32 pixel tile gathers the clusters whose integer window intersects the tile
// (from a uniform bin grid over the current centroids), every pixel loops over that list in shared memory.
// The distance is computed with the oracle's exact operation order in IEEE double (no FMA).
//
// The centroid update of the original is a raster-order SEQUENTIAL double sum per cluster; a tree/atomic
// reduction changes the last ulp and flips exact ties (flat image regions tie all the time).  It is
// reproduced exactly: one warp per cluster walks the cluster's window in raster order, ballots the member
// pixels of each 32-wide chunk, compacts their colours into shared memory in lane (= raster) order, and three
// lanes add them one at a time.  Coordinate sums are integers (exact in any order).
//
// Per sweep HBM traffic (algorithmic): read Lab 24 B/px + write label 4 B/px (assign); the update re-reads
// labels and member colours through L2.
#include "common.cuh"
#include "wgmma.cuh"
#include <float.h>
#include <string.h>

namespace {

constexpr int TILE = 32;   // pixel tile edge of the assignment kernel
constexpr int ACAP = 128;  // candidate clusters staged per round
constexpr int AROWS = 8;   // consecutive rows per thread (same column)
constexpr int AWARPS = TILE / AROWS;      // 4 warps
constexpr int ATHREADS = 32 * AWARPS;     // 128 threads per tile


struct __align__(16) Cand {
    double cy, cx, c0, c1, c2;
    int y0, y1, x0, x1;
    int k, pad;
};
static_assert(sizeof(Cand) == 64, "Cand must be 64 bytes");

struct KmState {
    // cluster state (SoA)
    double* cy; double* cx; double* c0; double* c1; double* c2;
    int4* win;       // [n] (y0, y1, x0, x1); empty (0,0,0,0) when dead
    int4* obb;       // [n] bbox of the cluster's member pixels (ymin, ymax, xmin, xmax), empty = (INT_MAX, -1, INT_MAX, -1)
    int* bin_start;  // [nbins + 1]
    int* bin_fill;   // [nbins]
    int* bin_of;     // [n]
    int* pack_done;  // [1] CTA counter of k_pack
    Cand* packed;    // [n] cluster records in bin order (what k_assign streams)
    double* packed_maxdc; // [n] SLICO: the maxima in bin order, beside `packed`
    unsigned long long* maxdc; // [n] SLICO colour-distance maxima as raw double bits (non-negative doubles order like their bits)
    int slico;
    int n, H, W, step_y, step_x, B, nby, nbx;
    double sw;       // spatial weight 1/step^2
    // Row-band mode (one band of a taller image per GPU, isb_slic_band_*): pixel memory is a slab of H rows whose row 0 is
    // global row y_off of an image Hg rows tall; cluster geometry (centres, windows, bins) is always global.  The
    // monolithic path is the band [0, H) of itself: y_off = 0, Hg = H, pstride = H * W.
    int Hg, y_off, own_lo, own_hi, halo;
    size_t pstride;  // distance between the Lab planes, in doubles
};

__device__ __forceinline__ int4 make_window(double cy, double cx, int step_y, int step_x, int H, int W)
{
    // <Py_ssize_t>max(c - 2*step, 0) / <Py_ssize_t>min(c + 2*step + 1, size): truncation of a non-negative double
    double lo, hi;
    int4 w;
    lo = __dsub_rn(cy, (double)(2 * step_y)); if (0.0 > lo) lo = 0.0;
    hi = __dadd_rn(__dadd_rn(cy, (double)(2 * step_y)), 1.0); if ((double)H < hi) hi = (double)H;
    w.x = (int)lo; w.y = (int)hi;
    lo = __dsub_rn(cx, (double)(2 * step_x)); if (0.0 > lo) lo = 0.0;
    hi = __dadd_rn(__dadd_rn(cx, (double)(2 * step_x)), 1.0); if ((double)W < hi) hi = (double)W;
    w.z = (int)lo; w.w = (int)hi;
    return w;
}

// Between two sweeps the clusters are re-binned in three small launches:
//   k_seed (first sweep only) or k_update / k_import : centres, windows, bin_of, and a count per bin in bin_fill
//   k_scan_bins (one CTA)  : exclusive scan of the counts -> bin_start; the counts are zeroed (they become the fill cursors)
//   k_pack (many CTAs)     : the packed, bin-ordered cluster records that k_assign streams; order inside a bin is irrelevant
//   (k_assign leaves bin_fill alone; k_update / k_import need it zero again, k_pack's last CTA does that)
__global__ void k_seed(KmState s, const double* __restrict__ seeds_yx)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= s.n) return;
    const double cy = seeds_yx[2 * k], cx = seeds_yx[2 * k + 1];
    s.cy[k] = cy; s.cx[k] = cx; s.c0[k] = 0.0; s.c1[k] = 0.0; s.c2[k] = 0.0;
    s.win[k] = make_window(cy, cx, s.step_y, s.step_x, s.Hg, s.W);
    const int by = min(max((int)cy / s.B, 0), s.nby - 1), bx = min(max((int)cx / s.B, 0), s.nbx - 1);
    s.bin_of[k] = by * s.nbx + bx;
    atomicAdd(&s.bin_fill[by * s.nbx + bx], 1);
    s.obb[k] = make_int4(INT_MAX, -1, INT_MAX, -1);
    s.maxdc[k] = (unsigned long long)__double_as_longlong(1.0);
}

__global__ void __launch_bounds__(1024) k_scan_bins(KmState s)
{
    const int nbins = s.nby * s.nbx;
    // exclusive scan of bin counts: warp shuffles + one partial per warp, chunks of blockDim
    __shared__ int s_wsum[32];
    __shared__ int s_part_total;
    __shared__ int s_carry;
    if (threadIdx.x == 0) { s_carry = 0; *s.pack_done = 0; }
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int base = 0; base < nbins; base += blockDim.x) {
        int b = base + threadIdx.x;
        int v = b < nbins ? s.bin_fill[b] : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        if (lane == 31) s_wsum[wid] = incl;
        __syncthreads();
        if (wid == 0) {
            int t = lane < nw ? s_wsum[lane] : 0, ti = t;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, ti, o); if (lane >= o) ti += u; }
            s_wsum[lane] = ti - t; // exclusive prefix of the warp sums
            if (lane == 31) s_part_total = ti;
        }
        __syncthreads();
        const int carry = s_carry;
        if (b < nbins) { s.bin_start[b] = carry + s_wsum[wid] + incl - v; s.bin_fill[b] = 0; }
        __syncthreads();
        if (threadIdx.x == 0) s_carry = carry + s_part_total;
        __syncthreads();
    }
    if (threadIdx.x == 0) s.bin_start[nbins] = s_carry;
}

__global__ void __launch_bounds__(256) k_pack(KmState s)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < s.n) {
        const int bin = s.bin_of[k];
        if (bin >= 0) {
            const int pos = s.bin_start[bin] + atomicAdd(&s.bin_fill[bin], 1);
            const int4 w = s.win[k];
            Cand c;
            c.cy = s.cy[k]; c.cx = s.cx[k]; c.c0 = s.c0[k]; c.c1 = s.c1[k]; c.c2 = s.c2[k];
            c.y0 = w.x; c.y1 = w.y; c.x0 = w.z; c.x1 = w.w; c.k = k; c.pad = 0;
            s.packed[pos] = c;
            if (s.slico) s.packed_maxdc[pos] = __longlong_as_double((long long)s.maxdc[k]);
        }
    }
    // the last CTA to finish zeroes the fill cursors: k_update / k_import count the next sweep's bins from zero
    __shared__ int s_last;
    __syncthreads();
    if (threadIdx.x == 0) { __threadfence(); s_last = atomicAdd(s.pack_done, 1) == (int)gridDim.x - 1; }
    __syncthreads();
    if (s_last) {
        const int nbins = s.nby * s.nbx;
        for (int b = threadIdx.x; b < nbins; b += blockDim.x) s.bin_fill[b] = 0;
    }
}

// non-negative doubles order like their bit patterns: compare on the integer pipe instead of the FP64 pipe
// (unsigned, so that a NaN of either sign ranks above every number and can never win)
__device__ __forceinline__ unsigned long long dbits(double v) { return (unsigned long long)__double_as_longlong(v); }

// assignment: one CTA (128 threads) per 32x32 tile; a thread owns one column and AROWS = 8 consecutive rows.
// The tile's Lab values are staged in shared memory, candidates are visited nearest-first and the loop stops as soon as
// the spatial lower bound of every remaining candidate exceeds the worst of the thread's current minima.
template <bool SLICO>
__global__ void __launch_bounds__(ATHREADS, 5) k_assign(const __grid_constant__ CUtensorMap lab_map, int use_tma, KmState s,
                                                        const double* __restrict__ lab, int* __restrict__ labels)
{
    __shared__ Cand cand[ACAP];
    __shared__ double s_maxdc[SLICO ? ACAP : 1];
    __shared__ float s_key[ACAP];
    __shared__ float2 s_cf[ACAP];         // (cy, cx) of the candidate as floats, for the per-thread spatial lower bound
    __shared__ double s_lb[ACAP];          // lower bound of the spatial term of the candidate at sorted position i, and of all later ones
    __shared__ unsigned char s_order[ACAP];
    __shared__ __align__(128) double s_px[3][TILE][TILE]; // Lab of the tile
    __shared__ __align__(8) unsigned long long s_bar;     // mbarrier of the TMA tile load
    __shared__ int s_ncand, s_done, s_row, s_off, s_total;
    const int tx0 = blockIdx.x * TILE, ty0 = blockIdx.y * TILE;
    const int tx1 = min(tx0 + TILE, s.W);
    const int gy0 = ty0 + s.y_off, gy1 = min(ty0 + TILE, s.H) + s.y_off; // the tile's rows in global coordinates
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t HW = s.pstride;
    const int x = tx0 + lane;
    const bool xin = x < s.W;
    const int yb = ty0 + warp * AROWS; // first row of this thread

    double best[AROWS];
    int bestk[AROWS];
#pragma unroll
    for (int j = 0; j < AROWS; ++j) { best[j] = DBL_MAX; bestk[j] = -1; }
    if (use_tma) {
        // the three Lab planes of the tile arrive as ONE 3-D tensor-map load (32 x 32 x 3 doubles, out-of-image elements read as 0)
        // while every warp gathers the candidate clusters; the distance loop waits on the mbarrier
        if (threadIdx.x == 0) {
            wgmma::mbar_init(wgmma::smem_u32(&s_bar), 1);
            wgmma::fence_mbar_init();
            wgmma::mbar_arrive_expect_tx(wgmma::smem_u32(&s_bar), 3 * TILE * TILE * 8);
            wgmma::tma_load_3d(wgmma::smem_u32(&s_px[0][0][0]), &lab_map, tx0, ty0, 0, wgmma::smem_u32(&s_bar));
        }
    } else {
        double v[3][AROWS];
#pragma unroll
        for (int j = 0; j < AROWS; ++j) {
            const int y = yb + j;
            if (xin && y < s.H) {
                const size_t p = (size_t)y * s.W + x;
                v[0][j] = lab[p]; v[1][j] = lab[HW + p]; v[2][j] = lab[2 * HW + p];
            } else { v[0][j] = v[1][j] = v[2][j] = 0.0; }
        }
#pragma unroll
        for (int j = 0; j < AROWS; ++j) {
            s_px[0][warp * AROWS + j][lane] = v[0][j]; s_px[1][warp * AROWS + j][lane] = v[1][j]; s_px[2][warp * AROWS + j][lane] = v[2][j];
        }
    }
    // bins that can hold a centroid whose window reaches this tile (superset; the exact window test follows)
    const int by0 = max(gy0 - 2 * s.step_y - 2, 0) / s.B, by1 = min(gy1 + 2 * s.step_y + 1, s.Hg - 1) / s.B;
    const int bx0 = max(tx0 - 2 * s.step_x - 2, 0) / s.B, bx1 = min(tx1 + 2 * s.step_x + 1, s.W - 1) / s.B;
    const float tcy = 0.5f * (gy0 + gy1 - 1), tcx = 0.5f * (tx0 + tx1 - 1);
    const int byl = min(by1, s.nby - 1), bxl = min(bx1, s.nbx - 1);
    // how many clusters sit in the bin rows that can reach this tile (bins of one row are contiguous in bin order)
    if (threadIdx.x == 0) { s_row = by0; s_off = 0; s_done = 0; s_ncand = 0; s_total = 0; }
    __syncthreads();
    if (warp == 0) {
        int t = 0;
        for (int row = by0 + lane; row <= byl; row += 32) t += s.bin_start[row * s.nbx + bxl + 1] - s.bin_start[row * s.nbx + bx0];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (lane == 0) s_total = t;
    }
    __syncthreads();
    const bool fast = s_total <= ACAP; // everything fits in one round: all warps build the list together

    while (true) {
        if (fast) {
            for (int row = by0 + warp; row <= byl; row += AWARPS) {
                const int beg = s.bin_start[row * s.nbx + bx0], end = s.bin_start[row * s.nbx + bxl + 1];
                for (int i = beg + lane; i < end; i += 32) {
                    const Cand c = s.packed[i];
                    if ((c.y0 < gy1) && (c.y1 > gy0) && (c.x0 < tx1) && (c.x1 > tx0)) {
                        const int pos = atomicAdd(&s_ncand, 1);
                        cand[pos] = c;
                        if (SLICO) s_maxdc[pos] = s.packed_maxdc[i];
                        const float fy = (float)c.cy - tcy, fx = (float)c.cx - tcx;
                        s_key[pos] = fy * fy + fx * fx;
                        s_cf[pos] = make_float2((float)c.cy, (float)c.cx);
                    }
                }
            }
            if (threadIdx.x == 0) s_done = 1;
        } else if (warp == 0) {
            // deterministic, resumable scan of the bin rows: fill up to ACAP candidates per round
            int n = 0;
            int row = s_row, off = s_off;
            while (row <= byl && n < ACAP) {
                int beg = s.bin_start[row * s.nbx + bx0] + off;
                int end = s.bin_start[row * s.nbx + bxl + 1];
                while (beg < end && n < ACAP) {
                    int room = ACAP - n;
                    int i = beg + lane;
                    bool ok = false;
                    Cand c;
                    if (i < end && lane < room) {
                        c = s.packed[i];
                        ok = (c.y0 < gy1) && (c.y1 > gy0) && (c.x0 < tx1) && (c.x1 > tx0);
                    }
                    unsigned m = __ballot_sync(0xffffffffu, ok);
                    if (ok) {
                        int pos = n + __popc(m & ((1u << lane) - 1u));
                        cand[pos] = c;
                        if (SLICO) s_maxdc[pos] = s.packed_maxdc[i];
                        const float fy = (float)c.cy - tcy, fx = (float)c.cx - tcx;
                        s_key[pos] = fy * fy + fx * fx;
                        s_cf[pos] = make_float2((float)c.cy, (float)c.cx);
                    }
                    n += __popc(m);
                    int adv = min(min(32, room), end - beg);
                    beg += adv; off += adv;
                }
                if (beg >= end) { ++row; off = 0; }
            }
            if (lane == 0) { s_ncand = n; s_row = row; s_off = off; s_done = row > byl; }
        }
        __syncthreads();
        const int nc = s_ncand;
        const int done = s_done;
        // nearest-first evaluation order (rank sort by distance of the centroid to the tile centre).  Any order gives the
        // same result -- the minimum over (distance, index) is order independent.
        for (int t = threadIdx.x; t < nc; t += ATHREADS) {
            const float key = s_key[t];
            int rank = 0;
            for (int j = 0; j < nc; ++j) {
                const float kj = s_key[j];
                rank += (kj < key) || (kj == key && j < t);
            }
            s_order[rank] = (unsigned char)t;
            // every pixel of the tile is within R of the tile centre, so a centroid at distance sqrt(key) from the centre is at
            // least sqrt(key) - R from the pixel; the bound is relaxed (R rounded up, 0.1 % slack) so that float rounding can
            // only make it smaller, i.e. it never rejects a candidate that could win or tie
            const float r = sqrtf(key) - 23.5f;
            s_lb[rank] = r > 0.f ? (double)(r * r * 0.999f) * s.sw * 0.999 : 0.0;
        }
        __syncthreads();
        if (use_tma) wgmma::mbar_wait(wgmma::smem_u32(&s_bar), 0);   // phase 0 completes once; later rounds pass immediately
        if (xin) {
            const double xd = (double)x;
            // this thread's pixels: column x, AROWS consecutive rows: the float form of the column and the centre of the run
            const float xf = (float)x, ymid = (float)(yb + s.y_off) + 0.5f * (AROWS - 1), swf = (float)s.sw * 0.998f;
            unsigned long long worst = dbits(DBL_MAX); // max over the rows of the current minima (bit pattern)
#pragma unroll
            for (int j = 0; j < AROWS; ++j) worst = max(worst, dbits(best[j]));
            float worstf = __double2float_ru(__longlong_as_double((long long)worst));
            for (int ci = 0; ci < nc; ++ci) {
                if (dbits(s_lb[ci]) > worst) break; // sorted by key: nobody further down the list can win either
                const int c = s_order[ci];
                {
                    // spatial lower bound of this candidate for ALL of the thread's pixels, in float: the centre is at least
                    // |cx - x| away in x and |cy - ymid| - (AROWS-1)/2 in y.  2e-3 px absorbs the float conversion of coordinates
                    // up to 16k, the factor 0.998 the rounding of the few float operations: the bound can only come out smaller
                    // than the exact double distance term, so it never rejects a candidate that could win or tie
                    const float2 cf = s_cf[c];
                    const float ax = fmaxf(fabsf(cf.y - xf) - 2e-3f, 0.f), ay = fmaxf(fabsf(cf.x - ymid) - (0.5f * (AROWS - 1) + 2e-3f), 0.f);
                    if ((ax * ax + ay * ay) * swf > worstf) continue;
                }
                const int cx0 = cand[c].x0, cx1 = cand[c].x1;
                if (x < cx0 || x >= cx1) continue;
                const int cy0 = cand[c].y0, ck = cand[c].k;
                const unsigned cyn = (unsigned)(cand[c].y1 - cy0);   // rows [cy0, cy0 + cyn) are inside the window
                const double ccy = cand[c].cy;
                const double tx = __dsub_rn(cand[c].cx, xd);
                const double dx2 = __dmul_rn(tx, tx);
                bool improved = false;
                // four rows at a time, straight-line code: the four spatial terms are independent chains (the FP64 latency of one
                // hides behind the others), then -- only if one of the four can still win -- the four colour terms likewise
#pragma unroll
                for (int jg = 0; jg < AROWS; jg += 4) {
                    double sp[4];
                    bool need[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int y = yb + jg + q + s.y_off;
                        // (double)y without the conversion unit: y < 2^31 sits in the low mantissa word of 2^52 + y (exact)
                        const double yd = __dsub_rn(__hiloint2double(0x43300000, y), 4503599627370496.0);
                        const double ty = __dsub_rn(ccy, yd);
                        sp[q] = __dmul_rn(__dadd_rn(__dmul_rn(ty, ty), dx2), s.sw);
                        // inside the window, and exact pruning: the colour term is >= 0 and fl(a + b) >= a for b >= 0, so
                        // d >= sp > best cannot win or tie (a NaN sp falls through: its NaN distance never compares less)
                        need[q] = (unsigned)(y - cy0) < cyn && !(sp[q] > best[jg + q]);
                    }
                    if (!(need[0] | need[1] | need[2] | need[3])) continue;
                    double dc[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int ry = warp * AROWS + jg + q;
                        const double d0 = __dsub_rn(s_px[0][ry][lane], cand[c].c0), d1 = __dsub_rn(s_px[1][ry][lane], cand[c].c1),
                                     d2 = __dsub_rn(s_px[2][ry][lane], cand[c].c2);
                        double dcol = __dmul_rn(d0, d0);
                        dcol = __dadd_rn(dcol, __dmul_rn(d1, d1));
                        dcol = __dadd_rn(dcol, __dmul_rn(d2, d2));
                        dc[q] = __dadd_rn(sp[q], SLICO ? __ddiv_rn(dcol, s_maxdc[c]) : dcol);
                    }
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int j = jg + q;
                        // distances are >= +0 or NaN: the floating-point order is the order of the bit patterns, a NaN never wins
                        if (need[q] && (dc[q] < best[j] || (dc[q] == best[j] && bestk[j] >= 0 && ck < bestk[j]))) {
                            best[j] = dc[q]; bestk[j] = ck; improved = true;
                        }
                    }
                }
                if (improved) {
                    worst = 0;
#pragma unroll
                    for (int j = 0; j < AROWS; ++j) if (yb + j < s.H) worst = max(worst, dbits(best[j]));
                    worstf = __double2float_ru(__longlong_as_double((long long)worst));
                }
            }
        }
        if (done) break;
        __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < AROWS; ++j) {
        const int y = yb + j;
        const bool in = xin && y < s.H;     // y is warp-uniform
        int k = -1;
        if (in) {
            const size_t p = (size_t)y * s.W + x;
            if (bestk[j] >= 0) { k = bestk[j]; labels[p] = k; }
            else k = labels[p];             // no window holds this pixel: it keeps its label (the original leaves it untouched)
        }
        // bounding box of every cluster's members (orphans included): one leader per (warp row, label) updates it
        const unsigned act = __ballot_sync(0xffffffffu, in);
        if (in) {
            const unsigned grp = __match_any_sync(act, k);
            if (lane == __ffs(grp) - 1) {
                const int xa = tx0 + __ffs(grp) - 1, xb = tx0 + 31 - __clz(grp);
                atomicMin(&s.obb[k].x, y); atomicMax(&s.obb[k].y, y);
                atomicMin(&s.obb[k].z, xa); atomicMax(&s.obb[k].w, xb);
            }
        }
    }
}

// centroid sums: one warp per cluster, raster-order sequential double adds (see header).
// BAND: this GPU holds a row band of the image.  A cluster is summed by the band that owns the row of its centre (every
// member lies within 2*step rows of the centre the assignment used, i.e. inside that band's slab -- checked, violations are
// counted in xchg[6n]); the result goes to the exchange record xchg[6k..6k+5] = bits(cy, cx, c0, c1, c2), state (1 alive,
// 2 died) and every other band leaves zeros there, so that an integer sum over the bands is an exact merge.
// A warp's time is the length of its cluster's dependent chain, so the launch should be ONE wave: UWARPS warps per CTA and UBLOCKS CTAs
// per SM give 132 x UWARPS x UBLOCKS resident warps on an H100 -- with 2 x 19 that is 5 016, enough for the ~5 000 clusters of a
// 2048 x 2048 image at sp_size 29 (a second wave for the last few percent costs as much as the first).  The 48 registers this allows
// spill a few words.
constexpr int UWARPS = 2, UBLOCKS = 19;
template <bool BAND>
__global__ void __launch_bounds__(32 * UWARPS, UBLOCKS) k_update(KmState s, const double* __restrict__ lab, const int* __restrict__ labels,
                                                                 long long* __restrict__ xchg)
{
    __shared__ double buf[UWARPS][3][72];   // two 32-pixel chunks + the zero padding + one look-ahead group
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    const int k = blockIdx.x * UWARPS + wl;
    if (k >= s.n) return;
    // the box of this cluster's members, gathered by k_assign (empty when the cluster has no pixel)
    const int4 o = s.obb[k];
    if (BAND) {
        __syncwarp(); // every lane has its copy of the box before lane 0 resets it
        const bool alive = s.bin_of[k] >= 0;
        const int cr = alive ? (int)s.cy[k] : 0;   // row of the centre the assignment used
        if (lane == 0) {
            if (o.y >= o.x && (!alive || o.x + s.y_off < cr - s.halo || o.y + s.y_off > cr + s.halo))
                atomicAdd((unsigned long long*)&xchg[6 * (size_t)s.n], 1ull);
            s.obb[k] = make_int4(INT_MAX, -1, INT_MAX, -1);
        }
        if (!alive || cr < s.own_lo || cr >= s.own_hi) return;
    }
    const int y0 = o.x, y1 = o.y + 1, x0 = o.z, x1 = o.w + 1;
    const size_t HW = s.pstride;
    double acc = 0.0;
    long long cnt = 0, sy = 0, sx = 0;
    // the box is walked in raster order, 32 pixels at a time.  The loads are the latency that bounds this kernel, so label AND
    // colours of the chunks two ahead are requested (unconditionally: the box is ~2x the members, the extra reads hit L2)
    // before the current chunk is compacted and added.
    const int nchunk = (x1 > x0) ? (x1 - x0 + 31) / 32 : 0;
    const int total = (y1 > y0) ? (y1 - y0) * nchunk : 0;
    int ly = y0, lxb = x0;   // load cursor
    int cy_ = y0, cxb = x0;  // consume cursor
    int Lq[2];
    double Vq[2][3];
    auto issue = [&](int sl, bool valid) {
        const int x = lxb + lane;
        Lq[sl] = -1;
        if (valid && x < x1) {
            const size_t p = (size_t)ly * s.W + x;
            Lq[sl] = labels[p];
            Vq[sl][0] = lab[p]; Vq[sl][1] = lab[HW + p]; Vq[sl][2] = lab[2 * HW + p];
        }
        lxb += 32;
        if (lxb >= x1) { lxb = x0; ++ly; }
    };
    issue(0, total > 0);
    issue(1, total > 1);
    for (int it = 0; it < total; it += 2) {
        // two consecutive chunks per round: one compaction, one pair of warp barriers, one run of adds
        const bool two = it + 1 < total;
        const int l0 = Lq[0], l1 = two ? Lq[1] : -1;
        const double a0_ = Vq[0][0], a1_ = Vq[0][1], a2_ = Vq[0][2];
        const double b0_ = Vq[1][0], b1_ = Vq[1][1], b2_ = Vq[1][2];
        const int ya = cy_, xa = cxb + lane;
        cxb += 32;
        if (cxb >= x1) { cxb = x0; ++cy_; }
        const int yb = cy_, xb_ = cxb + lane;
        cxb += 32;
        if (cxb >= x1) { cxb = x0; ++cy_; }
        issue(0, it + 2 < total);
        issue(1, it + 3 < total);
        const bool m0 = l0 == k, m1 = l1 == k;
        const unsigned mask0 = __ballot_sync(0xffffffffu, m0), mask1 = __ballot_sync(0xffffffffu, m1);
        if (!(mask0 | mask1)) continue;
        const int nm0 = __popc(mask0), nm1 = __popc(mask1), nm = nm0 + nm1;
        const unsigned below = (1u << lane) - 1u;
        if (m0) {
            const int pos = __popc(mask0 & below);
            buf[wl][0][pos] = a0_; buf[wl][1][pos] = a1_; buf[wl][2][pos] = a2_;
            sx += xa;
        }
        if (m1) {
            const int pos = nm0 + __popc(mask1 & below);
            buf[wl][0][pos] = b0_; buf[wl][1][pos] = b1_; buf[wl][2][pos] = b2_;
            sx += xb_;
        }
        cnt += nm;
        sy += (long long)(ya + s.y_off) * nm0 + (long long)(yb + s.y_off) * nm1;
        // pad the run to a multiple of four with +0.0: x + (+0.0) == x for every x the sum can take (it starts at +0.0 and can
        // therefore never be -0.0), so the padded adds change nothing and the add loop has no remainder
        if (lane < 4) { buf[wl][0][nm + lane] = 0.0; buf[wl][1][nm + lane] = 0.0; buf[wl][2][nm + lane] = 0.0; }
        __syncwarp();
        if (lane < 3) {
            // sequential adds in raster order; the next four operands are loaded while the current four are added (the loads do not
            // depend on the running sum, only the adds form the chain)
            const double* bsrc = buf[wl][lane];
            const int ng = (nm + 3) >> 2;
            double c0 = bsrc[0], c1 = bsrc[1], c2 = bsrc[2], c3 = bsrc[3];
            for (int g = 1; g <= ng; ++g) {
                const double n0 = bsrc[4 * g], n1 = bsrc[4 * g + 1], n2 = bsrc[4 * g + 2], n3 = bsrc[4 * g + 3];   // (one group past the end: inside the buffer)
                acc = __dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(acc, c0), c1), c2), c3);
                c0 = n0; c1 = n1; c2 = n2; c3 = n3;
            }
        }
        __syncwarp();
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) sx += __shfl_xor_sync(0xffffffffu, sx, d);
    // centroid = sums / count with IEEE divisions (the original divides every feature by the element count), new window,
    // bin of the new centre; a cluster without pixels is dead for good
    const double a0 = __shfl_sync(0xffffffffu, acc, 0), a1 = __shfl_sync(0xffffffffu, acc, 1), a2 = __shfl_sync(0xffffffffu, acc, 2);
    if (BAND) {
        if (lane == 0) {
            long long* r = xchg + 6 * (size_t)k;
            if (cnt > 0) {
                const double dn = (double)cnt;
                r[0] = __double_as_longlong(__ddiv_rn((double)sy, dn)); r[1] = __double_as_longlong(__ddiv_rn((double)sx, dn));
                r[2] = __double_as_longlong(__ddiv_rn(a0, dn)); r[3] = __double_as_longlong(__ddiv_rn(a1, dn));
                r[4] = __double_as_longlong(__ddiv_rn(a2, dn));
                r[5] = 1;
            } else r[5] = 2;
        }
        return;
    }
    if (lane == 0) {
        int4 w = make_int4(0, 0, 0, 0);
        int bin = -1;
        if (cnt > 0) {
            const double dn = (double)cnt;
            const double cy = __ddiv_rn((double)sy, dn), cx = __ddiv_rn((double)sx, dn);
            s.cy[k] = cy; s.cx[k] = cx;
            s.c0[k] = __ddiv_rn(a0, dn); s.c1[k] = __ddiv_rn(a1, dn); s.c2[k] = __ddiv_rn(a2, dn);
            w = make_window(cy, cx, s.step_y, s.step_x, s.Hg, s.W);
            const int by = min(max((int)cy / s.B, 0), s.nby - 1), bx = min(max((int)cx / s.B, 0), s.nbx - 1);
            bin = by * s.nbx + bx;
            atomicAdd(&s.bin_fill[bin], 1);
        }
        s.win[k] = w;
        s.bin_of[k] = bin;
        s.obb[k] = make_int4(INT_MAX, -1, INT_MAX, -1);
    }
}

// band mode: take the merged exchange records (see k_update<true>) into the replicated cluster state
__global__ void k_import(KmState s, const long long* __restrict__ xchg)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= s.n) return;
    const long long* r = xchg + 6 * (size_t)k;
    const long long state = r[5];
    if (state == 1) {
        const double cy = __longlong_as_double(r[0]), cx = __longlong_as_double(r[1]);
        s.cy[k] = cy; s.cx[k] = cx;
        s.c0[k] = __longlong_as_double(r[2]); s.c1[k] = __longlong_as_double(r[3]); s.c2[k] = __longlong_as_double(r[4]);
        s.win[k] = make_window(cy, cx, s.step_y, s.step_x, s.Hg, s.W);
        const int by = min(max((int)cy / s.B, 0), s.nby - 1), bx = min(max((int)cx / s.B, 0), s.nbx - 1);
        s.bin_of[k] = by * s.nbx + bx;
        atomicAdd(&s.bin_fill[by * s.nbx + bx], 1);
    } else {
        // 2: the owner found no member, the cluster is dead for good; 0: it was dead already.  (An alive cluster always has
        // exactly one owner, so 0 cannot occur for it.)
        s.win[k] = make_int4(0, 0, 0, 0);
        s.bin_of[k] = -1;
    }
}

// SLICO: after the centres moved, remember the largest colour distance inside every cluster (the original only ever raises it)
__global__ void __launch_bounds__(256) k_slico_max(KmState s, const double* __restrict__ lab, const int* __restrict__ labels)
{
    // the rows this band owns (all of them on the monolithic path)
    const size_t HW = s.pstride;
    const size_t first = (size_t)(s.own_lo - s.y_off) * s.W, npx = (size_t)(s.own_hi - s.own_lo) * s.W;
    const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= npx) return;
    const size_t p = first + q;
    const int k = labels[p];
    const double d0 = __dsub_rn(lab[p], s.c0[k]), d1 = __dsub_rn(lab[HW + p], s.c1[k]), d2 = __dsub_rn(lab[2 * HW + p], s.c2[k]);
    double dcol = __dmul_rn(d0, d0);
    dcol = __dadd_rn(dcol, __dmul_rn(d1, d1));
    dcol = __dadd_rn(dcol, __dmul_rn(d2, d2));
    if (dcol == dcol) atomicMax(&s.maxdc[k], (unsigned long long)__double_as_longlong(dcol));
}

__global__ void k_export_centroids(KmState s, double* out)
{
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= s.n) return;
    out[5 * k] = s.cy[k]; out[5 * k + 1] = s.cx[k];
    out[5 * k + 2] = s.c0[k]; out[5 * k + 3] = s.c1[k]; out[5 * k + 4] = s.c2[k];
}

static size_t carve(KmState& s, void* ws, size_t bytes, int H, int W, int n, int step_y, int step_x)
{
    WsCarver c(ws, bytes);
    // H here is the height the cluster geometry lives in (the whole image); band callers overwrite the slab fields afterwards
    s.n = n; s.H = H; s.W = W; s.step_y = step_y; s.step_x = step_x;
    s.Hg = H; s.y_off = 0; s.own_lo = 0; s.own_hi = H; s.halo = 0; s.pstride = (size_t)H * W;
    s.B = 2 * (step_y > step_x ? step_y : step_x); // bin edge: coarse enough that the per-sweep scan over the bins is short
    if (s.B < 16) s.B = 16;
    s.nby = (H + s.B - 1) / s.B; s.nbx = (W + s.B - 1) / s.B;
    s.cy = c.take<double>(n); s.cx = c.take<double>(n);
    s.c0 = c.take<double>(n); s.c1 = c.take<double>(n); s.c2 = c.take<double>(n);
    s.win = c.take<int4>(n); s.obb = c.take<int4>(n);
    s.bin_start = c.take<int>((size_t)s.nby * s.nbx + 1);
    s.bin_fill = c.take<int>((size_t)s.nby * s.nbx);
    s.bin_of = c.take<int>(n);
    s.pack_done = c.take<int>(1);
    s.packed = c.take<Cand>(n);
    s.maxdc = c.take<unsigned long long>(n);
    s.packed_maxdc = c.take<double>(n);
    return isb_align(c.off);
}

// seeds != nullptr: first binning (centres from the seed grid); else re-binning after k_update / k_import
static int rebin(KmState& s, const double* seeds_yx, cudaStream_t st)
{
    if (seeds_yx) {
        ISB_CUDA_CHECK(cudaMemsetAsync(s.bin_fill, 0, sizeof(int) * (size_t)s.nby * s.nbx, st));
        k_seed<<<(s.n + 255) / 256, 256, 0, st>>>(s, seeds_yx);
        ISB_LAUNCH_CHECK();
    }
    k_scan_bins<<<1, 1024, 0, st>>>(s);
    ISB_LAUNCH_CHECK();
    k_pack<<<(s.n + 255) / 256, 256, 0, st>>>(s);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// 3-D tensor map over the Lab planes of a slab: (x, y, plane) with a 32 x 32 x 3 box.  TMA needs 16-byte multiples for the row and
// plane pitches (W and plane stride even) and a 16-byte aligned base; otherwise the kernel stages the tile with ordinary loads.
static bool make_lab_map(CUtensorMap& map, const double* lab, int rows, int W, size_t plane_stride)
{
    wgmma::EncodeTiledFn encode = wgmma::encode_tiled_fn();
    if (!encode || (W & 1) || (plane_stride & 1) || ((uintptr_t)lab & 15)) return false;
    const cuuint64_t gdim[3] = { (cuuint64_t)W, (cuuint64_t)rows, 3 };
    const cuuint64_t gstride[2] = { (cuuint64_t)W * sizeof(double), (cuuint64_t)plane_stride * sizeof(double) };
    const cuuint32_t box[3] = { TILE, TILE, 3 };
    const cuuint32_t estr[3] = { 1, 1, 1 };
    return encode(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, (void*)lab, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static void launch_assign(const KmState& s, const CUtensorMap& map, int use_tma, const double* lab, int* labels, cudaStream_t st)
{
    dim3 agrid((s.W + TILE - 1) / TILE, (s.H + TILE - 1) / TILE);
    if (s.slico) k_assign<true><<<agrid, ATHREADS, 0, st>>>(map, use_tma, s, lab, labels);
    else k_assign<false><<<agrid, ATHREADS, 0, st>>>(map, use_tma, s, lab, labels);
}

} // namespace

extern "C" size_t isb_slic_kmeans_workspace_bytes(int H, int W, int n_seeds, int step_y, int step_x)
{
    KmState s;
    return carve(s, nullptr, 0, H, W, n_seeds, step_y, step_x);
}

extern "C" int isb_slic_kmeans(const double* lab_planar, int H, int W, const double* seeds_yx, int n_seeds, int step_y,
                               int step_x, double step, int max_iter, int slic_zero, int32_t* labels, double* centroids,
                               void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(lab_planar && seeds_yx && labels && ws, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && n_seeds > 0 && step_y > 0 && step_x > 0 && step > 0, "bad sizes");
    KmState s;
    size_t need = carve(s, ws, ws_bytes, H, W, n_seeds, step_y, step_x);
    ISB_REQUIRE(need <= ws_bytes, "workspace too small");
    s.sw = 1.0 / (step * step);
    s.slico = slic_zero ? 1 : 0;
    cudaStream_t st = (cudaStream_t)stream;
    ISB_CUDA_CHECK(cudaMemsetAsync(labels, 0, sizeof(int32_t) * (size_t)H * W, st));
    if (int rc = rebin(s, seeds_yx, st)) return rc;
    CUtensorMap lab_map;
    memset(&lab_map, 0, sizeof(lab_map));
    const int use_tma = make_lab_map(lab_map, lab_planar, H, W, s.pstride) ? 1 : 0;
    for (int it = 0; it < max_iter; ++it) {
        {
            ProfScope p(ISB_PROF_ASSIGN, st);
            launch_assign(s, lab_map, use_tma, lab_planar, labels, st);
        }
        ISB_LAUNCH_CHECK();
        { ProfScope p(ISB_PROF_UPDATE, st); k_update<false><<<(n_seeds + UWARPS - 1) / UWARPS, 32 * UWARPS, 0, st>>>(s, lab_planar, labels, nullptr); }
        ISB_LAUNCH_CHECK();
        if (slic_zero) {
            const size_t npx = (size_t)H * W;
            k_slico_max<<<(unsigned)((npx + 255) / 256), 256, 0, st>>>(s, lab_planar, labels);
            ISB_LAUNCH_CHECK();
        }
        { ProfScope p(ISB_PROF_FINALIZE, st); if (int rc = rebin(s, nullptr, st)) return rc; }
    }
    if (centroids) {
        k_export_centroids<<<(n_seeds + 255) / 256, 256, 0, st>>>(s, centroids);
        ISB_LAUNCH_CHECK();
    }
    return ISB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Row-band mode: the same sweeps with one band of the image per GPU.  The cluster state is replicated; what crosses the
// GPUs each sweep is the exchange buffer of k_update<true> (summed as int64 by the caller's collective).
// ---------------------------------------------------------------------------------------------------------------------
namespace {

static int band_state(const isb_slic_band_t* b, KmState& s)
{
    ISB_REQUIRE(b && b->lab_slab && b->seeds_yx && b->labels_slab && b->ws, "null pointer");
    ISB_REQUIRE(b->slab_rows > 0 && b->width > 0 && b->image_rows > 0 && b->n_seeds > 0 && b->step_y > 0 && b->step_x > 0 && b->step > 0,
                "bad sizes");
    ISB_REQUIRE(b->y_off >= 0 && b->y_off + b->slab_rows <= b->image_rows, "slab outside the image");
    ISB_REQUIRE(b->own_lo >= b->y_off && b->own_hi <= b->y_off + b->slab_rows && b->own_lo < b->own_hi, "owned rows outside the slab");
    ISB_REQUIRE(b->halo >= 2 * b->step_y, "halo must be at least 2 * step_y rows");
    ISB_REQUIRE(b->y_off <= (b->own_lo - b->halo > 0 ? b->own_lo - b->halo : 0), "slab does not cover the halo above the owned rows");
    ISB_REQUIRE(b->y_off + b->slab_rows >= (b->own_hi + b->halo < b->image_rows ? b->own_hi + b->halo : b->image_rows),
                "slab does not cover the halo below the owned rows");
    ISB_REQUIRE(b->plane_stride >= (size_t)b->slab_rows * b->width, "plane stride smaller than the slab");
    size_t need = carve(s, b->ws, b->ws_bytes, b->image_rows, b->width, b->n_seeds, b->step_y, b->step_x);
    ISB_REQUIRE(need <= b->ws_bytes, "workspace too small");
    s.H = b->slab_rows; s.Hg = b->image_rows; s.y_off = b->y_off; s.own_lo = b->own_lo; s.own_hi = b->own_hi; s.halo = b->halo;
    s.pstride = b->plane_stride;
    s.sw = 1.0 / (b->step * b->step);
    s.slico = b->slic_zero ? 1 : 0;
    return ISB_OK;
}

} // namespace

extern "C" int isb_slic_band_begin(const isb_slic_band_t* b, isb_stream_t stream)
{
    KmState s;
    if (int rc = band_state(b, s)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    ISB_CUDA_CHECK(cudaMemsetAsync(b->labels_slab, 0, sizeof(int32_t) * (size_t)b->slab_rows * b->width, st));
    return rebin(s, b->seeds_yx, st);
}

extern "C" int isb_slic_band_assign(const isb_slic_band_t* b, isb_stream_t stream)
{
    KmState s;
    if (int rc = band_state(b, s)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    CUtensorMap lab_map;
    memset(&lab_map, 0, sizeof(lab_map));
    const int use_tma = make_lab_map(lab_map, b->lab_slab, s.H, s.W, s.pstride) ? 1 : 0;
    ProfScope p(ISB_PROF_ASSIGN, st);
    launch_assign(s, lab_map, use_tma, b->lab_slab, b->labels_slab, st);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_slic_band_update(const isb_slic_band_t* b, int64_t* xchg, isb_stream_t stream)
{
    KmState s;
    if (int rc = band_state(b, s)) return rc;
    ISB_REQUIRE(xchg, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope p(ISB_PROF_UPDATE, st);
    ISB_CUDA_CHECK(cudaMemsetAsync(xchg, 0, sizeof(int64_t) * (6 * (size_t)s.n + 1), st));
    k_update<true><<<(s.n + UWARPS - 1) / UWARPS, 32 * UWARPS, 0, st>>>(s, b->lab_slab, b->labels_slab, (long long*)xchg);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_slic_band_import(const isb_slic_band_t* b, const int64_t* xchg, uint64_t* maxdc_xchg, isb_stream_t stream)
{
    KmState s;
    if (int rc = band_state(b, s)) return rc;
    ISB_REQUIRE(xchg && (!s.slico || maxdc_xchg), "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    k_import<<<(s.n + 255) / 256, 256, 0, st>>>(s, (const long long*)xchg);
    ISB_LAUNCH_CHECK();
    if (s.slico) {
        const size_t npx = (size_t)(s.own_hi - s.own_lo) * s.W;
        k_slico_max<<<(unsigned)((npx + 255) / 256), 256, 0, st>>>(s, b->lab_slab, b->labels_slab);
        ISB_LAUNCH_CHECK();
        ISB_CUDA_CHECK(cudaMemcpyAsync(maxdc_xchg, s.maxdc, sizeof(uint64_t) * (size_t)s.n, cudaMemcpyDeviceToDevice, st));
    }
    return ISB_OK;
}

extern "C" int isb_slic_band_finalize(const isb_slic_band_t* b, const uint64_t* maxdc_xchg, isb_stream_t stream)
{
    KmState s;
    if (int rc = band_state(b, s)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (s.slico) {
        ISB_REQUIRE(maxdc_xchg, "null pointer");
        ISB_CUDA_CHECK(cudaMemcpyAsync(s.maxdc, maxdc_xchg, sizeof(uint64_t) * (size_t)s.n, cudaMemcpyDeviceToDevice, st));
    }
    ProfScope p(ISB_PROF_FINALIZE, st);
    return rebin(s, nullptr, st);
}
