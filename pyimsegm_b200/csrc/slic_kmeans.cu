// slic_kmeans.cu -- the k-means sweeps of SLIC, pixel-centric and bit-exact with oracle/slic_oracle.c.
//
// Replaces skimage.segmentation._slic._slic_cython as called through imsegm/superpixels.py:61-63.
//
// The original is cluster-centric: for k ascending, scan the +-2*step window and take the pixel when
// `distance > d` (strict) -- i.e. every pixel ends with argmin over {clusters whose window holds it} of
// (d, k) in lexicographic order.  That per-pixel minimum is order-independent, so it is evaluated here
// pixel-centric: one CTA per 32x32 pixel tile takes the list of the clusters whose integer window intersects the tile
// (written by whoever last set the cluster's centre), every pixel loops over that list in shared memory.
// The distance is computed with the oracle's exact operation order in IEEE double (no FMA).
//
// The centroid update of the original is a raster-order SEQUENTIAL double sum per cluster; a tree/atomic
// reduction changes the last ulp and flips exact ties (flat image regions tie all the time).  It is
// reproduced exactly: one CTA per cluster walks the cluster's member box in raster order, its gather warps ballot
// the member pixels of each 32-wide chunk and compact their colours into shared memory in raster order, and three
// lanes of an adder warp add them one at a time.  Coordinate sums are integers (exact in any order).
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
    // per 32x32 tile of the pixel memory: the records of the clusters whose window meets it, in no particular order.  A tile whose
    // count exceeds tcap has overflowed (its list is incomplete) and k_assign scans every cluster for it instead.
    int* tile_cnt;   // [tiles]
    Cand* tile_cand; // [tiles * tcap]
    unsigned long long* maxdc; // [n] SLICO colour-distance maxima as raw double bits (non-negative doubles order like their bits)
    int slico;
    int n, H, W, step_y, step_x, ntx, tcap;   // ntx: tiles per row
    double sw;       // spatial weight 1/step^2
    // Row-band mode (one band of a taller image per GPU, isb_slic_band_*): pixel memory is a slab of H rows whose row 0 is
    // global row y_off of an image Hg rows tall; cluster geometry (centres, windows) is always global.  The
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

// Between two sweeps nothing is re-binned: whoever sets a cluster's centre -- k_seed (first sweep), k_update<false> or k_import
// (band mode) -- appends its record to the list of every tile its window meets, and k_assign zeroes its tile's count once it
// has read it, so that the next appends start from zero.  Dead clusters append nothing.
__device__ __forceinline__ Cand make_cand(int k, double cy, double cx, double c0, double c1, double c2, int4 w)
{
    Cand c;
    c.cy = cy; c.cx = cx; c.c0 = c0; c.c1 = c1; c.c2 = c2;
    c.y0 = w.x; c.y1 = w.y; c.x0 = w.z; c.x1 = w.w; c.k = k; c.pad = 0;
    return c;
}

// append c to the tiles of this slab that its window meets; thread t of nt takes every nt-th of those tiles
__device__ __forceinline__ void append_tiles(const KmState& s, const Cand& c, int t, int nt)
{
    const int ya = max(c.y0 - s.y_off, 0), yb = min(c.y1 - s.y_off, s.H);   // the window's rows in the slab
    if (ya >= yb || c.x0 >= c.x1) return;
    const int ty0 = ya / TILE, tx0 = c.x0 / TILE;
    const int nx = (c.x1 - 1) / TILE - tx0 + 1, nxy = ((yb - 1) / TILE - ty0 + 1) * nx;
    for (int i = t; i < nxy; i += nt) {
        const int tile = (ty0 + i / nx) * s.ntx + tx0 + i % nx;
        const int pos = atomicAdd(&s.tile_cnt[tile], 1);
        if (pos < s.tcap) s.tile_cand[(size_t)tile * s.tcap + pos] = c;
    }
}

__global__ void k_seed(KmState s, const double* __restrict__ seeds_yx)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= s.n) return;
    const double cy = seeds_yx[2 * k], cx = seeds_yx[2 * k + 1];
    s.cy[k] = cy; s.cx[k] = cx; s.c0[k] = 0.0; s.c1[k] = 0.0; s.c2[k] = 0.0;
    const int4 w = make_window(cy, cx, s.step_y, s.step_x, s.Hg, s.W);
    s.win[k] = w;
    s.obb[k] = make_int4(INT_MAX, -1, INT_MAX, -1);
    s.maxdc[k] = (unsigned long long)__double_as_longlong(1.0);
    append_tiles(s, make_cand(k, cy, cx, 0.0, 0.0, 0.0, w), 0, 1);
}

// non-negative doubles order like their bit patterns: compare on the integer pipe instead of the FP64 pipe
// (unsigned, so that a NaN of either sign ranks above every number and can never win)
__device__ __forceinline__ unsigned long long dbits(double v) { return (unsigned long long)__double_as_longlong(v); }

// tile assignments that scanned every cluster because their list overflowed (isb_slic_full_scan_tiles)
__device__ unsigned long long d_full_scans;

// per-candidate floats of the per-thread lower bounds: the centre, every colour channel rounded down (lo) and up (hi), and for
// SLICO 1 / maxdc rounded down
struct __align__(16) CandF {
    float cy, cx, inv, pad0;
    float lo0, lo1, lo2, pad1;
    float hi0, hi1, hi2, pad2;
};

// assignment: one CTA (128 threads) per 32x32 tile; a thread owns one column and AROWS = 8 consecutive rows.
// The tile's Lab values arrive in shared memory by a TMA load while the candidate list is staged and sorted, candidates are
// visited nearest-first and the loop stops as soon as the spatial lower bound of every remaining candidate exceeds the worst of
// the thread's current minima.
template <bool SLICO>
__global__ void __launch_bounds__(ATHREADS, 5) k_assign(const __grid_constant__ CUtensorMap lab_map, int use_tma, KmState s,
                                                        const double* __restrict__ lab, int* __restrict__ labels)
{
    __shared__ __align__(16) Cand cand[ACAP];
    __shared__ double s_maxdc[SLICO ? ACAP : 1];
    __shared__ float s_key[ACAP];
    __shared__ CandF s_cf[ACAP];
    __shared__ double s_lb[ACAP];          // lower bound of the spatial term of the candidate at sorted position i, and of all later ones
    __shared__ unsigned char s_order[ACAP];
    __shared__ __align__(128) double s_px[3][TILE][TILE]; // Lab of the tile
    __shared__ __align__(8) unsigned long long s_bar;     // mbarrier of the TMA tile load
    __shared__ int s_ncand, s_done;
    const int tx0 = blockIdx.x * TILE, ty0 = blockIdx.y * TILE;
    const int tx1 = min(tx0 + TILE, s.W);
    const int gy0 = ty0 + s.y_off, gy1 = min(ty0 + TILE, s.H) + s.y_off; // the tile's rows in global coordinates
    const int tile = blockIdx.y * s.ntx + blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t HW = s.pstride;
    const int x = tx0 + lane;
    const bool xin = x < s.W;
    const int yb = ty0 + warp * AROWS; // first row of this thread
    const uint32_t bar = wgmma::smem_u32(&s_bar);

    double best[AROWS];
    int bestk[AROWS];
#pragma unroll
    for (int j = 0; j < AROWS; ++j) { best[j] = DBL_MAX; bestk[j] = -1; }
    if (threadIdx.x == 0 && use_tma) {
        // the three Lab planes of the tile arrive as ONE 3-D tensor-map load (32 x 32 x 3 doubles, out-of-image elements read as 0)
        // while the candidates are staged and sorted; the distance loop waits for it
        wgmma::mbar_init(bar, 1);
        wgmma::fence_mbar_init();
        wgmma::mbar_arrive_expect_tx(bar, 3 * TILE * TILE * 8);
        wgmma::tma_load_3d(wgmma::smem_u32(&s_px[0][0][0]), &lab_map, tx0, ty0, 0, bar);
    }
    // the tile's list: every thread reads the count (one broadcast load); a complete list of one round is staged by 16-byte loads
    // spread over the CTA, a longer or overflowed one in rounds below
    const int total = s.tile_cnt[tile];
    const bool scan_all = total > s.tcap;   // the list overflowed: every cluster's window is tested instead
    const bool fast = total <= ACAP && !scan_all;
    if (fast) {
        const int4* src = reinterpret_cast<const int4*>(s.tile_cand + (size_t)tile * s.tcap);
        int4* dst = reinterpret_cast<int4*>(cand);
        for (int i = threadIdx.x; i < total * (int)(sizeof(Cand) / sizeof(int4)); i += ATHREADS) dst[i] = src[i];
    }
    if (!use_tma) {
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
    const float tcy = 0.5f * (gy0 + gy1 - 1), tcx = 0.5f * (tx0 + tx1 - 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        s.tile_cnt[tile] = 0;   // read by every thread before the barrier; the next sweep's appends start from zero
        if (scan_all) atomicAdd(&d_full_scans, 1ull);
    }

    int off = 0;   // warp 0, rounds: where the next round resumes
    while (true) {
        if (!fast && warp == 0) {
            // deterministic, resumable scan: up to ACAP candidates per round, from the tile's list while it is complete, else from
            // every cluster whose window meets the tile
            const int end = scan_all ? s.n : total;
            int n = 0;
            while (off < end && n < ACAP) {
                const int room = ACAP - n;
                const int i = off + lane;
                bool ok = false;
                Cand c;
                if (i < end && lane < room) {
                    if (scan_all) {
                        const int4 w = s.win[i];
                        ok = (w.x < gy1) && (w.y > gy0) && (w.z < tx1) && (w.w > tx0);
                        if (ok) c = make_cand(i, s.cy[i], s.cx[i], s.c0[i], s.c1[i], s.c2[i], w);
                    } else {
                        c = s.tile_cand[(size_t)tile * s.tcap + i];
                        ok = true;
                    }
                }
                const unsigned m = __ballot_sync(0xffffffffu, ok);
                if (ok) cand[n + __popc(m & ((1u << lane) - 1u))] = c;
                n += __popc(m);
                off += min(min(32, room), end - off);
            }
            if (lane == 0) { s_ncand = n; s_done = off >= end; }
        }
        if (!fast) __syncthreads();   // the round is staged
        const int nc = fast ? total : s_ncand;
        const int done = fast || s_done;
        for (int t = threadIdx.x; t < nc; t += ATHREADS) {
            const Cand& c = cand[t];
            const float fy = (float)c.cy - tcy, fx = (float)c.cx - tcx;
            s_key[t] = fy * fy + fx * fx;
            CandF f;
            f.cy = (float)c.cy; f.cx = (float)c.cx; f.inv = 1.f; f.pad0 = f.pad1 = f.pad2 = 0.f;
            f.lo0 = __double2float_rd(c.c0); f.lo1 = __double2float_rd(c.c1); f.lo2 = __double2float_rd(c.c2);
            f.hi0 = __double2float_ru(c.c0); f.hi1 = __double2float_ru(c.c1); f.hi2 = __double2float_ru(c.c2);
            if (SLICO) {
                // the maximum as it is now: k_slico_max raised it after the record was written
                const double m = __longlong_as_double((long long)s.maxdc[c.k]);
                s_maxdc[t] = m;
                f.inv = __frcp_rd(__double2float_ru(m));
            }
            s_cf[t] = f;
        }
        __syncthreads();
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
        if (use_tma) wgmma::mbar_wait(bar, 0);   // phase 0 completes once; later rounds pass immediately
        // the colour box of this thread's pixels (the rows inside the image), every bound rounded outwards
        float plo0 = INFINITY, plo1 = INFINITY, plo2 = INFINITY, phi0 = -INFINITY, phi1 = -INFINITY, phi2 = -INFINITY;
#pragma unroll
        for (int j = 0; j < AROWS; ++j) {
            if (yb + j < s.H) {
                const int ry = warp * AROWS + j;
                const double v0 = s_px[0][ry][lane], v1 = s_px[1][ry][lane], v2 = s_px[2][ry][lane];
                plo0 = fminf(plo0, __double2float_rd(v0)); phi0 = fmaxf(phi0, __double2float_ru(v0));
                plo1 = fminf(plo1, __double2float_rd(v1)); phi1 = fmaxf(phi1, __double2float_ru(v1));
                plo2 = fminf(plo2, __double2float_rd(v2)); phi2 = fmaxf(phi2, __double2float_ru(v2));
            }
        }
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
                    // lower bound of this candidate's distance for ALL of the thread's pixels, in float.  Spatial term: the centre is
                    // at least |cx - x| away in x and |cy - ymid| - (AROWS-1)/2 in y; 2e-3 px absorbs the float conversion of
                    // the centre for coordinates below 2^16 (half an ulp is 2^-9 px there), the factor 0.998 the rounding of the few
                    // float operations.  Past 2^16 the conversion moves a centre by up to 2^-8 px (2^-7 past 2^17), more than the
                    // slack, so the bound is proven only for sides below 65 536 px; on taller or wider images no input has been
                    // found where it rejects a candidate that wins or ties (tests/test_gpu_slic_edges.py).  Colour term: each channel
                    // is at least the gap between the pixels' box and the centre; the box, the centre and every operation round
                    // towards a smaller result, so the term is at most the exact sum of squares, and the factor 0.998 leaves room
                    // for the rounding of the double chain (the double distance is at least the exact one times 1 - 2^-50).
                    // Both terms can only come out smaller than the exact double distance, and fl(a + b) >= a for b >= 0, so a
                    // candidate whose bound exceeds every row's minimum cannot win or tie any row
                    const CandF f = s_cf[c];
                    const float ax = fmaxf(fabsf(f.cx - xf) - 2e-3f, 0.f), ay = fmaxf(fabsf(f.cy - ymid) - (0.5f * (AROWS - 1) + 2e-3f), 0.f);
                    const float lbs = (ax * ax + ay * ay) * swf;
                    if (lbs > worstf) continue;
                    const float g0 = fmaxf(fmaxf(__fsub_rd(plo0, f.hi0), __fsub_rd(f.lo0, phi0)), 0.f);
                    const float g1 = fmaxf(fmaxf(__fsub_rd(plo1, f.hi1), __fsub_rd(f.lo1, phi1)), 0.f);
                    const float g2 = fmaxf(fmaxf(__fsub_rd(plo2, f.hi2), __fsub_rd(f.lo2, phi2)), 0.f);
                    float lbc = __fadd_rd(__fadd_rd(__fmul_rd(g0, g0), __fmul_rd(g1, g1)), __fmul_rd(g2, g2));
                    if (SLICO) lbc = __fmul_rd(lbc, f.inv);
                    if (__fmaf_rd(lbc, 0.998f, lbs) > worstf) continue;
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

// centroid sums: one CTA per cluster, raster-order sequential double adds (see header).
// BAND: this GPU holds a row band of the image.  A cluster is summed by the band that owns the row of its centre (every
// member lies within 2*step rows of the centre the assignment used, i.e. inside that band's slab -- checked, violations are
// counted in xchg[6n]); the result goes to the exchange record xchg[6k..6k+5] = bits(cy, cx, c0, c1, c2), state (1 alive,
// 2 died) and every other band leaves zeros there, so that an integer sum over the bands is an exact merge.
//
// The member box is cut into strips of USTRIP chunks (a chunk = 32 pixels of one box row) in raster chunk order.  The UGATHER gather
// warps share a strip, UCPW consecutive chunks each: they load the labels and ballot the members, the per-chunk member counts are
// scanned across the gather warps, and only the member lanes load their colours and store them at their raster position in the
// strip buffer.  The last warp is the adder: three of its lanes (one per channel) run the sequential chain over one buffer while
// the gather warps fill the other.  Named barriers hand the buffers over (FULL: the strip is stored, EMPTY: its adds are done), so
// neither side waits for a whole-CTA barrier.  A strip is a fixed number of chunks: a large box just takes more strips.
// A CTA's time is mostly its adder's chain plus a few memory latencies (box, labels, colours of the first strip), so the kernel
// wants many clusters in flight per SM: 3 gather warps, 12-chunk strips (19 KB of shared memory) and 9 CTAs per SM, which leave 56
// registers -- the kernel fits them without spilling (at 10 CTAs it spills, and it was slower with 4 or 2 gather warps on H100).
// CTAs take the clusters from the last to the first: k_assign has just streamed the image top to bottom, so the bottom rows are
// still in L2 when the first CTAs need them, and the next k_assign finds the top rows there.
constexpr int UGATHER = 3, UCPW = 4, USTRIP = UGATHER * UCPW;
constexpr int UTHREADS = 32 * (UGATHER + 1), UBLOCKS = 9;
// one channel row of a strip buffer: the members, the zero padding and one look-ahead group of the adds; the extra 4 words put
// the three rows the adder lanes read at once on different banks
constexpr int USTRIDE = 32 * USTRIP + 12;
constexpr int UBAR_FULL = 1, UBAR_EMPTY = 3, UBAR_SCAN = 5;   // FULL and EMPTY: one barrier per buffer; 0 is __syncthreads

// named barriers with immediate operands (ptxas then reserves only the ids in use); ID + b selects the barrier of buffer b
template <int ID, int N> __device__ __forceinline__ void bar_sync(int b = 0)
{
    if (b) asm volatile("bar.sync %0, %1;" ::"n"(ID + 1), "n"(N) : "memory");
    else asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(N) : "memory");
}
template <int ID, int N> __device__ __forceinline__ void bar_arrive(int b)
{
    if (b) asm volatile("bar.arrive %0, %1;" ::"n"(ID + 1), "n"(N) : "memory");
    else asm volatile("bar.arrive %0, %1;" ::"n"(ID), "n"(N) : "memory");
}

template <bool BAND>
__global__ void __launch_bounds__(UTHREADS, UBLOCKS) k_update(KmState s, const double* __restrict__ lab, const int* __restrict__ labels,
                                                              long long* __restrict__ xchg)
{
    __shared__ __align__(16) double buf[2][3][USTRIDE];
    __shared__ int s_cnt[2][USTRIP];   // members per chunk of the strip in the buffer
    __shared__ int s_tot[2];           // members of the strip in the buffer
    __shared__ long long s_int[UGATHER][3];
    __shared__ double s_acc[3];
    __shared__ int4 s_box;
    __shared__ int s_skip;
    __shared__ Cand s_rec;             // the new record of the cluster
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    const int k = s.n - 1 - blockIdx.x;   // last cluster first (see above)
    if (threadIdx.x == 0) {
        // the box of this cluster's members, gathered by k_assign (empty when the cluster has no pixel)
        const int4 o = s.obb[k];
        int skip = 0;
        if (BAND) {
            const int4 w = s.win[k];
            const bool alive = w.y > w.x;   // an alive cluster's window holds its centre row; a dead one's is empty
            const int cr = alive ? (int)s.cy[k] : 0;   // row of the centre the assignment used
            if (o.y >= o.x && (!alive || o.x + s.y_off < cr - s.halo || o.y + s.y_off > cr + s.halo))
                atomicAdd((unsigned long long*)&xchg[6 * (size_t)s.n], 1ull);
            s.obb[k] = make_int4(INT_MAX, -1, INT_MAX, -1);
            skip = !alive || cr < s.own_lo || cr >= s.own_hi;
        }
        s_box = o; s_skip = skip;
    }
    __syncthreads();
    if (s_skip) return;
    const int4 o = s_box;
    const int y0 = o.x, y1 = o.y + 1, x0 = o.z, x1 = o.w + 1;
    const int nchunk = (x1 > x0) ? (x1 - x0 + 31) / 32 : 0;
    const int total = (y1 > y0) ? (y1 - y0) * nchunk : 0;
    const int nstrip = (total + USTRIP - 1) / USTRIP;
    if (wl < UGATHER) {
        const size_t HW = s.pstride;
        const unsigned below = (1u << lane) - 1u;
        long long cnt = 0, sy = 0, sx = 0;
        // chunk j of this warp in strip i: its row and this lane's column (out of the box: no pixel)
        auto chunk_at = [&](int i, int j, int& y, int& x) {
            const int c = i * USTRIP + wl * UCPW + j;
            const int r = c / nchunk;
            y = y0 + r; x = x0 + 32 * (c - r * nchunk) + lane;
            return c < total && x < x1;
        };
        // the labels of the next strip are requested while the current one is compacted
        int lbl[UCPW];
        auto load_labels = [&](int i) {
#pragma unroll
            for (int j = 0; j < UCPW; ++j) {
                int y, x;
                lbl[j] = (i < nstrip && chunk_at(i, j, y, x)) ? labels[(size_t)y * s.W + x] : -1;
            }
        };
        load_labels(0);
        for (int i = 0; i < nstrip; ++i) {
            const int b = i & 1;
            unsigned mask[UCPW];
            double v[UCPW][3];
#pragma unroll
            for (int j = 0; j < UCPW; ++j) {
                int y, x;
                chunk_at(i, j, y, x);
                const bool m = lbl[j] == k;
                mask[j] = __ballot_sync(0xffffffffu, m);
                if (m) {
                    const size_t p = (size_t)y * s.W + x;
                    v[j][0] = lab[p]; v[j][1] = lab[HW + p]; v[j][2] = lab[2 * HW + p];
                    ++cnt; sy += y + s.y_off; sx += x;
                }
            }
            load_labels(i + 1);
            if (lane == 0) {
#pragma unroll
                for (int j = 0; j < UCPW; ++j) s_cnt[b][wl * UCPW + j] = __popc(mask[j]);
            }
            bar_sync<UBAR_SCAN, 32 * UGATHER>();
            // exclusive scan of the chunk counts: where each chunk's members start in the strip
            const int cl = lane < USTRIP ? s_cnt[b][lane] : 0;
            int incl = cl;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
            const int excl = incl - cl, nm = __shfl_sync(0xffffffffu, incl, 31);
            if (i >= 2) bar_sync<UBAR_EMPTY, UTHREADS>(b);   // the adds of strip i - 2 are done with this buffer
#pragma unroll
            for (int j = 0; j < UCPW; ++j) {
                const int start = __shfl_sync(0xffffffffu, excl, wl * UCPW + j);
                if ((mask[j] >> lane) & 1u) {
                    const int pos = start + __popc(mask[j] & below);
                    buf[b][0][pos] = v[j][0]; buf[b][1][pos] = v[j][1]; buf[b][2][pos] = v[j][2];
                }
            }
            // pad the strip to a multiple of four with +0.0: x + (+0.0) == x for every x the sum can take (it starts at +0.0 and can
            // therefore never be -0.0), so the padded adds change nothing and the add loop has no remainder
            if (wl == 0 && lane < 4) {
                buf[b][0][nm + lane] = 0.0; buf[b][1][nm + lane] = 0.0; buf[b][2][nm + lane] = 0.0;
                if (lane == 0) s_tot[b] = nm;
            }
            bar_arrive<UBAR_FULL, UTHREADS>(b);
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            cnt += __shfl_xor_sync(0xffffffffu, cnt, d); sy += __shfl_xor_sync(0xffffffffu, sy, d); sx += __shfl_xor_sync(0xffffffffu, sx, d);
        }
        if (lane == 0) { s_int[wl][0] = cnt; s_int[wl][1] = sy; s_int[wl][2] = sx; }
    } else {
        double acc = 0.0;
        for (int i = 0; i < nstrip; ++i) {
            const int b = i & 1;
            bar_sync<UBAR_FULL, UTHREADS>(b);
            if (lane < 3) {
                // sequential adds in raster order; the next four operands are loaded while the current four are added (the loads do not
                // depend on the running sum, only the adds form the chain)
                const double2* bsrc = reinterpret_cast<const double2*>(buf[b][lane]);
                const int ng = (s_tot[b] + 3) >> 2;
                double2 c01 = bsrc[0], c23 = bsrc[1];
                for (int g = 1; g <= ng; ++g) {
                    const double2 n01 = bsrc[2 * g], n23 = bsrc[2 * g + 1];   // (one group past the end: inside the buffer)
                    acc = __dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(acc, c01.x), c01.y), c23.x), c23.y);
                    c01 = n01; c23 = n23;
                }
            }
            __syncwarp();
            if (i + 2 < nstrip) bar_arrive<UBAR_EMPTY, UTHREADS>(b);   // the gather warps wait for this only if they refill the buffer
        }
        if (lane < 3) s_acc[lane] = acc;
    }
    __syncthreads();
    if (wl != 0) return;
    if (lane == 0) {
        long long cnt = 0, sy = 0, sx = 0;
#pragma unroll
        for (int w = 0; w < UGATHER; ++w) { cnt += s_int[w][0]; sy += s_int[w][1]; sx += s_int[w][2]; }
        // centroid = sums / count with IEEE divisions (the original divides every feature by the element count), new window;
        // a cluster without pixels is dead for good
        const double a0 = s_acc[0], a1 = s_acc[1], a2 = s_acc[2];
        if (BAND) {
            long long* r = xchg + 6 * (size_t)k;
            if (cnt > 0) {
                const double dn = (double)cnt;
                r[0] = __double_as_longlong(__ddiv_rn((double)sy, dn)); r[1] = __double_as_longlong(__ddiv_rn((double)sx, dn));
                r[2] = __double_as_longlong(__ddiv_rn(a0, dn)); r[3] = __double_as_longlong(__ddiv_rn(a1, dn));
                r[4] = __double_as_longlong(__ddiv_rn(a2, dn));
                r[5] = 1;
            } else r[5] = 2;
        } else {
            int4 w = make_int4(0, 0, 0, 0);
            if (cnt > 0) {
                const double dn = (double)cnt;
                const double cy = __ddiv_rn((double)sy, dn), cx = __ddiv_rn((double)sx, dn);
                const double c0 = __ddiv_rn(a0, dn), c1 = __ddiv_rn(a1, dn), c2 = __ddiv_rn(a2, dn);
                s.cy[k] = cy; s.cx[k] = cx; s.c0[k] = c0; s.c1[k] = c1; s.c2[k] = c2;
                w = make_window(cy, cx, s.step_y, s.step_x, s.Hg, s.W);
                s_rec = make_cand(k, cy, cx, c0, c1, c2, w);
            } else s_rec.y0 = s_rec.y1 = 0;   // dead: an empty window, no tile
            s.win[k] = w;
            s.obb[k] = make_int4(INT_MAX, -1, INT_MAX, -1);
        }
    }
    if (BAND) return;   // band mode: k_import appends the merged centres
    // the next k_assign's candidate lists: the new record goes to every tile its window meets (up to 5 x 5 tiles at step 29),
    // one tile per lane of the first warp
    __syncwarp();
    append_tiles(s, s_rec, lane, 32);
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
        const int4 w = make_window(cy, cx, s.step_y, s.step_x, s.Hg, s.W);
        s.win[k] = w;
        append_tiles(s, make_cand(k, cy, cx, __longlong_as_double(r[2]), __longlong_as_double(r[3]), __longlong_as_double(r[4]), w), 0, 1);
    } else {
        // 2: the owner found no member, the cluster is dead for good; 0: it was dead already.  (An alive cluster always has
        // exactly one owner, so 0 cannot occur for it.)
        s.win[k] = make_int4(0, 0, 0, 0);
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

// > 0: cap on the tile lists below the sizing of carve (isb_slic_set_tile_cap), so that tests can force the full-scan path
static int g_tile_cap = 0;

static size_t carve(KmState& s, void* ws, size_t bytes, int H, int W, int n, int step_y, int step_x)
{
    WsCarver c(ws, bytes);
    // H here is the height the cluster geometry lives in (the whole image); band callers overwrite the slab fields afterwards
    s.n = n; s.H = H; s.W = W; s.step_y = step_y; s.step_x = step_x;
    s.Hg = H; s.y_off = 0; s.own_lo = 0; s.own_hi = H; s.halo = 0; s.pstride = (size_t)H * W;
    s.cy = c.take<double>(n); s.cx = c.take<double>(n);
    s.c0 = c.take<double>(n); s.c1 = c.take<double>(n); s.c2 = c.take<double>(n);
    s.win = c.take<int4>(n); s.obb = c.take<int4>(n);
    s.maxdc = c.take<unsigned long long>(n);
    // a window is 4 step + 1 wide, so about (TILE + 4 step + 2) / step + 1 centres of the seed grid per axis have a window that
    // meets a tile; one more per axis is the margin for clusters that drift together.  More than that is still exact (k_assign
    // then scans every cluster for the tile), only slower.
    s.ntx = (W + TILE - 1) / TILE;
    s.tcap = ((TILE + 4 * step_y + 2) / step_y + 2) * ((TILE + 4 * step_x + 2) / step_x + 2);
    if (g_tile_cap > 0 && g_tile_cap < s.tcap) s.tcap = g_tile_cap;
    const size_t tiles = (size_t)((H + TILE - 1) / TILE) * s.ntx;   // a band's slab has at most as many tile rows as the image
    s.tile_cnt = c.take<int>(tiles);
    s.tile_cand = c.take<Cand>(tiles * s.tcap);
    return isb_align(c.off);
}

// first sweep: centres from the seed grid, and their records in empty tile lists
static int seed(KmState& s, const double* seeds_yx, cudaStream_t st)
{
    ISB_CUDA_CHECK(cudaMemsetAsync(s.tile_cnt, 0, sizeof(int) * (size_t)((s.Hg + TILE - 1) / TILE) * s.ntx, st));
    k_seed<<<(s.n + 255) / 256, 256, 0, st>>>(s, seeds_yx);
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
    if (int rc = seed(s, seeds_yx, st)) return rc;
    CUtensorMap lab_map;
    memset(&lab_map, 0, sizeof(lab_map));
    const int use_tma = make_lab_map(lab_map, lab_planar, H, W, s.pstride) ? 1 : 0;
    for (int it = 0; it < max_iter; ++it) {
        {
            ProfScope p(ISB_PROF_ASSIGN, st);
            launch_assign(s, lab_map, use_tma, lab_planar, labels, st);
        }
        ISB_LAUNCH_CHECK();
        { ProfScope p(ISB_PROF_UPDATE, st); k_update<false><<<n_seeds, UTHREADS, 0, st>>>(s, lab_planar, labels, nullptr); }
        ISB_LAUNCH_CHECK();
        if (slic_zero) {
            const size_t npx = (size_t)H * W;
            k_slico_max<<<(unsigned)((npx + 255) / 256), 256, 0, st>>>(s, lab_planar, labels);
            ISB_LAUNCH_CHECK();
        }
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
    return seed(s, b->seeds_yx, st);
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
    k_update<true><<<s.n, UTHREADS, 0, st>>>(s, b->lab_slab, b->labels_slab, (long long*)xchg);
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
    return ISB_OK;
}

extern "C" int isb_slic_set_tile_cap(int cap)
{
    ISB_REQUIRE(cap >= 0, "bad tile cap");
    const int prev = g_tile_cap;
    g_tile_cap = cap;
    return prev;
}

extern "C" long long isb_slic_full_scan_tiles(void)
{
    unsigned long long v = 0;
    ISB_CUDA_CHECK(cudaMemcpyFromSymbol(&v, d_full_scans, sizeof(v)));
    return (long long)v;
}
