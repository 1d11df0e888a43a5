// center_detection.cu -- the device half of the reference's object-centre detection (experiments_ovary_centres/
// run_center_candidate_training.py:378-448, run_center_clustering.py:61-83):
//   isb_ring_label_hist  : compute_label_histograms_positions' disc label counts from run-length rows of the label map
//   isb_dbscan           : sklearn.cluster.DBSCAN(eps, min_samples).fit(points).labels_ over 2-D points, and the mean of every cluster
#include "common.cuh"
#include "block_scan.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

// ---------------------------------------------------------------------------------------------------------------------
// Ring label histograms.  The label map is stored as runs per row: row y owns the slots [y * W, y * W + count[y]) of start[] and
// label[], one per maximal run of equal labels, in column order.  A disc row dy of diameter d covers the columns
// [px - w, px + w] with w = floor(sqrt(d^2 - dy^2)) (skimage.morphology.disk(d): dy^2 + dx^2 <= d^2), clipped to the image as
// adjust_bounding_box_crop clips the disc's box; a binary search finds the run holding the first column and the walk adds the
// clipped length of every run up to the last column.  So a disc costs O(d * runs per span) instead of O(d^2) pixel visits.
// ---------------------------------------------------------------------------------------------------------------------
namespace {

constexpr int RUN_THREADS = 256;
constexpr int RING_THREADS = 256;
constexpr int RING_GROUP = 32;                 // diameters counted in one pass over their rows
constexpr int RING_STATIC_SMEM = 1024;         // room for k_ring_hist's static shared arrays (s_row0, s_off: 520 bytes)
// counters of one pass, (nb_labels + 1) per diameter, 8 bytes each: with the static arrays within the default 48 KiB per CTA
constexpr int RING_SMEM = 48 * 1024 - RING_STATIC_SMEM;

__global__ void __launch_bounds__(RUN_THREADS) k_row_runs(const int* __restrict__ segm, int W, int* __restrict__ run_start,
                                                          int* __restrict__ run_label, int* __restrict__ run_count)
{
    const size_t y = blockIdx.x;
    const int* row = segm + y * W;
    int* rs = run_start + y * W;
    int* rl = run_label + y * W;
    const int n = cta_scan_chunks<RUN_THREADS, int>(W, [&](int x) { return (x == 0 || row[x] != row[x - 1]) ? 1 : 0; },
                                                    [&](int x, int excl) {
                                                        const int l = row[x];
                                                        if (x == 0 || l != row[x - 1]) { rs[excl] = x; rl[excl] = l; }
                                                    });
    if (threadIdx.x == 0) run_count[y] = n;
}

// floor(sqrt(r2)) for r2 >= 0: a float root (no double-sqrt slow path, which would cost the kernel a call frame), then an integer
// correction so that w^2 <= r2 < (w + 1)^2 exactly.  The callers keep r2 below the square of the widest useful half-width, so
// the float root is off by a step or two at most.
__device__ __forceinline__ long long isqrt_floor(long long r2)
{
    if (r2 <= 0) return 0;
    const float f = (float)r2;
    long long w = (long long)(f * rsqrtf(f));
    while (w * w > r2) --w;
    while ((w + 1) * (w + 1) <= r2) ++w;
    return w;
}

// one CTA per position.  The diameters go in groups of `group`; the rows of every disc of a group form one flat index range that
// the threads stride through, each row adding its runs' clipped lengths to the group's per-label counters in shared memory.
__global__ void __launch_bounds__(RING_THREADS) k_ring_hist(const int* __restrict__ run_start, const int* __restrict__ run_label,
                                                            const int* __restrict__ run_count, int H, int W, const int* __restrict__ positions,
                                                            const int* __restrict__ diameters, int n_diam, int group, int nb_labels,
                                                            double* __restrict__ hist, double* __restrict__ sizes)
{
    extern __shared__ unsigned long long s_cnt[];          // [group][nb_labels + 1]: label counts, then the disc size
    __shared__ long long s_row0[RING_GROUP];               // first disc row (dy) of each diameter of the group
    __shared__ long long s_off[RING_GROUP + 1];            // flat row offsets of the group's discs
    static_assert(sizeof(s_row0) + sizeof(s_off) <= RING_STATIC_SMEM, "static shared arrays over their share of the 48 KiB");
    const int ip = blockIdx.x;
    const long long py = positions[2 * ip], px = positions[2 * ip + 1];
    const int stride = nb_labels + 1;
    // a half-width of `wcap` already spans the image row: clamping the squared half-width there changes no clipped span
    const long long wcap = min((long long)W + (px < 0 ? -px : px), 3037000499ll), r2cap = wcap * wcap;
    for (int g0 = 0; g0 < n_diam; g0 += group) {
        const int ng = min(group, n_diam - g0);
        for (int i = threadIdx.x; i < ng * stride; i += RING_THREADS) s_cnt[i] = 0ull;
        if (threadIdx.x == 0) {
            long long off = 0;
            for (int g = 0; g < ng; ++g) {
                const long long d = diameters[g0 + g];
                const long long lo = max(-d, -py), hi = min(d, (long long)H - 1 - py);   // disc rows inside the image
                s_row0[g] = lo;
                s_off[g] = off;
                off += hi >= lo ? hi - lo + 1 : 0;
            }
            s_off[ng] = off;
        }
        __syncthreads();
        const long long total = s_off[ng];
        int g = 0;
        for (long long t = threadIdx.x; t < total; t += RING_THREADS) {
            while (t >= s_off[g + 1]) ++g;
            const long long d = diameters[g0 + g];
            const long long dy = s_row0[g] + (t - s_off[g]);
            const long long w = isqrt_floor(min(d * d - dy * dy, r2cap));
            const long long x0 = max(px - w, 0ll), x1 = min(px + w, (long long)W - 1);
            if (x0 > x1) continue;
            unsigned long long* cnt = s_cnt + (size_t)g * stride;
            atomicAdd(&cnt[nb_labels], (unsigned long long)(x1 - x0 + 1));
            const size_t y = (size_t)(py + dy);
            const int* rs = run_start + y * W;
            const int* rl = run_label + y * W;
            const int nr = run_count[y];
            int a = 0, b = nr - 1;                         // the last run starting at or before x0 (run 0 starts at column 0)
            while (a < b) {
                const int m = (a + b + 1) >> 1;
                if (rs[m] <= x0) a = m; else b = m - 1;
            }
            for (int r = a; r < nr && rs[r] <= x1; ++r) {
                const int l = rl[r];
                if (l < 0 || l >= nb_labels) continue;
                const long long s = max((long long)rs[r], x0), e = min(r + 1 < nr ? (long long)rs[r + 1] - 1 : (long long)W - 1, x1);
                atomicAdd(&cnt[l], (unsigned long long)(e - s + 1));
            }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < ng * stride; i += RING_THREADS) {
            const int gi = i / stride, l = i - gi * stride;
            const size_t pd = (size_t)ip * n_diam + g0 + gi;
            if (l < nb_labels) hist[pd * nb_labels + l] = (double)s_cnt[i];
            else sizes[pd] = (double)s_cnt[i];
        }
        __syncthreads();
    }
}

int ring_group(int nb_labels) { return max(1, min(RING_GROUP, RING_SMEM / (int)(sizeof(unsigned long long) * (nb_labels + 1)))); }

} // namespace

extern "C" size_t isb_label_runs_workspace_bytes(int H, int W)
{
    if (H <= 0 || W <= 0) return 0;
    return 2 * isb_align(sizeof(int32_t) * (size_t)H * W) + isb_align(sizeof(int32_t) * (size_t)H) + 1024;
}

extern "C" int isb_ring_label_hist(const int32_t* segm, int H, int W, const int32_t* positions, int n_pos, const int32_t* diameters,
                                   int n_diam, int nb_labels, double* hist, double* sizes, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(segm && positions && diameters && hist && sizes && ws, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && n_pos > 0 && n_diam > 0 && nb_labels > 0 && nb_labels <= 4096, "bad sizes");
    ISB_REQUIRE(ws_bytes >= isb_label_runs_workspace_bytes(H, W), "workspace too small");
    WsCarver c(ws, ws_bytes);
    int* run_start = c.take<int>((size_t)H * W);
    int* run_label = c.take<int>((size_t)H * W);
    int* run_count = c.take<int>(H);
    cudaStream_t st = (cudaStream_t)stream;
    k_row_runs<<<H, RUN_THREADS, 0, st>>>(segm, W, run_start, run_label, run_count);
    ISB_LAUNCH_CHECK();
    const int group = ring_group(nb_labels);
    k_ring_hist<<<n_pos, RING_THREADS, sizeof(unsigned long long) * (size_t)group * (nb_labels + 1), st>>>(
        run_start, run_label, run_count, H, W, positions, diameters, n_diam, group, nb_labels, hist, sizes);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// DBSCAN over 2-D float64 points.  Points are binned into square cells of side eps * (1 + widen) (relative to the bounding box's
// lower corner) and sorted by (cell row, cell column), so that the three cells of a neighbouring cell row are one contiguous range of
// the sorted points.  widen is 2^-20, or more when the box is wider than 2^29 such cells: then the cells grow until 2^29 of them
// span the box, so every cell coordinate stays below 2^30 (30 bits of the sort key) whatever eps and the coordinates are.
// Two points are neighbours when dx * dx + dy * dy <= eps * eps, as scikit-learn's KD-tree decides it (rdist against
// _dist_to_rdist(eps)); the widened cell keeps every such pair in adjacent cells despite the rounding of the binning.  A point with at least min_samples neighbours (itself included) is a core point; core-core neighbours are joined
// by a lock-free union-find whose roots are always the smallest index of their set, so the clusters numbered by their roots are
// numbered as dbscan_inner numbers them (it starts each cluster at its smallest core index).  A non-core point takes the
// smallest cluster of its core neighbours -- the one that dbscan_inner expands first -- or -1.
// ---------------------------------------------------------------------------------------------------------------------
namespace {

constexpr int DB_THREADS = 256;
constexpr int DB_CELL_BITS = 30;               // cell coordinates below 2^30: the binning error stays under the cell's widening

enum { DB_OK = 0, DB_NONFINITE = 1 };

__device__ __forceinline__ unsigned long long f64_order_key(double v)
{
    const unsigned long long u = (unsigned long long)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

__device__ __forceinline__ double f64_from_order_key(unsigned long long k)
{
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// box = order keys of (min x, min y, max x, max y)
__global__ void __launch_bounds__(DB_THREADS) k_db_bbox(const double* __restrict__ pts, int n, unsigned long long* box, int* status)
{
    unsigned long long mx = ~0ull, my = ~0ull, Mx = 0ull, My = 0ull;
    bool bad = false;
    for (int i = blockIdx.x * DB_THREADS + threadIdx.x; i < n; i += gridDim.x * DB_THREADS) {
        const double x = pts[2 * (size_t)i], y = pts[2 * (size_t)i + 1];
        bad |= !isfinite(x) || !isfinite(y);
        const unsigned long long kx = f64_order_key(x), ky = f64_order_key(y);
        mx = min(mx, kx); my = min(my, ky);
        Mx = max(Mx, kx); My = max(My, ky);
    }
    atomicMin(&box[0], mx);
    atomicMin(&box[1], my);
    atomicMax(&box[2], Mx);
    atomicMax(&box[3], My);
    if (bad) atomicOr(&status[1], DB_NONFINITE);
}

// The binning's rounding moves a cell coordinate v < 2^30 by under 2^-21, and a pair within eps lies at most 1 / (1 + widen) cells
// apart, so with widen >= 2^-20 its cell coordinates differ by at most 1.  A box too wide in units of eps (or an infinite cell) only
// makes the cells larger: a coarser grid, never a missed pair.
__global__ void __launch_bounds__(DB_THREADS) k_db_cells(const double* __restrict__ pts, int n, double eps,
                                                         const unsigned long long* __restrict__ box, unsigned long long* __restrict__ keys,
                                                         int* __restrict__ idx)
{
    const int i = blockIdx.x * DB_THREADS + threadIdx.x;
    if (i >= n) return;
    const double x0 = f64_from_order_key(box[0]), y0 = f64_from_order_key(box[1]);
    const double span = __ddiv_rn(fmax(__dsub_rn(f64_from_order_key(box[2]), x0), __dsub_rn(f64_from_order_key(box[3]), y0)), eps);
    const double cell = __dmul_rn(eps, __dadd_rn(1.0, fmax(0x1p-20, __dmul_rn(span, 0x1p-29))));
    const double lim = (double)((1 << DB_CELL_BITS) - 1);
    double cx = 0.0, cy = 0.0;
    if (!isinf(cell)) {
        cx = fmin(fmax(floor(__ddiv_rn(__dsub_rn(pts[2 * (size_t)i], x0), cell)), 0.0), lim);
        cy = fmin(fmax(floor(__ddiv_rn(__dsub_rn(pts[2 * (size_t)i + 1], y0), cell)), 0.0), lim);
    }
    keys[i] = ((unsigned long long)cy << 32) | (unsigned long long)cx;
    idx[i] = i;
}

__global__ void __launch_bounds__(DB_THREADS) k_db_gather(const double* __restrict__ pts, const int* __restrict__ sidx, int n,
                                                          double* __restrict__ sx, double* __restrict__ sy)
{
    const int s = blockIdx.x * DB_THREADS + threadIdx.x;
    if (s >= n) return;
    const size_t i = sidx[s];
    sx[s] = pts[2 * i];
    sy[s] = pts[2 * i + 1];
}

// first sorted position whose key is >= k
__device__ __forceinline__ int lower_bound_u64(const unsigned long long* __restrict__ keys, int n, unsigned long long k)
{
    int a = 0, b = n;
    while (a < b) {
        const int m = (a + b) >> 1;
        if (keys[m] < k) a = m + 1; else b = m;
    }
    return a;
}

__device__ __forceinline__ bool db_close(double xa, double ya, double xb, double yb, double eps2)
{
    const double dx = __dsub_rn(xa, xb), dy = __dsub_rn(ya, yb);
    return __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)) <= eps2;
}

// visit(j) for every sorted position j in the 3 x 3 cells about sorted position s
template <typename Visit>
__device__ __forceinline__ void db_for_neighbour_cells(const unsigned long long* __restrict__ keys, int n, int s, Visit visit)
{
    const unsigned long long k = keys[s];
    const long long cy = (long long)(k >> 32), cx = (long long)(k & 0xffffffffull);
    const unsigned long long xlo = (unsigned long long)max(cx - 1, 0ll), xhi = (unsigned long long)(cx + 2);
    for (long long ry = max(cy - 1, 0ll); ry <= cy + 1; ++ry) {
        const unsigned long long row = (unsigned long long)ry << 32;
        const int b = lower_bound_u64(keys, n, row | xlo), e = lower_bound_u64(keys, n, row | xhi);
        for (int j = b; j < e; ++j) visit(j);
    }
}

__global__ void __launch_bounds__(DB_THREADS) k_db_core(const unsigned long long* __restrict__ keys, const double* __restrict__ sx,
                                                        const double* __restrict__ sy, int n, double eps2, int min_samples,
                                                        unsigned char* __restrict__ core_s)
{
    const int s = blockIdx.x * DB_THREADS + threadIdx.x;
    if (s >= n) return;
    const double x = sx[s], y = sy[s];
    long long cnt = 0;
    db_for_neighbour_cells(keys, n, s, [&](int j) { cnt += db_close(x, y, sx[j], sy[j], eps2); });
    core_s[s] = cnt >= min_samples;
}

// the root of x's set; halves the path on the way (parent[v] <= v always, so the writes only move nodes closer to their root)
__device__ __forceinline__ int uf_root(int* parent, int x)
{
    volatile int* p = parent;
    int cur = p[x];
    if (cur != x) {
        int prev = x, next;
        while (cur > (next = p[cur])) {
            p[prev] = next;
            prev = cur;
            cur = next;
        }
    }
    return cur;
}

// join the sets of a and b: the larger root is hooked under the smaller one, retried when another thread moved it first
__device__ __forceinline__ void uf_union(int* parent, int a, int b)
{
    int ra = uf_root(parent, a), rb = uf_root(parent, b);
    while (ra != rb) {
        if (ra < rb) { const int t = ra; ra = rb; rb = t; }
        const int old = atomicCAS(&parent[ra], ra, rb);
        if (old == ra) return;
        ra = uf_root(parent, old);
        rb = uf_root(parent, rb);
    }
}

__global__ void __launch_bounds__(DB_THREADS) k_db_union(const unsigned long long* __restrict__ keys, const double* __restrict__ sx,
                                                         const double* __restrict__ sy, const int* __restrict__ sidx,
                                                         const unsigned char* __restrict__ core_s, int n, double eps2, int* parent)
{
    const int s = blockIdx.x * DB_THREADS + threadIdx.x;
    if (s >= n || !core_s[s]) return;
    const double x = sx[s], y = sy[s];
    const int i = sidx[s];
    db_for_neighbour_cells(keys, n, s, [&](int j) {
        const int o = sidx[j];
        if (o < i && core_s[j] && db_close(x, y, sx[j], sy[j], eps2)) uf_union(parent, i, o);
    });
}

__global__ void __launch_bounds__(DB_THREADS) k_db_init(int n, int* parent)
{
    const int i = blockIdx.x * DB_THREADS + threadIdx.x;
    if (i < n) parent[i] = i;
}

// root of every core point; root_flag[i] = 1 for the roots (one per cluster), which the scan turns into cluster numbers
__global__ void __launch_bounds__(DB_THREADS) k_db_roots(const int* __restrict__ sidx, const unsigned char* __restrict__ core_s, int n,
                                                         int* parent, int* __restrict__ root_flag)
{
    const int s = blockIdx.x * DB_THREADS + threadIdx.x;
    if (s >= n) return;
    const int i = sidx[s];
    if (!core_s[s]) { root_flag[i] = 0; return; }
    root_flag[i] = uf_root(parent, i) == i;
}

__global__ void __launch_bounds__(DB_THREADS) k_db_labels(const unsigned long long* __restrict__ keys, const double* __restrict__ sx,
                                                          const double* __restrict__ sy, const int* __restrict__ sidx,
                                                          const unsigned char* __restrict__ core_s, int n, double eps2, int* parent,
                                                          const int* __restrict__ rank, int* __restrict__ labels)
{
    const int s = blockIdx.x * DB_THREADS + threadIdx.x;
    if (s >= n) return;
    const int i = sidx[s];
    if (core_s[s]) { labels[i] = rank[uf_root(parent, i)]; return; }
    const double x = sx[s], y = sy[s];
    int best = INT_MAX;                            // smallest root among the core neighbours = smallest cluster number
    db_for_neighbour_cells(keys, n, s, [&](int j) {
        if (core_s[j] && db_close(x, y, sx[j], sy[j], eps2)) best = min(best, uf_root(parent, sidx[j]));
    });
    labels[i] = best == INT_MAX ? -1 : rank[best];
}

__global__ void k_db_count(const int* __restrict__ rank, const int* __restrict__ root_flag, int n, int* status)
{
    status[0] = rank[n - 1] + root_flag[n - 1];
}

__global__ void __launch_bounds__(DB_THREADS) k_db_member_keys(const int* __restrict__ labels, int n, unsigned* __restrict__ keys,
                                                               int* __restrict__ idx)
{
    const int i = blockIdx.x * DB_THREADS + threadIdx.x;
    if (i >= n) return;
    keys[i] = (unsigned)(labels[i] + 1);           // noise first
    idx[i] = i;
}

// mean of every cluster: its members in index order (a stable sort by label), summed one after the other, over the count --
// np.mean(points[labels == c], axis=0), which reduces the rows of a C-ordered array sequentially
__global__ void __launch_bounds__(DB_THREADS) k_db_means(const double* __restrict__ pts, const unsigned* __restrict__ skeys,
                                                         const int* __restrict__ sidx, int n, const int* __restrict__ status,
                                                         double* __restrict__ centres)
{
    const int c = blockIdx.x * DB_THREADS + threadIdx.x;
    if (c >= status[0]) return;
    int a = 0, b = n;
    while (a < b) { const int m = (a + b) >> 1; if (skeys[m] < (unsigned)(c + 1)) a = m + 1; else b = m; }
    double sx = 0.0, sy = 0.0;
    int k = a;
    for (; k < n && skeys[k] == (unsigned)(c + 1); ++k) {
        const size_t i = sidx[k];
        sx = __dadd_rn(sx, pts[2 * i]);
        sy = __dadd_rn(sy, pts[2 * i + 1]);
    }
    const double cnt = (double)(k - a);
    centres[2 * (size_t)c] = __ddiv_rn(sx, cnt);
    centres[2 * (size_t)c + 1] = __ddiv_rn(sy, cnt);
}

struct DbWs {
    unsigned long long *box, *keys, *keys_s;
    int *status, *idx, *sidx, *parent, *root_flag, *rank;
    unsigned *mkeys, *mkeys_s;
    double *sx, *sy;
    unsigned char* core_s;
    void* tmp;
    size_t tmp_bytes;
};

size_t db_tmp_bytes(int n)
{
    size_t a = 0, b = 0, s = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (const int*)nullptr,
                                    (int*)nullptr, n, 0, 32 + DB_CELL_BITS);
    cub::DeviceRadixSort::SortPairs(nullptr, b, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr, n, 0, 32);
    cub::DeviceScan::ExclusiveSum(nullptr, s, (const int*)nullptr, (int*)nullptr, n);
    return max(a, max(b, s));
}

// the workspace's arrays; `used` = the bytes they take
DbWs db_carve(void* ws, size_t ws_bytes, int n, size_t& used)
{
    WsCarver c(ws, ws_bytes);
    DbWs w;
    w.box = c.take<unsigned long long>(4);
    w.status = c.take<int>(2);
    w.keys = c.take<unsigned long long>(n);
    w.keys_s = c.take<unsigned long long>(n);
    w.idx = c.take<int>(n);
    w.sidx = c.take<int>(n);
    w.parent = c.take<int>(n);
    w.root_flag = c.take<int>(n);
    w.rank = c.take<int>(n);
    w.mkeys = c.take<unsigned>(n);
    w.mkeys_s = c.take<unsigned>(n);
    w.sx = c.take<double>(n);
    w.sy = c.take<double>(n);
    w.core_s = c.take<unsigned char>(n);
    w.tmp_bytes = db_tmp_bytes(n);
    w.tmp = c.take<char>(w.tmp_bytes);
    used = c.off;
    return w;
}

} // namespace

extern "C" size_t isb_dbscan_workspace_bytes(int n)
{
    if (n <= 0) return 1024;
    size_t used = 0;
    db_carve(nullptr, 0, n, used);
    return used + 1024;
}

extern "C" int isb_dbscan(const double* points, int n, double eps, int min_samples, int32_t* labels, double* centres,
                          int* n_clusters, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(n_clusters && (n == 0 || (points && labels && ws)), "null pointer");
    ISB_REQUIRE(n >= 0 && min_samples >= 1, "bad sizes");
    ISB_REQUIRE(eps > 0 && eps <= 1.0e300, "eps must be a positive finite number");   // NaN fails too
    *n_clusters = 0;
    if (n == 0) return ISB_OK;
    ISB_REQUIRE(ws_bytes >= isb_dbscan_workspace_bytes(n), "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    size_t used = 0;
    DbWs w = db_carve(ws, ws_bytes, n, used);
    const unsigned blocks = (unsigned)((n + DB_THREADS - 1) / DB_THREADS);
    const double eps2 = eps * eps;
    ISB_CUDA_CHECK(cudaMemsetAsync(w.box, 0xff, 2 * sizeof(unsigned long long), st));
    ISB_CUDA_CHECK(cudaMemsetAsync(w.box + 2, 0, 2 * sizeof(unsigned long long), st));
    ISB_CUDA_CHECK(cudaMemsetAsync(w.status, 0, 2 * sizeof(int), st));
    k_db_bbox<<<min(blocks, 1024u), DB_THREADS, 0, st>>>(points, n, w.box, w.status);
    ISB_LAUNCH_CHECK();
    k_db_cells<<<blocks, DB_THREADS, 0, st>>>(points, n, eps, w.box, w.keys, w.idx);
    ISB_LAUNCH_CHECK();
    size_t tb = w.tmp_bytes;
    ISB_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(w.tmp, tb, w.keys, w.keys_s, w.idx, w.sidx, n, 0, 32 + DB_CELL_BITS, st));
    k_db_gather<<<blocks, DB_THREADS, 0, st>>>(points, w.sidx, n, w.sx, w.sy);
    ISB_LAUNCH_CHECK();
    k_db_core<<<blocks, DB_THREADS, 0, st>>>(w.keys_s, w.sx, w.sy, n, eps2, min_samples, w.core_s);
    ISB_LAUNCH_CHECK();
    k_db_init<<<blocks, DB_THREADS, 0, st>>>(n, w.parent);
    ISB_LAUNCH_CHECK();
    k_db_union<<<blocks, DB_THREADS, 0, st>>>(w.keys_s, w.sx, w.sy, w.sidx, w.core_s, n, eps2, w.parent);
    ISB_LAUNCH_CHECK();
    k_db_roots<<<blocks, DB_THREADS, 0, st>>>(w.sidx, w.core_s, n, w.parent, w.root_flag);
    ISB_LAUNCH_CHECK();
    tb = w.tmp_bytes;
    ISB_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(w.tmp, tb, w.root_flag, w.rank, n, st));
    k_db_labels<<<blocks, DB_THREADS, 0, st>>>(w.keys_s, w.sx, w.sy, w.sidx, w.core_s, n, eps2, w.parent, w.rank, labels);
    ISB_LAUNCH_CHECK();
    k_db_count<<<1, 1, 0, st>>>(w.rank, w.root_flag, n, w.status);
    ISB_LAUNCH_CHECK();
    if (centres) {
        k_db_member_keys<<<blocks, DB_THREADS, 0, st>>>(labels, n, w.mkeys, w.idx);
        ISB_LAUNCH_CHECK();
        tb = w.tmp_bytes;
        ISB_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(w.tmp, tb, w.mkeys, w.mkeys_s, w.idx, w.sidx, n, 0, 32, st));
        k_db_means<<<blocks, DB_THREADS, 0, st>>>(points, w.mkeys_s, w.sidx, n, w.status, centres);
        ISB_LAUNCH_CHECK();
    }
    int host_status[2];
    ISB_CUDA_CHECK(cudaMemcpyAsync(host_status, w.status, sizeof(host_status), cudaMemcpyDeviceToHost, st));
    ISB_CUDA_CHECK(cudaStreamSynchronize(st));
    if (host_status[1] & DB_NONFINITE) {
        isb_set_error("%s:%d the points have to be finite", __FILE__, __LINE__);
        return ISB_ERR_ARG;
    }
    *n_clusters = host_status[0];
    return ISB_OK;
}
