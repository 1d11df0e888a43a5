// forest_fit.cu -- exact-split Gini trees of scikit-learn's DecisionTreeClassifier / RandomForestClassifier (splitter 'best'),
// every tree of a forest built together, level by level.
//
// The trees may belong to G groups (isb_forest_fit_groups): a group is one training set of its own -- its own float32 copy of the n rows
// with D_g of the Dmax columns, its own max_features, min_samples_split and min_samples_leaf -- and every kernel that reads x or one of
// those parameters looks them up through the node's tree and that tree's group.  isb_forest_fit is the one-group call.
//
// Rows are "entries": a (tree, row) pair with a nonzero count (the bootstrap count, or 1).  Each level holds the nodes created by
// the level before (all trees together, in breadth-first order), and the active entries grouped by node.  Per level:
//   k_ff_stats       class counts and weight of every node (integer atomics: the same integers in any order)
//   k_ff_decide      Gini impurity; the depth-first builder's leaf tests that need no split
//   k_ff_nonconst    one min / max pass per (node, feature): a feature is constant at the node when max <= min + 1e-7f
//   k_ff_candidates  the m non-constant features of least (splitmix64 hash of (tree seed, breadth-first index, feature), feature), by a
//                    bitonic sort of the D keys in shared memory
//   k_ff_fill        one (segment, float32 value bits) key per (candidate, row), payload (count << 8 | class)
//   radix sort       all segments at once, on the composite key
//   k_ff_scan        one thread per segment walks its sorted values with integer class counts and sums of squared counts, and
//                    keeps the allowed position of largest proxy improvement (the first one on ties)
//   k_ff_choose      the best candidate of a node (lowest feature on ties), its improvement and the remaining leaf tests
//   k_ff_children    breadth-first ids of the children; k_ff_route sends each entry left when x <= threshold
//   radix sort       the entries of the next level grouped by child
// then the preorder numbering of the depth-first builder from subtree sizes, and one scatter into the caller's arrays.
//
// The FP64 expressions are those of scikit-learn's _criterion.pyx / _splitter.pyx in the same order, and the library is built with
// -fmad=false, so nothing is contracted into an FMA: the impurities, proxies, improvements and thresholds are the same bits as the
// oracle's (oracle/forest.py).  Class counts are integers below 2^26 per tree, so every sum of squared counts is exact in float64.
#include "common.cuh"
#include "tree_split.cuh"
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <vector>

namespace {

constexpr int FF_CMAX = (1 << 24) - 1;       // count of one row (24 bits of the sort payload)
constexpr int TB = 256;

inline int bits_for(unsigned long long v)   // bits to hold 0..v
{
    int b = 1;
    while (b < 64 && (v >> b)) ++b;
    return b;
}
inline int blocks_of(long long n, int t = TB) { return (int)((n + t - 1) / t); }

__host__ __device__ __forceinline__ unsigned long long splitmix64(unsigned long long z)
{
    z += 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

__device__ __forceinline__ unsigned f32_ordered(float v)
{
    const unsigned u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float f32_unordered(unsigned o)
{
    return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

// the groups as the kernels read them: x [G, n, Dmax] and, per tree, its group; per group its columns and parameters
struct FfGroups {
    const float* x;
    long long n;
    int Dmax;
    const int32_t* tree_group;                      // [T]
    const int32_t *D, *m, *mss, *msl;               // [G] each
    __device__ __forceinline__ int of_tree(int t) const { return tree_group[t]; }
    __device__ __forceinline__ const float* rows(int q) const { return x + (size_t)q * n * Dmax; }
};

struct FfWs {
    // entries
    int32_t *e_row, *e_tree, *e_node;
    uint32_t* e_pay;
    uint32_t *g_key, *g_key2, *g_idx, *g_idx2;     // grouped order of the active entries
    int32_t* flag_pos;                              // [T * n + 1] scan of the nonzero counts
    // nodes (breadth-first, all trees)
    int32_t *nd_tree, *nd_depth, *nd_left, *nd_right, *nd_feature, *nd_rows, *nd_split, *nd_mgl, *nd_size, *nd_pre, *nd_cc;
    unsigned long long *nd_local, *nd_w;
    double *nd_imp, *nd_thr;
    // per level
    int32_t *lv_rows, *lv_start, *lv_ncand, *lv_segoff, *lv_rank, *lv_flag, *cand;
    long long *lv_nelem, *lv_elemoff;
    uint32_t* nc_bits;
    // elements and segments
    unsigned long long *k_in, *k_out;
    uint32_t *p_in, *p_out;
    double *s_proxy, *s_thr, *s_wl;
    unsigned long long *s_sql, *s_sqr;
    int32_t* s_pos;
    // per tree, and the values read back
    unsigned long long *t_seed, *t_w, *t_next;
    int32_t *t_nnz, *t_first, *t_nsplit;
    int32_t* grp;                                   // tree_group [T], then D, m, mss, msl [G] each
    long long* info;                                // [0] error flags, [1] entries, [2] elements, [3] segments, [4] splits, [5] next entries
    void* tmp;
    size_t tmp_bytes, need;
};

FfWs carve(void* base, int n, int D, int T, int K, int m, int G)
{
    // E entries; NN nodes of all trees; M elements of a level (each entry in one node, m candidates); S segments of a level: they are
    // numbered over the splittable nodes only, which hold >= 2 entries each, so at most E / 2 of them
    const long long E = (long long)T * n, NN = 2 * E, M = E * m, S = (E / 2 + 1) * m;
    const int W = (D + 31) / 32;
    WsCarver c(base, ~size_t(0));
    FfWs w;
    w.e_row = c.take<int32_t>(E); w.e_tree = c.take<int32_t>(E); w.e_node = c.take<int32_t>(E); w.e_pay = c.take<uint32_t>(E);
    w.g_key = c.take<uint32_t>(E); w.g_key2 = c.take<uint32_t>(E); w.g_idx = c.take<uint32_t>(E); w.g_idx2 = c.take<uint32_t>(E);
    w.flag_pos = c.take<int32_t>(E + 1);
    w.nd_tree = c.take<int32_t>(NN); w.nd_depth = c.take<int32_t>(NN); w.nd_left = c.take<int32_t>(NN); w.nd_right = c.take<int32_t>(NN);
    w.nd_feature = c.take<int32_t>(NN); w.nd_rows = c.take<int32_t>(NN); w.nd_split = c.take<int32_t>(NN); w.nd_mgl = c.take<int32_t>(NN);
    w.nd_size = c.take<int32_t>(NN); w.nd_pre = c.take<int32_t>(NN); w.nd_cc = c.take<int32_t>(NN * K);
    w.nd_local = c.take<unsigned long long>(NN); w.nd_w = c.take<unsigned long long>(NN);
    w.nd_imp = c.take<double>(NN); w.nd_thr = c.take<double>(NN);
    w.lv_rows = c.take<int32_t>(E + 1); w.lv_start = c.take<int32_t>(E + 1); w.lv_ncand = c.take<int32_t>(E + 1);
    w.lv_segoff = c.take<int32_t>(E + 1); w.lv_rank = c.take<int32_t>(E + 1); w.lv_flag = c.take<int32_t>(E + 1);
    w.cand = c.take<int32_t>((E + 1) * m);           // indexed by the node's position in its level: up to E nodes
    w.lv_nelem = c.take<long long>(E + 1); w.lv_elemoff = c.take<long long>(E + 1);
    w.nc_bits = c.take<uint32_t>((E + 1) * W);
    w.k_in = c.take<unsigned long long>(M); w.k_out = c.take<unsigned long long>(M);
    w.p_in = c.take<uint32_t>(M); w.p_out = c.take<uint32_t>(M);
    w.s_proxy = c.take<double>(S); w.s_thr = c.take<double>(S); w.s_wl = c.take<double>(S);
    w.s_sql = c.take<unsigned long long>(S); w.s_sqr = c.take<unsigned long long>(S); w.s_pos = c.take<int32_t>(S);
    w.t_seed = c.take<unsigned long long>(T); w.t_w = c.take<unsigned long long>(T); w.t_next = c.take<unsigned long long>(T);
    w.t_nnz = c.take<int32_t>(T); w.t_first = c.take<int32_t>(T); w.t_nsplit = c.take<int32_t>(T);
    w.grp = c.take<int32_t>(T + 4ll * G);
    w.info = c.take<long long>(8);
    size_t a = 0, b = 0, s1 = 0, s2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (const uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)M, 0, 64);
    cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (int)E, 0, 32);
    cub::DeviceScan::ExclusiveSum(nullptr, s1, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(E + 1));
    cub::DeviceScan::ExclusiveSum(nullptr, s2, (const long long*)nullptr, (long long*)nullptr, (int)(E + 1));
    w.tmp_bytes = std::max(std::max(a, b), std::max(s1, s2));
    w.tmp = c.take<char>(w.tmp_bytes);
    w.need = c.off;
    return w;
}

// ---- set-up ----

__global__ void k_ff_flags(const int32_t* __restrict__ y, int K, const int32_t* __restrict__ counts, int n, int T, int32_t* __restrict__ flag,
                           int32_t* __restrict__ t_nnz, unsigned long long* __restrict__ t_w, long long* __restrict__ info)
{
    const long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (q >= (long long)T * n) {
        if (q == (long long)T * n) flag[q] = 0;
        return;
    }
    const int t = (int)(q / n), r = (int)(q % n);
    const int cnt = counts[q];
    flag[q] = cnt > 0;
    if (cnt < 0) atomicOr((unsigned long long*)info, 1ull);
    if (cnt > FF_CMAX) atomicOr((unsigned long long*)info, 2ull);
    if (t == 0 && (y[r] < 0 || y[r] >= K)) atomicOr((unsigned long long*)info, 4ull);
    if (cnt > 0) {
        atomicAdd(t_nnz + t, 1);
        atomicAdd(t_w + t, (unsigned long long)cnt);
    }
}

__global__ void k_ff_entries(const int32_t* __restrict__ y, const int32_t* __restrict__ counts, int n, int T, const int32_t* __restrict__ pos,
                             int32_t* __restrict__ e_row, int32_t* __restrict__ e_tree, int32_t* __restrict__ e_node, uint32_t* __restrict__ e_pay,
                             uint32_t* __restrict__ g_idx)
{
    const long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (q >= (long long)T * n) return;
    const int cnt = counts[q];
    if (cnt <= 0) return;
    const int t = (int)(q / n), r = (int)(q % n), e = pos[q];
    e_row[e] = r;
    e_tree[e] = t;
    e_node[e] = t;                                      // the root of tree t is node t
    e_pay[e] = ((uint32_t)cnt << 8) | (uint32_t)min(max(y[r], 0), 255);
    g_idx[e] = (uint32_t)e;                             // entries of a tree are contiguous: grouped by root already
}

__global__ void k_ff_init_nodes(int L0, int L1, int K, int32_t* __restrict__ nd_rows, unsigned long long* __restrict__ nd_w, int32_t* __restrict__ nd_cc)
{
    const long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const long long nl = L1 - L0;
    if (q >= nl * (K + 1)) return;
    if (q < nl) {
        nd_rows[L0 + q] = 0;
        nd_w[L0 + q] = 0;
    } else {
        nd_cc[(size_t)L0 * K + (q - nl)] = 0;
    }
}

__global__ void k_ff_roots(int T, int32_t* __restrict__ nd_tree, int32_t* __restrict__ nd_depth, unsigned long long* __restrict__ nd_local,
                           unsigned long long* __restrict__ t_next, int32_t* __restrict__ t_first, int32_t* __restrict__ t_nsplit)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    nd_tree[t] = t;
    nd_depth[t] = 0;
    nd_local[t] = 0;
    t_next[t] = 1;
    t_first[t] = 0x7fffffff;
    t_nsplit[t] = 0;
}

// ---- one level ----

// class counts, rows and weight of the level's nodes from the active entries
__global__ void k_ff_stats(const uint32_t* __restrict__ g_idx, int n_active, const int32_t* __restrict__ e_node, const uint32_t* __restrict__ e_pay,
                           int K, int32_t* __restrict__ nd_cc, int32_t* __restrict__ nd_rows, unsigned long long* __restrict__ nd_w)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_active) return;
    const int e = (int)g_idx[i];
    const int node = e_node[e];
    if (node < 0) return;
    const uint32_t pay = e_pay[e];
    atomicAdd(nd_cc + (size_t)node * K + (pay & 0xff), (int)(pay >> 8));
    atomicAdd(nd_rows + node, 1);
    atomicAdd(nd_w + node, (unsigned long long)(pay >> 8));
}

// impurity, and the leaf tests of the depth-first builder that come before node_split
__global__ void k_ff_decide(int L0, int nl, int K, const int32_t* __restrict__ nd_cc, const int32_t* __restrict__ nd_rows,
                            const unsigned long long* __restrict__ nd_w, const int32_t* __restrict__ nd_depth, const int32_t* __restrict__ nd_tree,
                            int max_depth, FfGroups gr, double* __restrict__ nd_imp, int32_t* __restrict__ nd_split, int32_t* __restrict__ lv_rows)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > nl) return;
    if (i == nl) { lv_rows[nl] = 0; return; }
    const int g = L0 + i;
    unsigned long long sq = 0;
    for (int c = 0; c < K; ++c) {
        const unsigned long long v = (unsigned long long)nd_cc[(size_t)g * K + c];
        sq += v * v;
    }
    const double imp = gini_of(sq, (double)nd_w[g]);
    nd_imp[g] = imp;
    const int rows = nd_rows[g];
    const int q = gr.of_tree(nd_tree[g]), mss = gr.mss[q], msl = gr.msl[q];
    const bool leaf = (max_depth >= 0 && nd_depth[g] >= max_depth) || rows < mss || rows < 2 * msl || imp <= FF_EPSILON;
    nd_split[g] = leaf ? 0 : 1;
    lv_rows[i] = rows;
}

// non-constant bits: block (node, 32-feature word); lanes are features (coalesced rows of x), warps stride the node's rows
constexpr int NC_WARPS = 4;
__global__ void __launch_bounds__(NC_WARPS * 32)
k_ff_nonconst(FfGroups gr, int L0, const int32_t* __restrict__ nd_split, const int32_t* __restrict__ nd_tree, const int32_t* __restrict__ lv_start,
              const uint32_t* __restrict__ g_idx, const int32_t* __restrict__ e_row, uint32_t* __restrict__ nc_bits, int W)
{
    const int i = blockIdx.x, word = blockIdx.y;
    if (!nd_split[L0 + i]) return;
    const int grp = gr.of_tree(nd_tree[L0 + i]), D = gr.D[grp];
    if (word * 32 >= D) return;                         // words past the group's columns are never read
    const float* x = gr.rows(grp);
    const int Dmax = gr.Dmax;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int f = word * 32 + lane;
    const int b = lv_start[i], e = lv_start[i + 1];
    float lo = __int_as_float(0x7f800000), hi = -__int_as_float(0x7f800000);
    if (f < D) {
        for (int q = b + warp; q < e; q += NC_WARPS) {
            const float v = x[(size_t)e_row[g_idx[q]] * Dmax + f];
            lo = fminf(lo, v);
            hi = fmaxf(hi, v);
        }
    }
    __shared__ float s_lo[NC_WARPS][32], s_hi[NC_WARPS][32];
    s_lo[warp][lane] = lo;
    s_hi[warp][lane] = hi;
    __syncthreads();
    if (warp == 0) {
        for (int w = 1; w < NC_WARPS; ++w) {
            lo = fminf(lo, s_lo[w][lane]);
            hi = fmaxf(hi, s_hi[w][lane]);
        }
        const bool nonconst = f < D && !(hi <= __fadd_rn(lo, FEATURE_THRESHOLD));
        const unsigned bits = __ballot_sync(0xffffffffu, nonconst);
        if (lane == 0) nc_bits[(size_t)i * W + word] = bits;
    }
}

// candidate features of every splittable node, ascending feature index; lv_ncand = their number, lv_nelem = rows * candidates
constexpr int CAND_THREADS = 128;
__global__ void __launch_bounds__(CAND_THREADS)
k_ff_candidates(FfGroups gr, int W, int L0, int nl, int32_t* __restrict__ nd_split, const int32_t* __restrict__ nd_tree,
                const unsigned long long* __restrict__ nd_local, const unsigned long long* __restrict__ t_seed, const uint32_t* __restrict__ nc_bits,
                const int32_t* __restrict__ nd_rows, int32_t* __restrict__ lv_ncand, long long* __restrict__ lv_nelem, int32_t* __restrict__ cand,
                int cand_stride)
{
    const int i = blockIdx.x;
    if (i == nl) {                                      // the extra block: trailing zeros of the scans
        if (threadIdx.x == 0) { lv_ncand[nl] = 0; lv_nelem[nl] = 0; }
        return;
    }
    const int g = L0 + i;
    if (!nd_split[g]) {
        if (threadIdx.x == 0) { lv_ncand[i] = 0; lv_nelem[i] = 0; }
        return;
    }
    __shared__ unsigned long long s_hash[FF_DMAX];
    __shared__ unsigned char s_sel[FF_DMAX];
    __shared__ int s_count;
    const int grp = gr.of_tree(nd_tree[g]), D = gr.D[grp], m = gr.m[grp];
    const uint32_t* bits = nc_bits + (size_t)i * W;
    const unsigned long long key = splitmix64(splitmix64(t_seed[nd_tree[g]]) ^ nd_local[g]);
    int mine = 0;
    for (int f = threadIdx.x; f < D; f += CAND_THREADS) {
        const bool nc = (bits[f >> 5] >> (f & 31)) & 1u;
        s_hash[f] = splitmix64(key ^ (unsigned long long)f);
        s_sel[f] = nc;
        mine += nc;
    }
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    atomicAdd(&s_count, mine);
    __syncthreads();
    const int nnc = s_count;
    if (nnc > m) {
        // keep the m non-constant features of least (hash, feature): a bitonic sort of the (class, hash, feature) keys in shared memory,
        // class 0 for the non-constant features and 1 for the rest, O(P log^2 P) with P the power of two at or above D
        __shared__ unsigned short s_idx[FF_DMAX];
        int P = 1;
        while (P < D) P <<= 1;
        for (int q = threadIdx.x; q < P; q += CAND_THREADS) s_idx[q] = (unsigned short)q;
        __syncthreads();
        auto before = [&](int a, int b) {               // key of feature a < key of feature b
            const int ca = !(a < D && s_sel[a]), cb = !(b < D && s_sel[b]);
            if (ca != cb) return ca < cb;
            if (ca) return a < b;
            return s_hash[a] < s_hash[b] || (s_hash[a] == s_hash[b] && a < b);
        };
        for (int k = 2; k <= P; k <<= 1)
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int q = threadIdx.x; q < P; q += CAND_THREADS) {
                    const int r = q ^ j;
                    if (r > q) {
                        const int a = s_idx[q], b = s_idx[r];
                        const bool up = (q & k) == 0;
                        if (up ? before(b, a) : before(a, b)) { s_idx[q] = (unsigned short)b; s_idx[r] = (unsigned short)a; }
                    }
                }
                __syncthreads();
            }
        // the first m sorted slots are the candidates; s_sel is rewritten only after every read of the sort
        int keep[FF_DMAX / CAND_THREADS];
        int nk = 0;
        for (int q = threadIdx.x; q < m; q += CAND_THREADS) keep[nk++] = s_idx[q];
        __syncthreads();
        for (int f = threadIdx.x; f < D; f += CAND_THREADS) s_sel[f] = 0;
        __syncthreads();
        for (int u = 0; u < nk; ++u) s_sel[keep[u]] = 1;
        __syncthreads();
    }
    const int c = nnc < m ? nnc : m;
    // the selected features in ascending order
    using Scan = cub::BlockScan<int, CAND_THREADS>;
    __shared__ typename Scan::TempStorage scan_tmp;
    int base = 0;
    int32_t* out = cand + (size_t)i * cand_stride;
    for (int f0 = 0; f0 < D; f0 += CAND_THREADS) {
        const int f = f0 + threadIdx.x;
        const int sel = f < D ? s_sel[f] : 0;
        int pos, tot;
        Scan(scan_tmp).ExclusiveSum(sel, pos, tot);
        if (sel) out[base + pos] = f;
        base += tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        lv_ncand[i] = c;
        lv_nelem[i] = (long long)c * nd_rows[g];
        if (c == 0) nd_split[g] = 0;                    // every feature constant: split.pos == end
    }
}

__device__ __forceinline__ int upper_index(const long long* off, int n, long long v)   // last i in [0, n) with off[i] <= v
{
    int lo = 0, hi = n;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (off[mid] <= v) lo = mid;
        else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ int upper_index32(const int32_t* off, int n, int v)
{
    int lo = 0, hi = n;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (off[mid] <= v) lo = mid;
        else hi = mid;
    }
    return lo;
}

// one (segment, ordered value) key per (candidate j, row) of every node; element layout = node, candidate, row
__global__ void k_ff_fill(FfGroups gr, const int32_t* __restrict__ nd_tree, int L0, int nl, long long n_elem, const long long* __restrict__ lv_elemoff,
                          const int32_t* __restrict__ lv_segoff, const int32_t* __restrict__ lv_start, const int32_t* __restrict__ nd_rows,
                          const int32_t* __restrict__ cand, int cand_stride, const uint32_t* __restrict__ g_idx, const int32_t* __restrict__ e_row,
                          const uint32_t* __restrict__ e_pay, unsigned long long* __restrict__ k_in, uint32_t* __restrict__ p_in)
{
    for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < n_elem; q += (long long)gridDim.x * blockDim.x) {
        const int i = upper_index(lv_elemoff, nl, q);
        const int rows = nd_rows[L0 + i];
        const long long r = q - lv_elemoff[i];
        const int j = (int)(r / rows), k = (int)(r % rows);
        const int e = (int)g_idx[lv_start[i] + k];
        const int f = cand[(size_t)i * cand_stride + j];
        const float* x = gr.rows(gr.of_tree(nd_tree[L0 + i]));
        k_in[q] = ((unsigned long long)(lv_segoff[i] + j) << 32) | f32_ordered(x[(size_t)e_row[e] * gr.Dmax + f]);
        p_in[q] = e_pay[e];
    }
}

// one thread per segment: the allowed position of largest proxy improvement, the first one on ties (the strict > of node_split_best)
__global__ void k_ff_scan(int L0, int nl, int n_seg, int K, FfGroups gr, const int32_t* __restrict__ nd_tree, const int32_t* __restrict__ lv_segoff, const long long* __restrict__ lv_elemoff,
                          const int32_t* __restrict__ nd_rows, const int32_t* __restrict__ nd_cc, const unsigned long long* __restrict__ nd_w,
                          const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ pay, double* __restrict__ s_proxy,
                          int32_t* __restrict__ s_pos, double* __restrict__ s_thr, double* __restrict__ s_wl, unsigned long long* __restrict__ s_sql,
                          unsigned long long* __restrict__ s_sqr)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seg) return;
    const int i = upper_index32(lv_segoff, nl, s);
    const int g = L0 + i, rows = nd_rows[g], msl = gr.msl[gr.of_tree(nd_tree[g])];
    const long long b = lv_elemoff[i] + (long long)(s - lv_segoff[i]) * rows;
    const int32_t* tot = nd_cc + (size_t)g * K;
    int left[FF_KMAX];
    unsigned long long sql = 0, sqr = 0;
    for (int c = 0; c < K; ++c) {
        left[c] = 0;
        sqr += (unsigned long long)tot[c] * (unsigned long long)tot[c];
    }
    const unsigned long long wtot = nd_w[g];
    unsigned long long wl = 0;
    double best = -__longlong_as_double(0x7ff0000000000000ll), bthr = 0.0, bwl = 0.0;
    unsigned long long bsql = 0, bsqr = 0;
    int bpos = rows;
    float cur = f32_unordered((unsigned)keys[b]);
    for (int p = 1; p < rows; ++p) {
        const uint32_t pl = pay[b + p - 1];
        const int c = pl & 0xff;
        const unsigned long long w = pl >> 8;
        const unsigned long long lc = (unsigned long long)left[c], rc = (unsigned long long)(tot[c] - left[c]);
        sql += 2ull * lc * w + w * w;                   // (lc + w)^2 - lc^2
        sqr -= 2ull * rc * w - w * w;                   // (rc - w)^2 - rc^2
        left[c] += (int)w;
        wl += w;
        const float nxt = f32_unordered((unsigned)keys[b + p]);
        const float prev = cur;
        cur = nxt;
        if (nxt <= __fadd_rn(prev, FEATURE_THRESHOLD)) continue;       // _partitioner.next_p skips ties
        if (p < msl || rows - p < msl) continue;
        const double dwl = (double)wl, dwr = (double)(wtot - wl);
        const double proxy = gini_proxy(sql, dwl, sqr, dwr);
        if (proxy > best) {
            best = proxy;
            bpos = p;
            bthr = (double)prev / 2.0 + (double)nxt / 2.0;
            bwl = dwl;
            bsql = sql;
            bsqr = sqr;
        }
    }
    s_proxy[s] = best;
    s_pos[s] = bpos;
    s_thr[s] = bthr;
    s_wl[s] = bwl;
    s_sql[s] = bsql;
    s_sqr[s] = bsqr;
}

// the best candidate of each node (lowest feature index on equal proxies), the improvement, and the last leaf tests
__global__ void k_ff_choose(int L0, int nl, const int32_t* __restrict__ lv_ncand, const int32_t* __restrict__ lv_segoff, const int32_t* __restrict__ cand,
                            int cand_stride, const double* __restrict__ s_proxy, const int32_t* __restrict__ s_pos, const double* __restrict__ s_thr,
                            const double* __restrict__ s_wl, const unsigned long long* __restrict__ s_sql, const unsigned long long* __restrict__ s_sqr,
                            const int32_t* __restrict__ nd_tree, const int32_t* __restrict__ nd_rows, const unsigned long long* __restrict__ nd_w,
                            const double* __restrict__ nd_imp, const unsigned long long* __restrict__ t_w, double min_impurity_decrease,
                            int32_t* __restrict__ nd_split, int32_t* __restrict__ nd_feature, double* __restrict__ nd_thr, int32_t* __restrict__ nd_mgl,
                            int32_t* __restrict__ lv_flag, long long* __restrict__ info)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > nl) return;
    if (i == nl) { lv_flag[nl] = 0; return; }
    const int g = L0 + i;
    lv_flag[i] = 0;
    if (!nd_split[g]) return;
    const int c = lv_ncand[i], s0 = lv_segoff[i], rows = nd_rows[g];
    int bj = -1;
    double best = -__longlong_as_double(0x7ff0000000000000ll);
    for (int j = 0; j < c; ++j)
        if (s_pos[s0 + j] < rows && s_proxy[s0 + j] > best) { best = s_proxy[s0 + j]; bj = j; }
    if (bj < 0) { nd_split[g] = 0; return; }                           // split.pos >= end
    const int s = s0 + bj;
    const double wn = (double)nd_w[g], wl = s_wl[s], wr = wn - wl;
    const double il = gini_of(s_sql[s], wl), ir = gini_of(s_sqr[s], wr);
    const double improvement = impurity_improvement(wn, (double)t_w[nd_tree[g]], nd_imp[g], wl, il, ir);
    if (improvement + FF_EPSILON < min_impurity_decrease) { nd_split[g] = 0; return; }
    const int n_left = s_pos[s];
    nd_feature[g] = cand[(size_t)i * cand_stride + bj];
    nd_thr[g] = s_thr[s];
    nd_mgl[g] = n_left > rows - n_left;
    lv_flag[i] = 1;
    atomicAdd((unsigned long long*)(info + 5), (unsigned long long)rows);   // entries of the next level
}

__global__ void k_ff_tree_first(int L0, int nl, const int32_t* __restrict__ lv_flag, const int32_t* __restrict__ lv_rank,
                                const int32_t* __restrict__ nd_tree, int32_t* __restrict__ t_first, int32_t* __restrict__ t_nsplit)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nl || !lv_flag[i]) return;
    const int t = nd_tree[L0 + i];
    atomicMin(t_first + t, lv_rank[i]);
    atomicAdd(t_nsplit + t, 1);
}

// children of the splitting nodes: global ids L1 + 2 rank (+1 right), breadth-first index within the tree
__global__ void k_ff_children(int L0, int L1, int nl, const int32_t* __restrict__ lv_flag, const int32_t* __restrict__ lv_rank,
                              const int32_t* __restrict__ t_first, const unsigned long long* __restrict__ t_next, int32_t* __restrict__ nd_tree,
                              int32_t* __restrict__ nd_depth, unsigned long long* __restrict__ nd_local, int32_t* __restrict__ nd_left,
                              int32_t* __restrict__ nd_right)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nl) return;
    const int g = L0 + i;
    if (!lv_flag[i]) {
        nd_left[g] = nd_right[g] = -1;
        return;
    }
    const int r = lv_rank[i], t = nd_tree[g];
    const int lc = L1 + 2 * r;
    const unsigned long long loc = t_next[t] + 2ull * (unsigned long long)(r - t_first[t]);
    nd_left[g] = lc;
    nd_right[g] = lc + 1;
    for (int h = 0; h < 2; ++h) {
        nd_tree[lc + h] = t;
        nd_depth[lc + h] = nd_depth[g] + 1;
        nd_local[lc + h] = loc + h;
    }
}

__global__ void k_ff_tree_advance(int T, unsigned long long* __restrict__ t_next, int32_t* __restrict__ t_first, int32_t* __restrict__ t_nsplit)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    t_next[t] += 2ull * (unsigned long long)t_nsplit[t];
    t_first[t] = 0x7fffffff;
    t_nsplit[t] = 0;
}

// each active entry to its child (x <= threshold goes left, as DecisionTreeClassifier.apply); entries of leaves leave the build
__global__ void k_ff_route(FfGroups gr, const int32_t* __restrict__ nd_tree, int L1, int n_child, const uint32_t* __restrict__ g_idx, int n_active,
                           int32_t* __restrict__ e_node, const int32_t* __restrict__ e_row, const int32_t* __restrict__ nd_split,
                           const int32_t* __restrict__ nd_feature, const double* __restrict__ nd_thr, const int32_t* __restrict__ nd_left,
                           uint32_t* __restrict__ g_key, uint32_t* __restrict__ g_val)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_active) return;
    const int e = (int)g_idx[i];
    const int node = e_node[e];
    int child = -1;
    if (node >= 0 && nd_split[node]) {
        const float v = gr.rows(gr.of_tree(nd_tree[node]))[(size_t)e_row[e] * gr.Dmax + nd_feature[node]];
        child = nd_left[node] + ((double)v <= nd_thr[node] ? 0 : 1);
    }
    e_node[e] = child;
    g_key[i] = child < 0 ? (uint32_t)n_child : (uint32_t)(child - L1);
    g_val[i] = (uint32_t)e;
}

// ---- preorder numbering and output ----

__global__ void k_ff_size(int L0, int nl, const int32_t* __restrict__ nd_split, const int32_t* __restrict__ nd_left,
                          const int32_t* __restrict__ nd_right, int32_t* __restrict__ nd_size)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nl) return;
    const int g = L0 + i;
    nd_size[g] = 1 + (nd_split[g] ? nd_size[nd_left[g]] + nd_size[nd_right[g]] : 0);
}

__global__ void k_ff_pre(int L0, int nl, const int32_t* __restrict__ nd_split, const int32_t* __restrict__ nd_left,
                         const int32_t* __restrict__ nd_right, const int32_t* __restrict__ nd_size, int32_t* __restrict__ nd_pre)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nl) return;
    const int g = L0 + i;
    if (L0 == 0) nd_pre[g] = 0;                         // the roots
    if (!nd_split[g]) return;
    nd_pre[nd_left[g]] = nd_pre[g] + 1;
    nd_pre[nd_right[g]] = nd_pre[g] + 1 + nd_size[nd_left[g]];
}

__global__ void k_ff_write(int n_nodes, int T, int K, int cap, const int32_t* __restrict__ nd_tree, const int32_t* __restrict__ nd_pre,
                           const int32_t* __restrict__ nd_split, const int32_t* __restrict__ nd_left, const int32_t* __restrict__ nd_right,
                           const int32_t* __restrict__ nd_feature, const double* __restrict__ nd_thr, const double* __restrict__ nd_imp,
                           const int32_t* __restrict__ nd_rows, const unsigned long long* __restrict__ nd_w, const int32_t* __restrict__ nd_mgl,
                           const int32_t* __restrict__ nd_cc, const int32_t* __restrict__ nd_size, int32_t* __restrict__ left, int32_t* __restrict__ right,
                           int32_t* __restrict__ feature, double* __restrict__ threshold, double* __restrict__ impurity, int32_t* __restrict__ n_node_samples,
                           double* __restrict__ weighted_n_node_samples, uint8_t* __restrict__ missing_go_to_left, int32_t* __restrict__ class_counts,
                           int32_t* __restrict__ node_count)
{
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_nodes) return;
    const int t = nd_tree[g];
    const size_t o = (size_t)t * cap + nd_pre[g];
    const bool split = nd_split[g];
    left[o] = split ? nd_pre[nd_left[g]] : -1;          // _TREE_LEAF
    right[o] = split ? nd_pre[nd_right[g]] : -1;
    feature[o] = split ? nd_feature[g] : -2;            // _TREE_UNDEFINED
    threshold[o] = split ? nd_thr[g] : -2.0;
    impurity[o] = nd_imp[g];
    n_node_samples[o] = nd_rows[g];
    weighted_n_node_samples[o] = (double)nd_w[g];
    missing_go_to_left[o] = split ? (uint8_t)nd_mgl[g] : 0;
    for (int c = 0; c < K; ++c) class_counts[o * K + c] = nd_cc[(size_t)g * K + c];
    if (g < T) node_count[g] = nd_size[g];
}

int check_sizes(int n, int D, int T, int K, int m)
{
    ISB_REQUIRE(n >= 1 && D >= 1 && T >= 1 && K >= 1, "need n, D, T, K >= 1");
    ISB_REQUIRE(m >= 1 && m <= D, "max_features must be in [1, D]");
    const long long E = (long long)T * n;
    if (K > FF_KMAX || D > FF_DMAX || 2 * E >= (1ll << 31) || E * m >= (1ll << 31) || E >= (1ll << 30)) {
        isb_set_error("forest fit of %d trees over %d rows x %d features, %d classes, max_features %d: at most %d classes, %d features, "
                      "and trees x rows x max_features below 2^31", T, n, D, K, m, FF_KMAX, FF_DMAX);
        return ISB_ERR_UNSUPPORTED;
    }
    return ISB_OK;
}

template <typename T>
int read_back(T* host, const T* dev, size_t n, cudaStream_t st)
{
    ISB_CUDA_CHECK(cudaMemcpyAsync(host, dev, n * sizeof(T), cudaMemcpyDeviceToHost, st));
    ISB_CUDA_CHECK(cudaStreamSynchronize(st));
    return ISB_OK;
}

// the per-group parameters and the trees' groups (host arrays): ISB_ERR_ARG before any device work
int check_groups(int Dmax, int G, const int32_t* D, const int32_t* m, const int32_t* mss, const int32_t* msl, int T, const int32_t* tree_group)
{
    ISB_REQUIRE(G >= 1 && D && m && mss && msl && tree_group, "need G >= 1 and the per-group and per-tree arrays");
    for (int q = 0; q < G; ++q) {
        if (D[q] < 1 || D[q] > Dmax) { isb_set_error("group %d has %d features, not in [1, Dmax = %d]", q, D[q], Dmax); return ISB_ERR_ARG; }
        if (m[q] < 1 || m[q] > D[q]) { isb_set_error("group %d: max_features %d not in [1, %d]", q, m[q], D[q]); return ISB_ERR_ARG; }
        if (mss[q] < 2 || msl[q] < 1) { isb_set_error("group %d: min_samples_split %d < 2 or min_samples_leaf %d < 1", q, mss[q], msl[q]); return ISB_ERR_ARG; }
    }
    for (int t = 0; t < T; ++t)
        if (tree_group[t] < 0 || tree_group[t] >= G) { isb_set_error("tree %d: group %d not in [0, %d)", t, tree_group[t], G); return ISB_ERR_ARG; }
    return ISB_OK;
}

int max_of(const int32_t* v, int n)
{
    int r = v[0];
    for (int i = 1; i < n; ++i) r = std::max(r, (int)v[i]);
    return r;
}

// the level loop of both entry points, over validated arguments
int fit_groups(const float* x, int n, int Dmax, int G, const int32_t* hD, const int32_t* hm, const int32_t* hmss, const int32_t* hmsl,
               const int32_t* y, int K, const int32_t* counts, int T, const int32_t* htree_group, const uint64_t* seeds, int max_depth,
               double min_impurity_decrease, int cap, int32_t* left, int32_t* right, int32_t* feature, double* threshold, double* impurity,
               int32_t* n_node_samples, double* weighted_n_node_samples, uint8_t* missing_go_to_left, int32_t* class_counts,
               int32_t* node_count, int* n_levels, void* ws, cudaStream_t st)
{
    const int mmax = max_of(hm, G), W = (Dmax + 31) / 32;
    const long long TN = (long long)T * n;
    FfWs w = carve(ws, n, Dmax, T, K, mmax, G);
    const int cand_stride = mmax;
    std::vector<int32_t> grp(htree_group, htree_group + T);
    for (const int32_t* a : {hD, hm, hmss, hmsl}) grp.insert(grp.end(), a, a + G);
    ISB_CUDA_CHECK(cudaMemcpyAsync(w.grp, grp.data(), grp.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    const FfGroups gr{x, n, Dmax, w.grp, w.grp + T, w.grp + T + G, w.grp + T + 2 * G, w.grp + T + 3 * G};

    // entries, roots, per-tree totals
    ISB_CUDA_CHECK(cudaMemsetAsync(w.t_nnz, 0, T * sizeof(int32_t), st));
    ISB_CUDA_CHECK(cudaMemsetAsync(w.t_w, 0, T * sizeof(unsigned long long), st));
    ISB_CUDA_CHECK(cudaMemsetAsync(w.info, 0, 8 * sizeof(long long), st));
    ISB_CUDA_CHECK(cudaMemcpyAsync(w.t_seed, seeds, T * sizeof(uint64_t), cudaMemcpyDeviceToDevice, st));
    k_ff_flags<<<blocks_of(TN + 1), TB, 0, st>>>(y, K, counts, n, T, w.lv_rows, w.t_nnz, w.t_w, w.info);
    ISB_LAUNCH_CHECK();
    size_t tb = w.tmp_bytes;
    ISB_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(w.tmp, tb, w.lv_rows, w.flag_pos, (int)(TN + 1), st));
    ISB_CUDA_CHECK(cudaMemcpyAsync(w.info + 1, w.flag_pos + TN, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    long long info[8];
    std::vector<int32_t> nnz(T);
    std::vector<unsigned long long> tw(T);
    if (int s = read_back(info, w.info, 8, st)) return s;
    if (int s = read_back(nnz.data(), w.t_nnz, T, st)) return s;
    if (int s = read_back(tw.data(), w.t_w, T, st)) return s;
    if (info[0] & 1) { isb_set_error("negative count"); return ISB_ERR_ARG; }
    if (info[0] & 4) { isb_set_error("class index outside [0, K)"); return ISB_ERR_ARG; }
    if (info[0] & 2) { isb_set_error("a row count above %d", FF_CMAX); return ISB_ERR_UNSUPPORTED; }
    for (int t = 0; t < T; ++t) {
        if (nnz[t] < 1) { isb_set_error("tree %d has no row with a nonzero count", t); return ISB_ERR_ARG; }
        if ((long long)tw[t] >= FF_WMAX) { isb_set_error("tree %d: total count %llu, at most 2^26 - 1", t, tw[t]); return ISB_ERR_UNSUPPORTED; }
        if (2ll * nnz[t] - 1 > cap) { isb_set_error("tree %d needs capacity %d, has %d", t, 2 * nnz[t] - 1, cap); return ISB_ERR_CAPACITY; }
    }
    const int E = (int)info[1];                         // 4-byte copies into zeroed 8-byte slots
    k_ff_entries<<<blocks_of(TN), TB, 0, st>>>(y, counts, n, T, w.flag_pos, w.e_row, w.e_tree, w.e_node, w.e_pay, w.g_idx);
    ISB_LAUNCH_CHECK();
    k_ff_roots<<<blocks_of(T), TB, 0, st>>>(T, w.nd_tree, w.nd_depth, w.nd_local, w.t_next, w.t_first, w.t_nsplit);
    ISB_LAUNCH_CHECK();

    std::vector<int> level_begin;
    int L0 = 0, L1 = T, n_active = E;
    while (L1 > L0) {
        level_begin.push_back(L0);
        const int nl = L1 - L0;
        k_ff_init_nodes<<<blocks_of((long long)nl * (K + 1)), TB, 0, st>>>(L0, L1, K, w.nd_rows, w.nd_w, w.nd_cc);
        ISB_LAUNCH_CHECK();
        k_ff_stats<<<blocks_of(n_active), TB, 0, st>>>(w.g_idx, n_active, w.e_node, w.e_pay, K, w.nd_cc, w.nd_rows, w.nd_w);
        ISB_LAUNCH_CHECK();
        k_ff_decide<<<blocks_of(nl + 1), TB, 0, st>>>(L0, nl, K, w.nd_cc, w.nd_rows, w.nd_w, w.nd_depth, w.nd_tree, max_depth, gr, w.nd_imp,
                                                      w.nd_split, w.lv_rows);
        ISB_LAUNCH_CHECK();
        tb = w.tmp_bytes;
        ISB_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(w.tmp, tb, w.lv_rows, w.lv_start, nl + 1, st));
        k_ff_nonconst<<<dim3(nl, W), NC_WARPS * 32, 0, st>>>(gr, L0, w.nd_split, w.nd_tree, w.lv_start, w.g_idx, w.e_row, w.nc_bits, W);
        ISB_LAUNCH_CHECK();
        k_ff_candidates<<<nl + 1, CAND_THREADS, 0, st>>>(gr, W, L0, nl, w.nd_split, w.nd_tree, w.nd_local, w.t_seed, w.nc_bits, w.nd_rows,
                                                          w.lv_ncand, w.lv_nelem, w.cand, cand_stride);
        ISB_LAUNCH_CHECK();
        tb = w.tmp_bytes;
        ISB_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(w.tmp, tb, w.lv_ncand, w.lv_segoff, nl + 1, st));
        tb = w.tmp_bytes;
        ISB_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(w.tmp, tb, w.lv_nelem, w.lv_elemoff, nl + 1, st));
        ISB_CUDA_CHECK(cudaMemcpyAsync(w.info + 2, w.lv_elemoff + nl, sizeof(long long), cudaMemcpyDeviceToDevice, st));
        ISB_CUDA_CHECK(cudaMemcpyAsync(w.info + 3, w.lv_segoff + nl, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
        if (int s = read_back(info, w.info, 8, st)) return s;
        const long long n_elem = info[2];
        const int n_seg = (int)info[3];
        if (n_seg > 0) {
            k_ff_fill<<<(int)std::min<long long>(blocks_of(n_elem), 65535ll * 8), TB, 0, st>>>(
                gr, w.nd_tree, L0, nl, n_elem, w.lv_elemoff, w.lv_segoff, w.lv_start, w.nd_rows, w.cand, cand_stride, w.g_idx, w.e_row, w.e_pay, w.k_in, w.p_in);
            ISB_LAUNCH_CHECK();
            tb = w.tmp_bytes;
            ISB_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(w.tmp, tb, w.k_in, w.k_out, w.p_in, w.p_out, (int)n_elem, 0,
                                                           32 + bits_for((unsigned long long)n_seg), st));
            ISB_LAUNCH_CHECK();
            k_ff_scan<<<blocks_of(n_seg, 128), 128, 0, st>>>(L0, nl, n_seg, K, gr, w.nd_tree, w.lv_segoff, w.lv_elemoff, w.nd_rows, w.nd_cc,
                                                             w.nd_w, w.k_out, w.p_out, w.s_proxy, w.s_pos, w.s_thr, w.s_wl, w.s_sql, w.s_sqr);
            ISB_LAUNCH_CHECK();
        }
        ISB_CUDA_CHECK(cudaMemsetAsync(w.info + 3, 0, 3 * sizeof(long long), st));
        k_ff_choose<<<blocks_of(nl + 1), TB, 0, st>>>(L0, nl, w.lv_ncand, w.lv_segoff, w.cand, cand_stride, w.s_proxy, w.s_pos, w.s_thr, w.s_wl,
                                                      w.s_sql, w.s_sqr, w.nd_tree, w.nd_rows, w.nd_w, w.nd_imp, w.t_w, min_impurity_decrease,
                                                      w.nd_split, w.nd_feature, w.nd_thr, w.nd_mgl, w.lv_flag, w.info);
        ISB_LAUNCH_CHECK();
        tb = w.tmp_bytes;
        ISB_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(w.tmp, tb, w.lv_flag, w.lv_rank, nl + 1, st));
        ISB_CUDA_CHECK(cudaMemcpyAsync(w.info + 4, w.lv_rank + nl, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
        if (int s = read_back(info, w.info, 8, st)) return s;
        const int n_split = (int)info[4], n_next = (int)info[5];
        k_ff_tree_first<<<blocks_of(nl), TB, 0, st>>>(L0, nl, w.lv_flag, w.lv_rank, w.nd_tree, w.t_first, w.t_nsplit);
        ISB_LAUNCH_CHECK();
        k_ff_children<<<blocks_of(nl), TB, 0, st>>>(L0, L1, nl, w.lv_flag, w.lv_rank, w.t_first, w.t_next, w.nd_tree, w.nd_depth, w.nd_local,
                                                    w.nd_left, w.nd_right);
        ISB_LAUNCH_CHECK();
        k_ff_tree_advance<<<blocks_of(T), TB, 0, st>>>(T, w.t_next, w.t_first, w.t_nsplit);
        ISB_LAUNCH_CHECK();
        if (n_split == 0) { L0 = L1; break; }
        const int n_child = 2 * n_split;
        k_ff_route<<<blocks_of(n_active), TB, 0, st>>>(gr, w.nd_tree, L1, n_child, w.g_idx, n_active, w.e_node, w.e_row, w.nd_split, w.nd_feature, w.nd_thr,
                                                       w.nd_left, w.g_key, w.g_idx2);
        ISB_LAUNCH_CHECK();
        tb = w.tmp_bytes;
        ISB_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(w.tmp, tb, w.g_key, w.g_key2, w.g_idx2, w.g_idx, n_active, 0,
                                                       bits_for((unsigned long long)n_child), st));
        ISB_LAUNCH_CHECK();
        n_active = n_next;                              // the entries of leaves sort behind every child
        L0 = L1;
        L1 += n_child;
    }
    const int n_nodes = L0;
    for (int lv = (int)level_begin.size() - 1; lv >= 0; --lv) {
        const int b = level_begin[lv], e = lv + 1 < (int)level_begin.size() ? level_begin[lv + 1] : n_nodes;
        k_ff_size<<<blocks_of(e - b), TB, 0, st>>>(b, e - b, w.nd_split, w.nd_left, w.nd_right, w.nd_size);
        ISB_LAUNCH_CHECK();
    }
    for (int lv = 0; lv < (int)level_begin.size(); ++lv) {
        const int b = level_begin[lv], e = lv + 1 < (int)level_begin.size() ? level_begin[lv + 1] : n_nodes;
        k_ff_pre<<<blocks_of(e - b), TB, 0, st>>>(b, e - b, w.nd_split, w.nd_left, w.nd_right, w.nd_size, w.nd_pre);
        ISB_LAUNCH_CHECK();
    }
    k_ff_write<<<blocks_of(n_nodes), TB, 0, st>>>(n_nodes, T, K, cap, w.nd_tree, w.nd_pre, w.nd_split, w.nd_left, w.nd_right, w.nd_feature, w.nd_thr,
                                                  w.nd_imp, w.nd_rows, w.nd_w, w.nd_mgl, w.nd_cc, w.nd_size, left, right, feature, threshold, impurity,
                                                  n_node_samples, weighted_n_node_samples, missing_go_to_left, class_counts, node_count);
    ISB_LAUNCH_CHECK();
    if (n_levels) *n_levels = (int)level_begin.size();
    return ISB_OK;
}

} // namespace

extern "C" size_t isb_forest_fit_workspace_bytes(int n, int D, int T, int K, int max_features)
{
    if (check_sizes(n, D, T, K, max_features) != ISB_OK) return 0;
    return carve(nullptr, n, D, T, K, max_features, 1).need;
}

extern "C" int isb_forest_fit(const float* x, int n, int D, const int32_t* y, int K, const int32_t* counts, int T, const uint64_t* seeds,
                              int max_features, int min_samples_split, int min_samples_leaf, int max_depth, double min_impurity_decrease, int cap,
                              int32_t* left, int32_t* right, int32_t* feature, double* threshold, double* impurity, int32_t* n_node_samples,
                              double* weighted_n_node_samples, uint8_t* missing_go_to_left, int32_t* class_counts, int32_t* node_count,
                              int* n_levels, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    if (int s = check_sizes(n, D, T, K, max_features)) return s;
    ISB_REQUIRE(x && y && counts && seeds && left && right && feature && threshold && impurity && n_node_samples && weighted_n_node_samples &&
                    missing_go_to_left && class_counts && node_count && ws, "null pointer");
    ISB_REQUIRE(min_samples_split >= 2 && min_samples_leaf >= 1 && max_depth >= -1 && cap >= 1, "bad tree parameter");
    ISB_REQUIRE(min_impurity_decrease == min_impurity_decrease, "min_impurity_decrease is NaN");
    ISB_REQUIRE(ws_bytes >= isb_forest_fit_workspace_bytes(n, D, T, K, max_features), "workspace too small");
    const std::vector<int32_t> tree_group(T, 0);
    return fit_groups(x, n, D, 1, &D, &max_features, &min_samples_split, &min_samples_leaf, y, K, counts, T, tree_group.data(), seeds,
                      max_depth, min_impurity_decrease, cap, left, right, feature, threshold, impurity, n_node_samples, weighted_n_node_samples,
                      missing_go_to_left, class_counts, node_count, n_levels, ws, (cudaStream_t)stream);
}

extern "C" size_t isb_forest_fit_groups_workspace_bytes(int n, int Dmax, int G, int T, int K, int max_features_max)
{
    if (G < 1 || check_sizes(n, Dmax, T, K, max_features_max) != ISB_OK) return 0;
    return carve(nullptr, n, Dmax, T, K, max_features_max, G).need;
}

extern "C" int isb_forest_fit_groups(const float* x, int n, int Dmax, int G, const int32_t* D, const int32_t* max_features,
                                     const int32_t* min_samples_split, const int32_t* min_samples_leaf, const int32_t* y, int K,
                                     const int32_t* counts, int T, const int32_t* tree_group, const uint64_t* seeds, int max_depth,
                                     double min_impurity_decrease, int cap, int32_t* left, int32_t* right, int32_t* feature, double* threshold,
                                     double* impurity, int32_t* n_node_samples, double* weighted_n_node_samples, uint8_t* missing_go_to_left,
                                     int32_t* class_counts, int32_t* node_count, int* n_levels, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(n >= 1 && Dmax >= 1 && T >= 1 && K >= 1, "need n, Dmax, T, K >= 1");
    if (int s = check_groups(Dmax, G, D, max_features, min_samples_split, min_samples_leaf, T, tree_group)) return s;
    const int mmax = max_of(max_features, G);
    if (int s = check_sizes(n, Dmax, T, K, mmax)) return s;
    ISB_REQUIRE(x && y && counts && seeds && left && right && feature && threshold && impurity && n_node_samples && weighted_n_node_samples &&
                    missing_go_to_left && class_counts && node_count && ws, "null pointer");
    ISB_REQUIRE(max_depth >= -1 && cap >= 1, "bad tree parameter");
    ISB_REQUIRE(min_impurity_decrease == min_impurity_decrease, "min_impurity_decrease is NaN");
    ISB_REQUIRE(ws_bytes >= isb_forest_fit_groups_workspace_bytes(n, Dmax, G, T, K, mmax), "workspace too small");
    return fit_groups(x, n, Dmax, G, D, max_features, min_samples_split, min_samples_leaf, y, K, counts, T, tree_group, seeds, max_depth,
                      min_impurity_decrease, cap, left, right, feature, threshold, impurity, n_node_samples, weighted_n_node_samples,
                      missing_go_to_left, class_counts, node_count, n_levels, ws, (cudaStream_t)stream);
}
