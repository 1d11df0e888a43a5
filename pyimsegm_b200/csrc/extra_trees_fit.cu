// extra_trees_fit.cu -- the random-split Gini trees of scikit-learn's ExtraTreesClassifier, node for node the trees scikit-learn 1.9
// builds: one CTA per tree replays DepthFirstTreeBuilder.build (_tree.pyx) and every draw of node_split_random (_splitter.pyx).
//
// Why one tree is sequential: the splitter's xorshift state (our_rand_r) and its `features` / `constant_features` permutations run
// from node to node in the builder's depth-first order, so a node's draws depend on every node built before it.  Trees are
// independent, so all of them run at once, one CTA each.  A node needs only its own rows, and extra trees need no sort, so the
// order in which a node visits its rows does not matter: class counts are integers, and only which rows go to which side does.
//
// Per tree: samples [nnz] (the rows of nonzero count, partitioned in place per node), a depth-first stack, and features /
// constant_features in shared memory.  Thread 0 owns the draw loop and the RNG.  Two paths:
//   block path  a node of more than `small` rows: the whole CTA makes the passes over its rows (class counts; min / max of each
//               drawn feature; rows and class counts left of each threshold; the final partition), thread 0 decides between them;
//   warp path   a node of at most `small` rows: warp 0 stages the rows (D contiguous floats each, with class and count) in shared
//               memory once and builds that node's whole subtree depth first with no block barrier; every lane runs the same draws.
// The FP64 expressions are tree_split.cuh's (shared with forest_fit.cu); the library is built with -fmad=false.
#include "common.cuh"
#include "block_scan.cuh"
#include "tree_split.cuh"
#include <vector>

namespace {

constexpr int ET_THREADS = 512;
constexpr int ET_SMALL_DEFAULT = 64;          // rows at or below which a subtree goes to the warp path (DESIGN.md §8)
constexpr int ET_SMALL_MAX = 256;
constexpr size_t ET_STAGE_BYTES = 96 * 1024;  // shared memory for the staged rows of the warp path
constexpr uint32_t RAND_R_MAX = 0x7fffffffu;
constexpr unsigned FULL = 0xffffffffu;

// sklearn/utils/_random.pxd our_rand_r; tree/_utils.pyx rand_int / rand_uniform
__device__ __forceinline__ uint32_t our_rand_r(uint32_t& s)
{
    if (s == 0) s = 1;                                 // DEFAULT_SEED
    s ^= s << 13;
    s ^= s >> 17;
    s ^= s << 5;
    return s % (RAND_R_MAX + 1u);
}
__device__ __forceinline__ int rand_int(int low, int high, uint32_t& s) { return low + (int)(our_rand_r(s) % (uint32_t)(high - low)); }
__device__ __forceinline__ double rand_uniform(double low, double high, uint32_t& s)
{
    return ((high - low) * (double)our_rand_r(s) / (double)RAND_R_MAX) + low;
}

__device__ __forceinline__ unsigned f32_ordered(float v)
{
    const unsigned u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float f32_unordered(unsigned o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o); }

// the Fisher-Yates draw of node_split_random over the tree's features array; `mask` the lanes that run it in lockstep (lane 0 writes)
struct Draw {
    int f_i, f_j, n_found, n_drawn, n_known, n_total, n_visited, m;
    __device__ void init(int D, int n_constant, int max_features)
    {
        f_i = D;
        f_j = n_found = n_drawn = n_visited = 0;
        n_known = n_total = n_constant;
        m = max_features;
    }
    __device__ static void swap(short* f, int a, int b, unsigned mask)
    {
        const short va = f[a], vb = f[b];
        __syncwarp(mask);
        if ((threadIdx.x & 31) == 0) { f[a] = vb; f[b] = va; }
        __syncwarp(mask);
    }
    // the next feature to evaluate, or -1 when the loop ends; draws of known constants are consumed here
    __device__ int next(short* features, uint32_t& rng, unsigned mask)
    {
        while (f_i > n_total && (n_visited < m || n_visited <= n_found + n_drawn)) {
            ++n_visited;
            int j = rand_int(n_drawn, f_i - n_found, rng);
            if (j < n_known) {
                swap(features, n_drawn, j, mask);
                ++n_drawn;
                continue;
            }
            f_j = j + n_found;
            return features[f_j];
        }
        return -1;
    }
    __device__ void constant(short* features, unsigned mask)
    {
        swap(features, f_j, n_total, mask);
        ++n_found;
        ++n_total;
    }
    __device__ void accept(short* features, unsigned mask)
    {
        --f_i;
        swap(features, f_i, f_j, mask);
    }
};

// the best split of a node so far
struct Best {
    int feature, n_left;                               // n_left < 0: none
    double threshold, proxy, wl;
    unsigned long long sql, sqr;
    __device__ void clear()
    {
        feature = 0;
        n_left = -1;
        threshold = 0.0;
        proxy = -__longlong_as_double(0x7ff0000000000000ll);
        wl = 0.0;
        sql = sqr = 0;
    }
};

struct EtArgs {
    const float* x;
    int n, D;
    const int32_t* y;
    int K;
    const int32_t* counts;
    const uint32_t* states;
    int m, mss, msl, max_depth;
    double mid;
    int cap, small;
    int32_t *left, *right, *feature;
    double *threshold, *impurity;
    int32_t* n_node_samples;
    double* weighted_n_node_samples;
    uint8_t* missing_go_to_left;
    int32_t *class_counts, *node_count;
    // workspace
    int32_t *samples, *tmp, *stk_nc;
    int4* stk;                                         // start, end, depth, link (parent << 1 | is_left, -1 at the root)
    const unsigned long long* t_w;
};

struct EtShared {                                      // the CTA's scalars
    int top, nodes, cmd, f, n_left, nnz;
    unsigned lo, hi;
    uint32_t rng;
    double thr;
    int4 rec;
    int nc;
};

enum { CMD_MINMAX, CMD_LEFT, CMD_PART, CMD_DONE };

// the dynamic shared memory: features, constant_features [D] i16; class counts of the node and of a left side [K] i32; the warp path's
// staged rows xs [small, D] f32, counts [small] i32, classes [small] u8, row order loc / loc2 [small] i16, stack [small + 1] x 5 i32
struct EtSmem {
    short *feat, *cfeat;
    int *cc, *lcc;
    float* xs;
    int* wcnt;
    unsigned char* wcls;
    short *loc, *loc2;
    int *k_start, *k_end, *k_depth, *k_link, *k_nc;
};

__host__ __device__ inline size_t et_smem_layout(int D, int K, int S, char* base, EtSmem* s)
{
    size_t o = 0;
    auto take = [&](size_t bytes) { char* p = base + o; o = (o + bytes + 15) & ~size_t(15); return p; };
    char* feat = take(2 * (size_t)D);
    char* cfeat = take(2 * (size_t)D);
    char* cc = take(4 * (size_t)K);
    char* lcc = take(4 * (size_t)K);
    char* xs = take(4 * (size_t)S * D);
    char* wcnt = take(4 * (size_t)S);
    char* wcls = take((size_t)S);
    char* loc = take(2 * (size_t)S);
    char* loc2 = take(2 * (size_t)S);
    char* stack = take(4 * 5 * (size_t)(S + 1));
    if (s) {
        s->feat = (short*)feat; s->cfeat = (short*)cfeat; s->cc = (int*)cc; s->lcc = (int*)lcc; s->xs = (float*)xs; s->wcnt = (int*)wcnt;
        s->wcls = (unsigned char*)wcls; s->loc = (short*)loc; s->loc2 = (short*)loc2;
        s->k_start = (int*)stack; s->k_end = s->k_start + S + 1; s->k_depth = s->k_end + S + 1; s->k_link = s->k_depth + S + 1;
        s->k_nc = s->k_link + S + 1;
    }
    return o;
}

__device__ __forceinline__ unsigned long long warp_sum64(unsigned long long v)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}

// one node's output row: everything but the split fields, and the parent's link to it
__device__ void write_node(const EtArgs& a, size_t base, int nid, int link, double imp, int rows, unsigned long long w, const int* cc)
{
    const size_t o = base + nid;
    a.impurity[o] = imp;
    a.n_node_samples[o] = rows;
    a.weighted_n_node_samples[o] = (double)w;
    for (int c = 0; c < a.K; ++c) a.class_counts[o * a.K + c] = cc[c];
    if (link >= 0) (link & 1 ? a.left : a.right)[base + (link >> 1)] = nid;
}
__device__ void write_leaf(const EtArgs& a, size_t o)
{
    a.left[o] = a.right[o] = -1;                       // _TREE_LEAF
    a.feature[o] = -2;                                 // _TREE_UNDEFINED
    a.threshold[o] = -2.0;
    a.missing_go_to_left[o] = 0;
}
__device__ void write_split(const EtArgs& a, size_t o, const Best& b, int rows)
{
    a.feature[o] = b.feature;
    a.threshold[o] = b.threshold;
    a.missing_go_to_left[o] = b.n_left > rows - b.n_left;
}

// the leaf tests of DepthFirstTreeBuilder.build that come before node_split
__device__ __forceinline__ bool leaf_before_split(const EtArgs& a, int depth, int rows, double imp)
{
    return (a.max_depth >= 0 && depth >= a.max_depth) || rows < a.mss || rows < 2 * a.msl || imp <= FF_EPSILON;
}

// the split's children impurities and improvement, and the last leaf test; true when the node splits
__device__ __forceinline__ bool split_holds(const EtArgs& a, const Best& b, int rows, double w, double W, double imp)
{
    if (b.n_left < 0) return false;                    // split.pos >= end
    const double wr = w - b.wl;
    const double il = gini_of(b.sql, b.wl), ir = gini_of(b.sqr, wr);
    return !(impurity_improvement(w, W, imp, b.wl, il, ir) + FF_EPSILON < a.mid);
}

// the end of node_split_random: restore features[:n_known], keep the newly found constants
__device__ __forceinline__ void keep_constants(short* feat, short* cfeat, const Draw& d, int lane, int stride)
{
    for (int q = lane; q < d.n_known; q += stride) feat[q] = cfeat[q];
    for (int q = lane; q < d.n_found; q += stride) cfeat[d.n_known + q] = feat[d.n_known + q];
}

// ---- warp path: the whole subtree of a node of at most `small` rows, by warp 0 ----
__device__ void warp_subtree(const EtArgs& a, const EtSmem& sm, EtShared& sh, int t, double W)
{
    const int lane = threadIdx.x & 31, D = a.D, K = a.K;
    const int4 rec = sh.rec;
    const int rows0 = rec.y - rec.x;
    const size_t base = (size_t)t * a.cap;
    const int32_t* samples = a.samples + (size_t)t * a.n;
    const int32_t* cnt_t = a.counts + (size_t)t * a.n;
    for (int i = 0; i < rows0; ++i) {
        const int r = samples[rec.x + i];
        const float* xr = a.x + (size_t)r * D;
        for (int f = lane; f < D; f += 32) sm.xs[i * D + f] = xr[f];
    }
    for (int i = lane; i < rows0; i += 32) {
        const int r = samples[rec.x + i];
        sm.wcnt[i] = cnt_t[r];
        sm.wcls[i] = (unsigned char)a.y[r];
        sm.loc[i] = (short)i;
    }
    uint32_t rng = sh.rng;
    int nid = sh.nodes;
    int top = 1;
    if (lane == 0) {
        sm.k_start[0] = 0; sm.k_end[0] = rows0; sm.k_depth[0] = rec.z; sm.k_link[0] = rec.w; sm.k_nc[0] = sh.nc;
    }
    __syncwarp();
    while (top > 0) {
        --top;
        const int s = sm.k_start[top], e = sm.k_end[top], depth = sm.k_depth[top], link = sm.k_link[top], nc = sm.k_nc[top];
        const int rows = e - s;
        for (int c = lane; c < K; c += 32) sm.cc[c] = 0;
        __syncwarp();
        for (int i = s + lane; i < e; i += 32) atomicAdd(&sm.cc[sm.wcls[sm.loc[i]]], sm.wcnt[sm.loc[i]]);
        __syncwarp();
        unsigned long long sq = 0, w = 0;
        for (int c = lane; c < K; c += 32) {
            const unsigned long long v = (unsigned long long)sm.cc[c];
            sq += v * v;
            w += v;
        }
        sq = warp_sum64(sq);
        w = warp_sum64(w);
        const double dw = (double)w, imp = gini_of(sq, dw);
        const size_t o = base + nid;
        if (lane == 0) write_node(a, base, nid, link, imp, rows, w, sm.cc);
        bool leaf = leaf_before_split(a, depth, rows, imp);
        Best b;
        b.clear();
        Draw d;
        if (!leaf) {
            d.init(D, nc, a.m);
            int f;
            while ((f = d.next(sm.feat, rng, FULL)) >= 0) {
                unsigned lo = 0xffffffffu, hi = 0u;
                for (int i = s + lane; i < e; i += 32) {
                    const unsigned u = f32_ordered(sm.xs[sm.loc[i] * D + f]);
                    lo = min(lo, u);
                    hi = max(hi, u);
                }
                const float mn = f32_unordered(__reduce_min_sync(FULL, lo)), mx = f32_unordered(__reduce_max_sync(FULL, hi));
                if (mx <= __fadd_rn(mn, FEATURE_THRESHOLD)) {
                    d.constant(sm.feat, FULL);
                    continue;
                }
                d.accept(sm.feat, FULL);
                double thr = rand_uniform((double)mn, (double)mx, rng);
                if (thr == (double)mx) thr = (double)mn;
                for (int c = lane; c < K; c += 32) sm.lcc[c] = 0;
                __syncwarp();
                int nl = 0;
                for (int i = s + lane; i < e; i += 32) {
                    const int q = sm.loc[i];
                    if ((double)sm.xs[q * D + f] <= thr) {
                        ++nl;
                        atomicAdd(&sm.lcc[sm.wcls[q]], sm.wcnt[q]);
                    }
                }
                nl = __reduce_add_sync(FULL, nl);
                __syncwarp();
                if (nl < a.msl || rows - nl < a.msl) continue;
                unsigned long long sql = 0, sqr = 0, wl = 0;
                for (int c = lane; c < K; c += 32) {
                    const unsigned long long l = (unsigned long long)sm.lcc[c], r = (unsigned long long)(sm.cc[c] - sm.lcc[c]);
                    sql += l * l;
                    sqr += r * r;
                    wl += l;
                }
                sql = warp_sum64(sql);
                sqr = warp_sum64(sqr);
                wl = warp_sum64(wl);
                const double proxy = gini_proxy(sql, (double)wl, sqr, (double)(w - wl));
                if (proxy > b.proxy) {
                    b.proxy = proxy; b.feature = f; b.threshold = thr; b.n_left = nl; b.wl = (double)wl; b.sql = sql; b.sqr = sqr;
                }
            }
            keep_constants(sm.feat, sm.cfeat, d, lane, 32);
            __syncwarp();
            leaf = !split_holds(a, b, rows, dw, W, imp);
        }
        if (leaf) {
            if (lane == 0) write_leaf(a, o);
        } else {
            if (lane == 0) write_split(a, o, b, rows);
            // partition loc[s, e) by the split: left rows to [s, s + n_left), right rows after
            int nl = 0, nr = 0;
            for (int i0 = s; i0 < e; i0 += 32) {
                const int i = i0 + lane;
                const int q = i < e ? sm.loc[i] : 0;
                const bool go = i < e && (double)sm.xs[q * D + b.feature] <= b.threshold;
                const unsigned bl = __ballot_sync(FULL, go), br = __ballot_sync(FULL, i < e && !go);
                const unsigned below = (1u << lane) - 1u;
                if (go) sm.loc2[s + nl + __popc(bl & below)] = (short)q;
                else if (i < e) sm.loc2[s + b.n_left + nr + __popc(br & below)] = (short)q;
                nl += __popc(bl);
                nr += __popc(br);
            }
            __syncwarp();
            for (int i = s + lane; i < e; i += 32) sm.loc[i] = sm.loc2[i];
            if (lane == 0) {
                sm.k_start[top] = s + b.n_left; sm.k_end[top] = e; sm.k_depth[top] = depth + 1; sm.k_link[top] = nid << 1; sm.k_nc[top] = d.n_total;
                sm.k_start[top + 1] = s; sm.k_end[top + 1] = s + b.n_left; sm.k_depth[top + 1] = depth + 1; sm.k_link[top + 1] = nid << 1 | 1;
                sm.k_nc[top + 1] = d.n_total;
            }
            top += 2;
            __syncwarp();
        }
        ++nid;
    }
    if (lane == 0) {
        sh.rng = rng;
        sh.nodes = nid;
    }
}

// ---- one CTA per tree ----
__global__ void __launch_bounds__(ET_THREADS, 1) k_et_build(EtArgs a)
{
    extern __shared__ __align__(16) char smem[];
    __shared__ EtShared sh;
    EtSmem sm;
    et_smem_layout(a.D, a.K, a.small, smem, &sm);
    const int t = blockIdx.x, tid = threadIdx.x, D = a.D, K = a.K;
    const size_t base = (size_t)t * a.cap;
    int32_t* samples = a.samples + (size_t)t * a.n;
    int32_t* tmp = a.tmp + (size_t)t * a.n;
    const int32_t* cnt_t = a.counts + (size_t)t * a.n;
    int4* stk = a.stk + (size_t)t * (a.n + 1);
    int32_t* stk_nc = a.stk_nc + (size_t)t * (a.n + 1);
    const double W = (double)a.t_w[t];

    // Splitter.init: the rows of nonzero weight in ascending order, features = arange(D)
    const int nnz = cta_scan_chunks<ET_THREADS, int>(a.n, [&](int i) { return cnt_t[i] > 0 ? 1 : 0; },
                                                     [&](int i, int pos) { if (cnt_t[i] > 0) samples[pos] = i; });
    for (int f = tid; f < D; f += ET_THREADS) sm.feat[f] = (short)f;
    if (tid == 0) {
        stk[0] = make_int4(0, nnz, 0, -1);
        stk_nc[0] = 0;
        sh.top = 1;
        sh.nodes = 0;
        sh.rng = a.states[t];
    }
    __syncthreads();

    // thread 0's state across the phases of a block-path node
    Draw d;
    Best b;
    uint32_t rng = 0;
    int rows = 0, nid = 0;
    unsigned long long w = 0;
    double imp = 0.0;
    while (true) {
        if (tid == 0) {
            if (sh.top > 0) {
                --sh.top;
                sh.rec = stk[sh.top];
                sh.nc = stk_nc[sh.top];
            } else {
                sh.rec = make_int4(0, 0, -1, 0);
            }
        }
        __syncthreads();
        const int4 rec = sh.rec;
        if (rec.z < 0) break;
        const int start = rec.x, end = rec.y;
        if (end - start <= a.small) {
            if (tid < 32) warp_subtree(a, sm, sh, t, W);
            __syncthreads();
            continue;
        }
        // class counts of the node
        for (int c = tid; c < K; c += ET_THREADS) sm.cc[c] = 0;
        __syncthreads();
        for (int i = start + tid; i < end; i += ET_THREADS) {
            const int r = samples[i];
            atomicAdd(&sm.cc[a.y[r]], cnt_t[r]);
        }
        __syncthreads();
        // thread 0 walks the node's decisions; between two of them the CTA makes one pass (sh.cmd) over the node's rows
        auto next_candidate = [&]() {
            const int f = d.next(sm.feat, rng, 1u);
            if (f >= 0) {
                sh.f = f;
                sh.lo = 0xffffffffu;
                sh.hi = 0u;
                sh.cmd = CMD_MINMAX;
                return;
            }
            keep_constants(sm.feat, sm.cfeat, d, 0, 1);
            if (!split_holds(a, b, rows, (double)w, W, imp)) {
                write_leaf(a, base + nid);
                sh.cmd = CMD_DONE;
                return;
            }
            write_split(a, base + nid, b, rows);
            sh.f = b.feature;
            sh.thr = b.threshold;
            sh.n_left = b.n_left;
            sh.cmd = CMD_PART;
        };
        if (tid == 0) {
            rows = end - start;
            unsigned long long sq = 0;
            w = 0;
            for (int c = 0; c < K; ++c) {
                const unsigned long long v = (unsigned long long)sm.cc[c];
                sq += v * v;
                w += v;
            }
            imp = gini_of(sq, (double)w);
            nid = sh.nodes++;
            write_node(a, base, nid, rec.w, imp, rows, w, sm.cc);
            rng = sh.rng;
            b.clear();
            if (leaf_before_split(a, rec.z, rows, imp)) {
                write_leaf(a, base + nid);
                sh.cmd = CMD_DONE;
            } else {
                d.init(D, sh.nc, a.m);
                next_candidate();
            }
            sh.rng = rng;
        }
        __syncthreads();
        while (true) {
            const int cmd = sh.cmd, f = sh.f;
            if (cmd == CMD_DONE) break;
            if (cmd == CMD_MINMAX) {
                unsigned lo = 0xffffffffu, hi = 0u;
                for (int i = start + tid; i < end; i += ET_THREADS) {
                    const unsigned u = f32_ordered(a.x[(size_t)samples[i] * D + f]);
                    lo = min(lo, u);
                    hi = max(hi, u);
                }
                lo = __reduce_min_sync(FULL, lo);
                hi = __reduce_max_sync(FULL, hi);
                if ((tid & 31) == 0) {
                    atomicMin(&sh.lo, lo);
                    atomicMax(&sh.hi, hi);
                }
            } else if (cmd == CMD_LEFT) {
                const double thr = sh.thr;
                int nl = 0;
                for (int i = start + tid; i < end; i += ET_THREADS) {
                    const int r = samples[i];
                    if ((double)a.x[(size_t)r * D + f] <= thr) {
                        ++nl;
                        atomicAdd(&sm.lcc[a.y[r]], cnt_t[r]);
                    }
                }
                nl = __reduce_add_sync(FULL, nl);
                if ((tid & 31) == 0) atomicAdd(&sh.n_left, nl);
            } else {                                   // CMD_PART: left rows to [start, start + n_left), right rows after
                const double thr = sh.thr;
                const int n_left = sh.n_left;
                int carry = 0;
                for (int i0 = start; i0 < end; i0 += ET_THREADS) {
                    const int i = i0 + tid;
                    const int r = i < end ? samples[i] : 0;
                    const int go = i < end && (double)a.x[(size_t)r * D + f] <= thr;
                    int total;
                    const int before = cta_exclusive_sum<ET_THREADS>(go, total);
                    if (i < end) tmp[go ? start + carry + before : start + n_left + (i0 - start - carry) + (tid - before)] = r;
                    carry += total;
                }
                __syncthreads();
                for (int i = start + tid; i < end; i += ET_THREADS) samples[i] = tmp[i];
            }
            __syncthreads();
            if (tid == 0) {
                if (cmd == CMD_MINMAX) {
                    const float mn = f32_unordered(sh.lo), mx = f32_unordered(sh.hi);
                    if (mx <= __fadd_rn(mn, FEATURE_THRESHOLD)) {
                        d.constant(sm.feat, 1u);
                        next_candidate();
                    } else {
                        d.accept(sm.feat, 1u);
                        double thr = rand_uniform((double)mn, (double)mx, rng);
                        if (thr == (double)mx) thr = (double)mn;
                        sh.thr = thr;
                        sh.n_left = 0;
                        for (int c = 0; c < K; ++c) sm.lcc[c] = 0;
                        sh.cmd = CMD_LEFT;
                    }
                } else if (cmd == CMD_LEFT) {
                    const int nl = sh.n_left;
                    if (nl >= a.msl && rows - nl >= a.msl) {
                        unsigned long long sql = 0, sqr = 0, wl = 0;
                        for (int c = 0; c < K; ++c) {
                            const unsigned long long l = (unsigned long long)sm.lcc[c], r = (unsigned long long)(sm.cc[c] - sm.lcc[c]);
                            sql += l * l;
                            sqr += r * r;
                            wl += l;
                        }
                        const double proxy = gini_proxy(sql, (double)wl, sqr, (double)(w - wl));
                        if (proxy > b.proxy) {
                            b.proxy = proxy; b.feature = f; b.threshold = sh.thr; b.n_left = nl; b.wl = (double)wl; b.sql = sql; b.sqr = sqr;
                        }
                    }
                    next_candidate();
                } else {                               // push the right child, then the left one (built first)
                    const int top = sh.top;
                    stk[top] = make_int4(start + b.n_left, end, rec.z + 1, nid << 1);
                    stk[top + 1] = make_int4(start, start + b.n_left, rec.z + 1, nid << 1 | 1);
                    stk_nc[top] = stk_nc[top + 1] = d.n_total;
                    sh.top = top + 2;
                    sh.cmd = CMD_DONE;
                }
                sh.rng = rng;
            }
            __syncthreads();
        }
    }
    if (tid == 0) a.node_count[t] = sh.nodes;
}

// per tree: rows of nonzero count and total count; error flags 1 negative count, 4 class outside [0, K)
__global__ void k_et_check(const int32_t* __restrict__ y, int K, const int32_t* __restrict__ counts, int n, int T, int32_t* __restrict__ t_nnz,
                           unsigned long long* __restrict__ t_w, unsigned long long* __restrict__ info)
{
    const long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (q >= (long long)T * n) return;
    const int t = (int)(q / n), r = (int)(q % n);
    const int cnt = counts[q];
    if (cnt < 0) atomicOr(info, 1ull);
    if (t == 0 && (y[r] < 0 || y[r] >= K)) atomicOr(info, 4ull);
    if (cnt > 0) {
        atomicAdd(t_nnz + t, 1);
        atomicAdd(t_w + t, (unsigned long long)cnt);
    }
}

struct EtWs {
    int32_t *samples, *tmp, *stk_nc, *t_nnz;
    int4* stk;
    unsigned long long *t_w, *info;
    size_t need;
};

EtWs et_carve(void* base, int n, int T)
{
    WsCarver c(base, ~size_t(0));
    const size_t E = (size_t)T * n, S = (size_t)T * (n + 1);
    EtWs w;
    w.samples = c.take<int32_t>(E);
    w.tmp = c.take<int32_t>(E);
    w.stk = c.take<int4>(S);
    w.stk_nc = c.take<int32_t>(S);
    w.t_nnz = c.take<int32_t>(T);
    w.t_w = c.take<unsigned long long>(T);
    w.info = c.take<unsigned long long>(1);
    w.need = c.off;
    return w;
}

int et_small_rows(int D, int K, int small_rows)
{
    int s = small_rows > 0 ? std::min(small_rows, ET_SMALL_MAX) : ET_SMALL_DEFAULT;
    while (s > 1 && et_smem_layout(D, K, s, nullptr, nullptr) > ET_STAGE_BYTES + et_smem_layout(D, K, 0, nullptr, nullptr)) --s;
    return s;
}

int et_check_sizes(int n, int D, int T, int K, int m)
{
    ISB_REQUIRE(n >= 1 && D >= 1 && T >= 1 && K >= 1, "need n, D, T, K >= 1");
    ISB_REQUIRE(m >= 1 && m <= D, "max_features must be in [1, D]");
    if (K > FF_KMAX || D > FF_DMAX || (long long)T * n >= (1ll << 31) || n >= (1 << 30)) {
        isb_set_error("extra-trees fit of %d trees over %d rows x %d features, %d classes: at most %d classes, %d features, and "
                      "trees x rows below 2^31", T, n, D, K, FF_KMAX, FF_DMAX);
        return ISB_ERR_UNSUPPORTED;
    }
    return ISB_OK;
}

} // namespace

extern "C" size_t isb_extra_trees_fit_workspace_bytes(int n, int D, int T, int K, int max_features)
{
    if (et_check_sizes(n, D, T, K, max_features) != ISB_OK) return 0;
    return et_carve(nullptr, n, T).need;
}

extern "C" int isb_extra_trees_fit(const float* x, int n, int D, const int32_t* y, int K, const int32_t* counts, int T, const uint32_t* rand_r_state,
                                   int max_features, int min_samples_split, int min_samples_leaf, int max_depth, double min_impurity_decrease,
                                   int small_rows, int cap, int32_t* left, int32_t* right, int32_t* feature, double* threshold, double* impurity,
                                   int32_t* n_node_samples, double* weighted_n_node_samples, uint8_t* missing_go_to_left, int32_t* class_counts,
                                   int32_t* node_count, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    if (int s = et_check_sizes(n, D, T, K, max_features)) return s;
    ISB_REQUIRE(x && y && counts && rand_r_state && left && right && feature && threshold && impurity && n_node_samples &&
                    weighted_n_node_samples && missing_go_to_left && class_counts && node_count && ws, "null pointer");
    ISB_REQUIRE(min_samples_split >= 2 && min_samples_leaf >= 1 && max_depth >= -1 && cap >= 1 && small_rows >= 0, "bad tree parameter");
    ISB_REQUIRE(min_impurity_decrease == min_impurity_decrease, "min_impurity_decrease is NaN");
    ISB_REQUIRE(ws_bytes >= isb_extra_trees_fit_workspace_bytes(n, D, T, K, max_features), "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    EtWs w = et_carve(ws, n, T);
    ISB_CUDA_CHECK(cudaMemsetAsync(w.t_nnz, 0, T * sizeof(int32_t), st));
    ISB_CUDA_CHECK(cudaMemsetAsync(w.t_w, 0, T * sizeof(unsigned long long), st));
    ISB_CUDA_CHECK(cudaMemsetAsync(w.info, 0, sizeof(unsigned long long), st));
    const long long TN = (long long)T * n;
    k_et_check<<<(int)((TN + 255) / 256), 256, 0, st>>>(y, K, counts, n, T, w.t_nnz, w.t_w, w.info);
    ISB_LAUNCH_CHECK();
    std::vector<int32_t> nnz(T);
    std::vector<unsigned long long> tw(T);
    unsigned long long info = 0;
    ISB_CUDA_CHECK(cudaMemcpyAsync(nnz.data(), w.t_nnz, T * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    ISB_CUDA_CHECK(cudaMemcpyAsync(tw.data(), w.t_w, T * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    ISB_CUDA_CHECK(cudaMemcpyAsync(&info, w.info, sizeof(info), cudaMemcpyDeviceToHost, st));
    ISB_CUDA_CHECK(cudaStreamSynchronize(st));
    if (info & 1) { isb_set_error("negative count"); return ISB_ERR_ARG; }
    if (info & 4) { isb_set_error("class index outside [0, K)"); return ISB_ERR_ARG; }
    for (int t = 0; t < T; ++t) {
        if (nnz[t] < 1) { isb_set_error("tree %d has no row with a nonzero count", t); return ISB_ERR_ARG; }
        if ((long long)tw[t] >= FF_WMAX) { isb_set_error("tree %d: total count %llu, at most 2^26 - 1", t, tw[t]); return ISB_ERR_UNSUPPORTED; }
        if (2ll * nnz[t] - 1 > cap) { isb_set_error("tree %d needs capacity %d, has %d", t, 2 * nnz[t] - 1, cap); return ISB_ERR_CAPACITY; }
    }
    const int small = et_small_rows(D, K, small_rows);
    const size_t smem = et_smem_layout(D, K, small, nullptr, nullptr);
    ISB_CUDA_CHECK(cudaFuncSetAttribute(k_et_build, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    EtArgs a{x, n, D, y, K, counts, rand_r_state, max_features, min_samples_split, min_samples_leaf, max_depth, min_impurity_decrease, cap, small,
             left, right, feature, threshold, impurity, n_node_samples, weighted_n_node_samples, missing_go_to_left, class_counts, node_count,
             w.samples, w.tmp, w.stk_nc, w.stk, w.t_w};
    k_et_build<<<T, ET_THREADS, smem, st>>>(a);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
