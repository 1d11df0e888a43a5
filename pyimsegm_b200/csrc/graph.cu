// graph.cu -- superpixel adjacency graph, GraphCut energies and the final LUT gathers.
//
// Replaces (reference Python, no native code):
//   imsegm/superpixels.py:115-177  make_graph_segm_connect_grid2d_conn4 / get_segment_diffs_2d_conn4 /
//                                  make_graph_segment_connect_edges   (per-pixel dict loop + np.unique)
//   imsegm/graph_cuts.py:303-336   compute_spatial_dist (centres (y, x) of a label map, (z, y, x) of a label volume)
//   imsegm/graph_cuts.py:383-439   compute_edge_model
//   imsegm/graph_cuts.py:523-540   compute_unary_cost
//   imsegm/graph_cuts.py:574-657   compute_edge_weights (clamp to [1e-3, 1e3]; 'color' / 'features' vectors compared by
//                                  isb_gc_vector_edge_weights, the 'color' image scaled by isb_image_unit_scale)
//   pyGCO cut_general_graph        float -> int conversion (see oracle/gc_oracle.cpp header)
//   imsegm/pipelines.py:104,109    proba[slic], graph_labels[slic]
#include "common.cuh"
#include "block_scan.cuh"
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace {

// ------------------------------------------------------------------ adjacency ------------------------------------------------------

struct AdjWs {
    unsigned long long* table; // [slots] keys (b << 32 | a), empty = 0 (b > a >= 0, so no key is 0)
    int* ctr;                  // [4] 0: unique edges, 1: overflow flag
    int* deg;                  // [nb]    number of edges whose larger endpoint is b
    int* off;                  // [nb+1]
    int* fill;                 // [nb]
    int* tmp_a;                // [cap]
    int slots;
    size_t zeroed;             // bytes from `table` through `deg`: cleared by one memset before the scan
};

__device__ __forceinline__ unsigned hash64(unsigned long long k)
{
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return (unsigned)k;
}

__device__ __forceinline__ unsigned long long edge_key(int l0, int l1)
{
    return ((unsigned long long)(unsigned)max(l0, l1) << 32) | (unsigned)min(l0, l1);
}

__device__ void table_insert(const AdjWs& w, unsigned long long key)
{
    unsigned mask = (unsigned)w.slots - 1u;
    unsigned h = hash64(key) & mask;
    for (int probe = 0; probe < w.slots; ++probe) {
        unsigned long long cur = w.table[h];
        if (cur == key) return;
        if (cur == 0) {
            unsigned long long old = atomicCAS(&w.table[h], 0ull, key);
            if (old == 0) { atomicAdd(&w.deg[key >> 32], 1); atomicAdd(&w.ctr[0], 1); return; }
            if (old == key) return;
        }
        h = (h + 1) & mask;
    }
    atomicExch(&w.ctr[1], 1); // table full
}

// A CTA's pixels meet a few dozen label pairs, each many times: the CTA collects its pairs in a shared-memory set and inserts each
// into the global table once.  A pair that finds no free slot within CTA_PROBES goes to the global table directly.
constexpr int CTA_SLOTS = 512, CTA_PROBES = 32;

__device__ void cta_set_clear(unsigned long long* s)
{
    for (int i = threadIdx.x; i < CTA_SLOTS; i += blockDim.x) s[i] = 0;
    __syncthreads();
}

__device__ void cta_set_insert(unsigned long long* s, const AdjWs& w, unsigned long long key)
{
    unsigned h = hash64(key) & (CTA_SLOTS - 1);
    for (int probe = 0; probe < CTA_PROBES; ++probe) {
        unsigned long long cur = s[h];
        if (cur == key) return;
        if (cur == 0) {
            cur = atomicCAS(&s[h], 0ull, key);
            if (cur == 0 || cur == key) return;
        }
        h = (h + 1) & (CTA_SLOTS - 1);
    }
    table_insert(w, key);
}

__device__ void cta_set_flush(const unsigned long long* s, const AdjWs& w)
{
    __syncthreads();
    for (int i = threadIdx.x; i < CTA_SLOTS; i += blockDim.x)
        if (s[i]) table_insert(w, s[i]);
}

// a CTA takes a tile of ETW columns x ETH rows, a thread one column of ETR rows: the thread skips a pair it has just inserted (a
// boundary across its rows gives the same horizontal pair row after row), the set the rest
constexpr int ETW = 64, ETR = 4, ETH = ETR * (256 / ETW);

__global__ void __launch_bounds__(256) k_edge_scan(const int* __restrict__ seg, int H, int W, AdjWs w)
{
    __shared__ unsigned long long s_set[CTA_SLOTS];
    cta_set_clear(s_set);
    const int x = blockIdx.x * ETW + (int)(threadIdx.x % ETW);
    const int y0 = blockIdx.y * ETH + (int)(threadIdx.x / ETW) * ETR, y1 = min(y0 + ETR, H);
    if (x < W && y0 < H) {
        unsigned long long last = 0;
        int l = seg[(size_t)y0 * W + x];
        for (int y = y0; y < y1; ++y) {
            const size_t p = (size_t)y * W + x;
            const int d = y + 1 < H ? seg[p + W] : l;
            if (x + 1 < W) {
                const int r = seg[p + 1];
                if (r != l && edge_key(l, r) != last) { last = edge_key(l, r); cta_set_insert(s_set, w, last); }
            }
            if (d != l && edge_key(l, d) != last) { last = edge_key(l, d); cta_set_insert(s_set, w, last); }
            l = d;
        }
    }
    cta_set_flush(s_set, w);
}

// the same for a volume: 6-connectivity = the pairs with the x+1, y+1 and z+1 neighbour (reference superpixels.py:145-154)
__global__ void __launch_bounds__(256) k_edge_scan3d(const int* __restrict__ seg, int D, int H, int W, AdjWs w)
{
    __shared__ unsigned long long s_set[CTA_SLOTS];
    cta_set_clear(s_set);
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p < (size_t)D * H * W) {
        const int x = (int)(p % W), y = (int)((p / W) % H), z = (int)(p / ((size_t)H * W));
        const int l = seg[p];
        if (x + 1 < W) { const int r = seg[p + 1]; if (r != l) cta_set_insert(s_set, w, edge_key(l, r)); }
        if (y + 1 < H) { const int d = seg[p + W]; if (d != l) cta_set_insert(s_set, w, edge_key(l, d)); }
        if (z + 1 < D) { const int b = seg[p + (size_t)H * W]; if (b != l) cta_set_insert(s_set, w, edge_key(l, b)); }
    }
    cta_set_flush(s_set, w);
}

// centroids (z, y, x) of the labels of a volume, (-1, -1, -1) for absent labels (superpixels.py:205-242 for 3-D input)
__global__ void k_centroid3d_acc(const int* __restrict__ seg, int D, int H, int W, unsigned long long* acc)
{
    size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (size_t)D * H * W) return;
    const int x = (int)(p % W), y = (int)((p / W) % H), z = (int)(p / ((size_t)H * W));
    unsigned long long* a = acc + 4 * (size_t)seg[p];
    atomicAdd(a, 1ull); atomicAdd(a + 1, (unsigned long long)z); atomicAdd(a + 2, (unsigned long long)y); atomicAdd(a + 3, (unsigned long long)x);
}

__global__ void k_centroid3d_fin(int nb, const unsigned long long* acc, double* centres)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nb) return;
    const double c = (double)acc[4 * (size_t)k];
    for (int d = 0; d < 3; ++d) centres[3 * (size_t)k + d] = c > 0 ? (double)acc[4 * (size_t)k + 1 + d] / c : -1.0;
}

// exclusive scan of deg -> off (single CTA)
__global__ void __launch_bounds__(1024) k_edge_offsets(int nb, AdjWs w, int cap, int* n_edges_out)
{
    const int total = cta_scan_chunks<1024, int>(nb, [&](int i) { return w.deg[i]; },
                                                 [&](int i, int off) { w.off[i] = off; w.fill[i] = 0; });
    if (threadIdx.x == 0) {
        w.off[nb] = total;
        *n_edges_out = (w.ctr[1] || total > cap) ? cap + 1 : total;
    }
}

__global__ void k_edge_fill(AdjWs w, int cap)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= w.slots) return;
    unsigned long long key = w.table[i];
    if (key == 0) return;
    int b = (int)(key >> 32), a = (int)(key & 0xffffffffu);
    int pos = w.off[b] + atomicAdd(&w.fill[b], 1);
    if (pos < cap) w.tmp_a[pos] = a;
}

// per larger endpoint b: sort the smaller endpoints and emit (a, b) rows -> edges sorted by (b, a)
__global__ void k_edge_emit(int nb, AdjWs w, int cap, int* __restrict__ edges)
{
    int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    int beg = w.off[b], end = w.off[b + 1];
    if (end > cap) return;
    for (int i = beg + 1; i < end; ++i) { // insertion sort (degree is small)
        int v = w.tmp_a[i], j = i - 1;
        while (j >= beg && w.tmp_a[j] > v) { w.tmp_a[j + 1] = w.tmp_a[j]; --j; }
        w.tmp_a[j + 1] = v;
    }
    for (int i = beg; i < end; ++i) { edges[2 * (size_t)i] = w.tmp_a[i]; edges[2 * (size_t)i + 1] = b; }
}

static int pow2_at_least(long long v) { int p = 1024; while (p < v) p <<= 1; return p; }

static size_t carve_adj(AdjWs& w, void* ws, size_t bytes, int nb, int cap)
{
    WsCarver c(ws, bytes);
    w.slots = pow2_at_least(2LL * cap);
    w.table = c.take<unsigned long long>((size_t)w.slots);
    w.ctr = c.take<int>(4);
    w.deg = c.take<int>(nb);
    w.zeroed = c.off;
    w.off = c.take<int>((size_t)nb + 1);
    w.fill = c.take<int>(nb);
    w.tmp_a = c.take<int>(cap);
    return isb_align(c.off);
}

// ------------------------------------------------------------------ energies -------------------------------------------------------

__device__ double block_sum(double v, double* s_red)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += s_red[i];
    return t;
}

__device__ double block_max(double v, double* s_red)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = s_red[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) t = fmax(t, s_red[i]);
    return t;
}

constexpr int ECL = 8;   // CTAs of the energy kernel's thread-block cluster
// The cluster kernels below declare __launch_bounds__(1024, 1): with the thread bound alone, nvcc 12.9 gives k_gc_energies 32 registers
// and 56 bytes of spills; with one CTA per SM stated it takes 64 registers and spills nothing.  1024 threads
// at 64 registers fill an SM's register file, so such a CTA runs alone on its SM either way.

// the four global quantities of the energy construction (largest unary, mean / deviation of the edge distances, largest weight) are
// reduced over the cluster through distributed shared memory: partials added / compared in rank order, the same value in every CTA
__device__ double cluster_reduce(double v, bool is_max, double* s_red, double* s_x)
{
    const double t = is_max ? block_max(v, s_red) : block_sum(v, s_red);
    cg::cluster_group cl = cg::this_cluster();
    if (threadIdx.x == 0) *s_x = t;
    cl.sync();
    double tot = is_max ? -1.0 : 0.0;
    for (int r = 0; r < ECL; ++r) { const double pr = *cl.map_shared_rank(s_x, r); tot = is_max ? fmax(tot, pr) : tot + pr; }
    cl.sync();
    return tot;
}

// the clamped weight of every edge (reference graph_cuts.py:574-657) into edge_w [E], run by every thread of the cluster: the distance
// of the two endpoints' rows of vfeat [., ld] by `metric` (0 none, 1 lT, 2 l1, 3 l2), w = exp(-d / (2 std(d)^2)) with numpy's
// population std (mean first, then the mean of the squared deviations, each reduced over the cluster), divided by the relative
// centroid distance when `spatial` is set, clamped to [1e-3, 1e3] by comparisons that leave a NaN weight NaN.  sp [E]: scratch.
__device__ __forceinline__ void cluster_edge_weights(const int* __restrict__ edges, int E, const double* __restrict__ centres, const double* __restrict__ vfeat,
                                     int D, int ld, int metric, int spatial, double* edge_w, double* sp, double* s_red, double* s_x, int tid,
                                     int nth)
{
    double dsum = 0.0, ssum = 0.0;
    for (int e = tid; e < E; e += nth) {
        int a = edges[2 * e], b = edges[2 * e + 1];
        double dist = 0.0;
        if (metric != 0) {
            const double* va = vfeat + (size_t)a * ld;
            const double* vb = vfeat + (size_t)b * ld;
            for (int k = 0; k < D; ++k) {
                double df = va[k] - vb[k];
                if (metric == 1) dist = fmax(dist, df * df);        // lT: max_k (dp)^2
                else if (metric == 2) dist += fabs(df);               // l1
                else dist += df * df;                                 // l2 (sqrt below)
            }
            if (metric == 3) dist = sqrt(dist);
        }
        edge_w[e] = dist;
        dsum += dist;
        if (spatial == 3) {   // np.einsum('ij,ij->i', diff, diff) over (z, y, x), left to right
            const double cz = centres[3 * a] - centres[3 * b], cy = centres[3 * a + 1] - centres[3 * b + 1];
            const double cx = centres[3 * a + 2] - centres[3 * b + 2];
            const double s = sqrt(cz * cz + cy * cy + cx * cx);
            sp[e] = s;
            ssum += s;
        } else if (spatial) {
            double cy = centres[2 * a] - centres[2 * b], cx = centres[2 * a + 1] - centres[2 * b + 1];
            double s = sqrt(cy * cy + cx * cx);
            sp[e] = s;
            ssum += s;
        }
    }
    dsum = cluster_reduce(dsum, false, s_red, s_x);
    ssum = cluster_reduce(ssum, false, s_red, s_x);
    const double dmean = E > 0 ? dsum / E : 0.0, smean = E > 0 ? ssum / E : 1.0;
    double vsum = 0.0;
    if (metric != 0)
        for (int e = tid; e < E; e += nth) { double t = edge_w[e] - dmean; vsum += t * t; }
    vsum = cluster_reduce(vsum, false, s_red, s_x);
    const double sd = sqrt(E > 0 ? vsum / E : 0.0);
    const double denom = 2.0 * (sd * sd);
    for (int e = tid; e < E; e += nth) {
        double wv = metric != 0 ? exp(-edge_w[e] / denom) : 1.0;
        if (spatial) wv = wv / (sp[e] / smean);
        if (wv < 1e-3) wv = 1e-3;
        if (wv > 1e3) wv = 1e3;
        edge_w[e] = wv;
    }
}

// an overflowed edge table (count > capacity) holds unspecified rows: no edge is read, the host redoes the image
__device__ __forceinline__ int edge_count(const int* n_edges_dev, int E_in)
{
    return n_edges_dev ? (*n_edges_dev > E_in ? 0 : *n_edges_dev) : E_in;
}

constexpr int METRIC_GIVEN = 4;   // edge_w already holds the clamped weights (isb_gc_vector_edge_weights)

// one cluster of ECL CTAs per graph.  vfeat [N, D]: the per-vertex vectors the edge metric compares (proba for 'model').
__global__ void __cluster_dims__(ECL, 1, 1) __launch_bounds__(1024, 1) k_gc_energies(const double* __restrict__ proba, int N_in, const int* n_nodes_dev, int K, const int* __restrict__ edges, int E_in,
                                                      const int* n_edges_dev, const double* __restrict__ centres,
                                                      const double* __restrict__ vfeat, int D, int metric, int spatial,
                                                      double edge_cost, const double* __restrict__ pairwise, double* unary,
                                                      double* edge_w, int* unary_i, int* edge_wi, int* smooth_i, double* sp)
{
    __shared__ double s_red[32];
    __shared__ double s_x;
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;   // the cluster is the whole grid
    const int E = edge_count(n_edges_dev, E_in);
    const int N = n_nodes_dev ? min(*n_nodes_dev, N_in) : N_in;
    // unary = |-log(clip(p, 0.01, 0.99))|
    double umax = 0.0;
    for (int i = tid; i < N * K; i += nth) {
        double p = proba[i];
        if (p < 0.01) p = 0.01;
        if (p > 1.0 - 0.01) p = 1.0 - 0.01;
        double u = fabs(-log(p));
        unary[i] = u;
        umax = fmax(umax, fabs(u));
    }
    umax = cluster_reduce(umax, true, s_red, &s_x);
    if (metric != METRIC_GIVEN) cluster_edge_weights(edges, E, centres, vfeat, D, D, metric, spatial, edge_w, sp, s_red, &s_x, tid, nth);
    double wmax = 0.0;
    for (int e = tid; e < E; e += nth) {
        const double wv = edge_w[e] * edge_cost;
        edge_w[e] = wv;
        wmax = fmax(wmax, fabs(wv));
    }
    wmax = cluster_reduce(wmax, true, s_red, &s_x);
    double pmax = pairwise[0];
    for (int i = 1; i < K * K; ++i) pmax = fmax(pmax, pairwise[i]);
    // pyGCO: down_weight_factor = max(|unary|.max(), |w|.max() * pairwise.max()) + 1e-10
    const double dwf = fmax(umax, wmax * pmax) + 1e-10;
    for (int i = tid; i < N * K; i += nth) unary_i[i] = (int)((unary[i] / dwf) * 100000.0);
    // a degenerate edge model (std(d) = 0 with d = 0, coincident centroids under a weight of 0) leaves a NaN weight: it stays NaN in
    // edge_w as in the reference, fmax above kept it out of wmax, and its capacity is 0 (graph_cuts.integerise_energies on the host)
    for (int e = tid; e < E; e += nth) { const double wv = edge_w[e]; edge_wi[e] = isnan(wv) ? 0 : (int)((wv / dwf) * 1000.0); }
    for (int i = tid; i < K * K; i += nth) smooth_i[i] = (int)(pairwise[i] * 100.0);
}

// the 'color' / 'features' weights of compute_edge_weights over one graph (the energy kernel's cluster, without the energies)
__global__ void __cluster_dims__(ECL, 1, 1) __launch_bounds__(1024, 1) k_vector_edge_weights(const double* __restrict__ vec, int D, int ld,
                                                                                          const int* __restrict__ edges, int E_in,
                                                                                          const int* n_edges_dev,
                                                                                          const double* __restrict__ centres, int metric,
                                                                                          double* edge_w, double* sp)
{
    __shared__ double s_red[32];
    __shared__ double s_x;
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
    cluster_edge_weights(edges, edge_count(n_edges_dev, E_in), centres, vec, D, ld, metric, 1, edge_w, sp, s_red, &s_x, tid, nth);
}

// ------------------------------------------------------------------ gathers --------------------------------------------------------

constexpr int GV = 4, GW = 32 * GV; // pixels per thread and per warp of k_gather

// n_vec: the pixels covered by whole warps of GW when every pointer is 16-byte aligned (0 otherwise); the rest goes pixel by pixel.
// A warp's GW pixels are read and written as 16-byte pieces by consecutive lanes, so every store instruction covers 512 contiguous
// bytes: a lane loads four labels and stores four classes; segm_soft's GW * K values are stored in order as pairs, each lane
// looking up the labels of its pair in shared memory.
__global__ void __launch_bounds__(256) k_gather(const int* __restrict__ seg, long long n, long long n_vec, const int* __restrict__ lut_i,
                                                const double* __restrict__ lut_p, int K, int* __restrict__ out_i, double* __restrict__ out_p)
{
    __shared__ int s_lab[256 * GV];
    const long long p0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * GV;
    if (p0 >= n) return;
    if (p0 < n_vec) {
        const int4 l = *reinterpret_cast<const int4*>(seg + p0);
        if (out_i) *reinterpret_cast<int4*>(out_i + p0) = make_int4(__ldg(lut_i + l.x), __ldg(lut_i + l.y), __ldg(lut_i + l.z), __ldg(lut_i + l.w));
        if (out_p) {
            const int lane = threadIdx.x & 31;
            *reinterpret_cast<int4*>(s_lab + threadIdx.x * GV) = l;
            __syncwarp();
            const int* lab = s_lab + (threadIdx.x - lane) * GV;
            double2* dst = reinterpret_cast<double2*>(out_p + (p0 - lane * GV) * K);
            // pair i holds values 2i and 2i + 1 of the warp; value e is channel e % K of pixel e / K.  i steps by 32, e by 64.
            int q = 2 * lane / K, k = 2 * lane % K;
            const int dq = 64 / K, dk = 64 % K;
#pragma unroll 2
            for (int i = lane; i < GW * K / 2; i += 32) {
                const double v0 = __ldg(lut_p + (size_t)lab[q] * K + k);
                const int q1 = k + 1 == K ? q + 1 : q, k1 = k + 1 == K ? 0 : k + 1;
                const double v1 = __ldg(lut_p + (size_t)lab[q1] * K + k1);
                dst[i] = make_double2(v0, v1);
                q += dq; k += dk;
                if (k >= K) { k -= K; ++q; }
            }
        }
        return;
    }
    for (long long p = p0; p < min(p0 + GV, n); ++p) {
        const int l = seg[p];
        if (out_i) out_i[p] = lut_i[l];
        if (out_p) {
            const double* src = lut_p + (size_t)l * K;
            double* dst = out_p + (size_t)p * K;
            for (int k = 0; k < K; ++k) dst[k] = src[k];
        }
    }
}

} // namespace

extern "C" size_t isb_adjacency_workspace_bytes(int nb, int cap)
{
    AdjWs w;
    return carve_adj(w, nullptr, 0, nb, cap);
}

extern "C" int isb_adjacency_edges(const int32_t* seg, int H, int W, int nb, int32_t* edges, int cap, int32_t* n_edges_out, void* ws,
                                   size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(seg && edges && n_edges_out && ws, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && nb > 0 && cap > 0, "bad sizes");
    ISB_REQUIRE((H + ETH - 1) / ETH <= 65535, "label map taller than the scan grid (1 048 560 rows)");
    AdjWs w;
    size_t need = carve_adj(w, ws, ws_bytes, nb, cap);
    ISB_REQUIRE(need <= ws_bytes, "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_ADJ, st);
    ISB_CUDA_CHECK(cudaMemsetAsync(w.table, 0, w.zeroed, st));
    k_edge_scan<<<dim3((W + ETW - 1) / ETW, (H + ETH - 1) / ETH), 256, 0, st>>>(seg, H, W, w);
    ISB_LAUNCH_CHECK();
    k_edge_offsets<<<1, 1024, 0, st>>>(nb, w, cap, n_edges_out);
    ISB_LAUNCH_CHECK();
    k_edge_fill<<<(w.slots + 255) / 256, 256, 0, st>>>(w, cap);
    ISB_LAUNCH_CHECK();
    k_edge_emit<<<(nb + 127) / 128, 128, 0, st>>>(nb, w, cap, edges);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_adjacency_edges_3d(const int32_t* seg, int D, int H, int W, int nb, int32_t* edges, int cap, int32_t* n_edges_out,
                                      void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(seg && edges && n_edges_out && ws, "null pointer");
    ISB_REQUIRE(D > 0 && H > 0 && W > 0 && nb > 0 && cap > 0, "bad sizes");
    AdjWs w;
    size_t need = carve_adj(w, ws, ws_bytes, nb, cap);
    ISB_REQUIRE(need <= ws_bytes, "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_ADJ, st);
    ISB_CUDA_CHECK(cudaMemsetAsync(w.table, 0, w.zeroed, st));
    size_t n = (size_t)D * H * W;
    k_edge_scan3d<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(seg, D, H, W, w);
    ISB_LAUNCH_CHECK();
    k_edge_offsets<<<1, 1024, 0, st>>>(nb, w, cap, n_edges_out);
    ISB_LAUNCH_CHECK();
    k_edge_fill<<<(w.slots + 255) / 256, 256, 0, st>>>(w, cap);
    ISB_LAUNCH_CHECK();
    k_edge_emit<<<(nb + 127) / 128, 128, 0, st>>>(nb, w, cap, edges);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_centroids_3d(const int32_t* seg, int D, int H, int W, int nb, double* centres, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(seg && centres && ws, "null pointer");
    ISB_REQUIRE(D > 0 && H > 0 && W > 0 && nb > 0, "bad sizes");
    ISB_REQUIRE(ws_bytes >= sizeof(unsigned long long) * 4 * (size_t)nb, "workspace too small (4 * nb uint64)");
    cudaStream_t st = (cudaStream_t)stream;
    ISB_CUDA_CHECK(cudaMemsetAsync(ws, 0, sizeof(unsigned long long) * 4 * (size_t)nb, st));
    size_t n = (size_t)D * H * W;
    k_centroid3d_acc<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(seg, D, H, W, (unsigned long long*)ws);
    ISB_LAUNCH_CHECK();
    k_centroid3d_fin<<<(nb + 255) / 256, 256, 0, st>>>(nb, (const unsigned long long*)ws, centres);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" size_t isb_gc_energies_workspace_bytes(int N, int K, int E) { return isb_align(sizeof(double) * (size_t)(E > 0 ? E : 1)); }

extern "C" int isb_gc_energies(const double* proba, int N, const int32_t* n_nodes_dev, int K, const int32_t* edges, int E, const int32_t* n_edges_dev,
                               const double* centres, int metric, int spatial, double edge_cost, const double* pairwise, double* unary,
                               double* edge_w, int32_t* unary_i, int32_t* edge_wi, int32_t* smooth_i, void* ws, size_t ws_bytes,
                               isb_stream_t stream)
{
    ISB_REQUIRE(proba && edges && pairwise && unary && edge_w && unary_i && edge_wi && smooth_i && ws, "null pointer");
    ISB_REQUIRE(N > 0 && K > 0 && E >= 0, "bad sizes");
    ISB_REQUIRE(metric >= 0 && metric <= METRIC_GIVEN, "metric must be 0..4");
    ISB_REQUIRE(metric != METRIC_GIVEN || !spatial, "given edge weights (metric 4) are already spatially normalised: spatial must be 0");
    ISB_REQUIRE(spatial >= 0 && spatial <= 3, "spatial must be 0 (off), 1 or 2 (centres [N, 2]) or 3 (centres [N, 3])");
    ISB_REQUIRE(!spatial || centres, "centres are required for spatially normalised edge weights");
    ISB_REQUIRE(ws_bytes >= isb_gc_energies_workspace_bytes(N, K, E), "workspace too small");
    ProfScope prof(ISB_PROF_ENERGY, (cudaStream_t)stream);
    k_gc_energies<<<ECL, 1024, 0, (cudaStream_t)stream>>>(proba, N, n_nodes_dev, K, edges, E, n_edges_dev, centres, proba, K, metric, spatial, edge_cost,
                                                         pairwise, unary, edge_w, unary_i, edge_wi, smooth_i, (double*)ws);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_gc_vector_edge_weights(const double* vec, int nb, int D, int ld, const int32_t* edges, int cap, const int32_t* n_edges_dev,
                                          const double* centres, int metric, double* edge_w, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(vec && edges && centres && edge_w && ws, "null pointer");
    ISB_REQUIRE(nb > 0 && D > 0 && cap > 0, "bad sizes");
    ISB_REQUIRE(ld >= D, "ld must be >= D");
    ISB_REQUIRE(metric == 2 || metric == 3, "metric must be 2 (l1, 'color') or 3 (l2, 'features')");
    ISB_REQUIRE(ws_bytes >= isb_gc_energies_workspace_bytes(nb, 1, cap), "workspace too small");
    ProfScope prof(ISB_PROF_ENERGY, (cudaStream_t)stream);
    k_vector_edge_weights<<<ECL, 1024, 0, (cudaStream_t)stream>>>(vec, D, ld, edges, cap, n_edges_dev, centres, metric, edge_w, (double*)ws);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// np.array(image, dtype=float), divided by 255 when max(image) > 1 (compute_edge_weights' 'color' vectors): max from minmax[1] on the
// device, so a NaN maximum (numpy's np.max of an image with a NaN) compares false and leaves the image unscaled
__global__ void k_unit_scale(const void* img, int dtype, long long n, const double* minmax, double* out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double v = load_as_f64(img, dtype, (size_t)i);
    out[i] = minmax[1] > 1.0 ? v / 255.0 : v;
}

extern "C" int isb_image_unit_scale(const void* img, int dtype, long long n, const double* minmax, double* out, isb_stream_t stream)
{
    ISB_REQUIRE(img && minmax && out && n > 0, "bad arguments");
    ISB_REQUIRE(dtype >= ISB_U8 && dtype <= ISB_F64, "bad dtype");
    k_unit_scale<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(img, dtype, n, minmax, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

__global__ void k_fill_i32(int* p, long long n, int v)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

extern "C" int isb_fill_i32(int32_t* dst, long long n, int32_t value, isb_stream_t stream)
{
    ISB_REQUIRE(dst && n > 0, "bad arguments");
    k_fill_i32<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(dst, n, value);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// dst = dst (op) src on 8-byte words: the in-process stand-in for the collectives of the row-band mode (several bands on one GPU)
__global__ void k_combine(void* dst, const void* src, long long n, int op)
{
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (op == 0) ((long long*)dst)[i] += ((const long long*)src)[i];
    else if (op == 1) { long long a = ((long long*)dst)[i], b = ((const long long*)src)[i]; ((long long*)dst)[i] = a > b ? a : b; }
    else if (op == 2 || op == 3) {
        // numpy's minimum / maximum: NaN on either side gives NaN (fmin / fmax would drop it)
        const double a = ((double*)dst)[i], b = ((const double*)src)[i];
        ((double*)dst)[i] = (a != a || b != b) ? a + b : (op == 2 ? fmin(a, b) : fmax(a, b));
    }
    else ((double*)dst)[i] = ((double*)dst)[i] + ((const double*)src)[i];
}

extern "C" int isb_combine(void* dst, const void* src, long long n, int op, isb_stream_t stream)
{
    ISB_REQUIRE(dst && src && n > 0 && op >= 0 && op <= 4, "bad arguments");
    k_combine<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(dst, src, n, op);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_gather(const int32_t* seg, long long npx, const int32_t* lut_i, const double* lut_p, int K, int32_t* out_i,
                          double* out_p, isb_stream_t stream)
{
    ISB_REQUIRE(seg && npx > 0, "bad arguments");
    ISB_REQUIRE((!out_i || lut_i) && (!out_p || (lut_p && K > 0)), "LUT missing for a requested output");
    ProfScope prof(ISB_PROF_GATHER, (cudaStream_t)stream);
    const bool aligned = (((uintptr_t)seg | (uintptr_t)out_i | (uintptr_t)out_p) & 15) == 0;
    const long long groups = (npx + GV - 1) / GV;
    k_gather<<<(unsigned)((groups + 255) / 256), 256, 0, (cudaStream_t)stream>>>(seg, npx, aligned ? npx / GW * GW : 0, lut_i, lut_p, K,
                                                                                out_i, out_p);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
