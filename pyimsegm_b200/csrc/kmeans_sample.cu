// kmeans_sample.cu -- the k-means of down_sample_dict_features_kmean (imsegm/classification.py:1110-1134): Lloyd runs of
// scikit-learn's KMeans(init='random', n_init=3, max_iter=5) on centred features, and the sample nearest to every final centre.
//
// One isb_kmeans_lloyd call enqueues every sweep of a run without reading anything back: each sweep's kernels first read the
// run's status word and do nothing once the run has stopped, so the host synchronises once per run.  A sweep that leaves a
// cluster empty stops the run with status 3 and hands its sums to the host, which relocates the empty clusters as
// scikit-learn's _relocate_empty_clusters_dense does and continues the run with a second call.
//
// Per sweep:
//   k_km_norms   |c_j|^2
//   k_km_assign  label = argmin_j |c_j|^2 - 2 x.c_j (lowest j on ties): X.C^T on the FP64 tensor cores (mma.sync m8n8k4), 128 rows
//                x 64 centres per CTA, K streamed in 32-wide chunks through a two-stage cp.async ring, the row argmin fused into the
//                epilogue -- no n x k matrix is written
//   radix sort   (label, sample index) pairs; the sort is stable, so every cluster's members come out in ascending index order
//   k_km_sums    one warp per cluster adds its members' rows in that order: sums that are the same bits on every run
//   k_km_update  centre = sum * (1 / count) and its shift, unless a cluster is empty
//   k_km_converge  strict convergence (no label changed), else sum shift^2 <= tol, else the next sweep
// then the final E-step of a run that did not converge strictly, and the inertia sum (x - c)^2 in a fixed order.
#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>

namespace {

constexpr int KM_DMAX = 256;                 // widest feature row (the widest feature table of the package has 232 columns)
constexpr int AM = 128, AN = 64, AK = 32;    // assignment tile: rows x centres x depth chunk
constexpr int AS = AK + 4;                   // smem row stride: the 8 rows x 4 columns of a fragment load hit each bank pair twice
constexpr int A_THREADS = 256;               // 8 warps, 4 (rows) x 2 (centres), 32 x 32 outputs each
constexpr size_t A_SMEM = 2ull * (AM + AN) * AS * sizeof(double);
constexpr int NB = 64, N_THREADS = 256;      // nearest-sample tile: 64 samples x 64 centres, 4 x 4 per thread
constexpr int R_THREADS = 256;               // reductions

// status[0]: 0 running, 1 strict convergence, 2 shift within tol, 3 stopped on an empty cluster, 4 max_iter sweeps done;
// status[1]: sweeps done; status[2]: labels changed in the current sweep; status[3]: empty clusters in the current sweep
enum { ST_RUN = 0, ST_STRICT = 1, ST_TOL = 2, ST_EMPTY = 3, ST_MAXITER = 4 };

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

struct KmWs {
    double *xp, *cp, *cnorm, *shift, *partial;
    uint32_t *keys, *idx_in, *idx_sorted;
    unsigned long long* dmin;
    void* sort_tmp;
    size_t sort_bytes, need;
};

int sort_bits(int k)
{
    int b = 1;
    while ((1ll << b) < k) ++b;
    return b;
}

KmWs carve(void* base, int n, int k, int D)
{
    const int n_pad = round_up(n, AM), k_pad = round_up(k, AN), Dp = round_up(D, AK);
    WsCarver c(base, ~size_t(0));
    KmWs w;
    w.xp = c.take<double>((size_t)n_pad * Dp);
    w.cp = c.take<double>((size_t)k_pad * Dp);
    w.cnorm = c.take<double>(k_pad);
    w.shift = c.take<double>(k);
    w.partial = c.take<double>((n + R_THREADS - 1) / R_THREADS);
    w.keys = c.take<uint32_t>(n);
    w.idx_in = c.take<uint32_t>(n);
    w.idx_sorted = c.take<uint32_t>(n);
    w.dmin = c.take<unsigned long long>(k);
    w.sort_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, w.sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                    (uint32_t*)nullptr, n, 0, sort_bits(k));
    w.sort_tmp = c.take<char>(w.sort_bytes);
    w.need = c.off;
    return w;
}

// dst [rows_pad, Dp] = src [rows, D] with zero rows and columns around it
__global__ void k_km_pad(const double* __restrict__ src, int rows, int D, int rows_pad, int Dp, double* __restrict__ dst)
{
    const size_t total = (size_t)rows_pad * Dp;
    for (size_t q = blockIdx.x * (size_t)blockDim.x + threadIdx.x; q < total; q += (size_t)gridDim.x * blockDim.x) {
        const size_t r = q / Dp;
        const int d = (int)(q % Dp);
        dst[q] = (r < (size_t)rows && d < D) ? src[r * D + d] : 0.0;
    }
}

__global__ void k_km_unpad(const double* __restrict__ src, int rows, int D, int Dp, double* __restrict__ dst)
{
    const size_t total = (size_t)rows * D;
    for (size_t q = blockIdx.x * (size_t)blockDim.x + threadIdx.x; q < total; q += (size_t)gridDim.x * blockDim.x)
        dst[q] = src[(q / D) * Dp + q % D];
}

__global__ void k_km_iota(uint32_t* __restrict__ idx, int n)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) idx[i] = (uint32_t)i;
}

// the assignment's condition on the status: a sweep runs while the status is ST_RUN; the final E-step after a run that stopped
// without strict convergence
template <bool final_estep>
__device__ __forceinline__ bool assign_runs(const int32_t* status)
{
    const int st = status[0];
    return final_estep ? (st == ST_TOL || st == ST_MAXITER) : (st == ST_RUN);
}

template <bool final_estep>
__global__ void k_km_norms(const double* __restrict__ cp, int k, int D, int Dp, double* __restrict__ cnorm, const int32_t* __restrict__ status)
{
    if (!assign_runs<final_estep>(status)) return;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= k) return;
    const double* c = cp + (size_t)j * Dp;
    double s = 0.0;
    for (int d = 0; d < D; ++d) s = __fma_rn(c[d], c[d], s);
    cnorm[j] = s;
}

__device__ __forceinline__ void mma_f64(double (&acc)[2], double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n"
                 : "+d"(acc[0]), "+d"(acc[1])
                 : "d"(a), "d"(b));
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem)
{
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_one() { asm volatile("cp.async.wait_group 1;\n" ::); }

// (v, j) < (bv, bj) lexicographically
__device__ __forceinline__ void take_min(double& bv, int& bj, double v, int j)
{
    if (v < bv || (v == bv && j < bj)) { bv = v; bj = j; }
}

// labels[i] = argmin_j (cnorm[j] - 2 x_i . c_j) over j < k, lowest j on ties; a sweep also counts the labels that change
template <bool final_estep>
__global__ void __launch_bounds__(A_THREADS, 2)
k_km_assign(const double* __restrict__ xp, int n, const double* __restrict__ cp, const double* __restrict__ cnorm, int k, int Dp,
            int32_t* __restrict__ labels, int32_t* __restrict__ status)
{
    if (!assign_runs<final_estep>(status)) return;
    extern __shared__ __align__(16) double sm[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wr = warp >> 1, wc = warp & 1;            // warp rows wr*32.., warp centres wc*32..
    const int row0 = blockIdx.x * AM;
    const int nkc = Dp / AK, n_tiles = (k + AN - 1) / AN, T = n_tiles * nkc;

    auto load = [&](int t, int buf) {
        const int jt = t / nkc, kc = (t % nkc) * AK;
        double* s = sm + (size_t)buf * (AM + AN) * AS;
        const double* gx = xp + (size_t)row0 * Dp + kc;
        const double* gc = cp + (size_t)jt * AN * Dp + kc;
        for (int q = tid; q < (AM + AN) * (AK / 2); q += A_THREADS) {
            const int r = q / (AK / 2), c2 = (q % (AK / 2)) * 2;
            const double* g = (r < AM) ? gx + (size_t)r * Dp + c2 : gc + (size_t)(r - AM) * Dp + c2;
            cp_async16(s + r * AS + c2, g);
        }
        cp_async_commit();
    };

    double best[4];
    int bidx[4];
#pragma unroll
    for (int mi = 0; mi < 4; ++mi) { best[mi] = __longlong_as_double(0x7ff0000000000000ll); bidx[mi] = 0; }
    double acc[4][4][2];

    load(0, 0);
    for (int t = 0; t < T; ++t) {
        if (t % nkc == 0) {
#pragma unroll
            for (int mi = 0; mi < 4; ++mi)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) acc[mi][ni][0] = acc[mi][ni][1] = 0.0;
        }
        if (t + 1 < T) load(t + 1, (t + 1) & 1);
        else cp_async_commit();
        cp_async_wait_one();
        __syncthreads();
        const double* sa = sm + (size_t)(t & 1) * (AM + AN) * AS + (wr * 32 + (lane >> 2)) * AS + (lane & 3);
        const double* sb = sm + (size_t)(t & 1) * (AM + AN) * AS + (AM + wc * 32 + (lane >> 2)) * AS + (lane & 3);
#pragma unroll
        for (int ks = 0; ks < AK; ks += 4) {
            double a[4], b[4];
#pragma unroll
            for (int mi = 0; mi < 4; ++mi) a[mi] = sa[mi * 8 * AS + ks];
#pragma unroll
            for (int ni = 0; ni < 4; ++ni) b[ni] = sb[ni * 8 * AS + ks];
#pragma unroll
            for (int mi = 0; mi < 4; ++mi)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) mma_f64(acc[mi][ni], a[mi], b[ni]);
        }
        if (t % nkc == nkc - 1) {
            // thread's columns in ascending order, so a strict < keeps the lowest index among equal values
            const int jbase = (t / nkc) * AN + wc * 32 + (lane & 3) * 2;
#pragma unroll
            for (int ni = 0; ni < 4; ++ni)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int j = jbase + ni * 8 + e;
                    if (j < k) {
                        const double cn = cnorm[j];
#pragma unroll
                        for (int mi = 0; mi < 4; ++mi) {
                            const double v = __fma_rn(-2.0, acc[mi][ni][e], cn);
                            if (v < best[mi]) { best[mi] = v; bidx[mi] = j; }
                        }
                    }
                }
        }
        __syncthreads();
    }
    // the four lanes of a row, then the two warps of a row
#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, best[mi], o);
            const int oj = __shfl_xor_sync(0xffffffffu, bidx[mi], o);
            take_min(best[mi], bidx[mi], ov, oj);
        }
    double* sv = sm;                                     // [2][AM] values, then [2][AM] indices
    int* sj = (int*)(sm + 2 * AM);
    if ((lane & 3) == 0) {
#pragma unroll
        for (int mi = 0; mi < 4; ++mi) {
            const int r = wr * 32 + mi * 8 + (lane >> 2);
            sv[wc * AM + r] = best[mi];
            sj[wc * AM + r] = bidx[mi];
        }
    }
    __syncthreads();
    int changed = 0;
    if (tid < AM && row0 + tid < n) {
        double v = sv[tid];
        int j = sj[tid];
        take_min(v, j, sv[AM + tid], sj[AM + tid]);
        if (!final_estep) changed = labels[row0 + tid] != j;
        labels[row0 + tid] = j;
    }
    if (!final_estep) {
        const int c = __syncthreads_count(changed);
        if (tid == 0 && c) atomicAdd(status + 2, c);
    }
}

// one warp per cluster: members (ascending sample index) from the sorted pairs, their rows added in that order
__global__ void k_km_sums(const double* __restrict__ xp, int D, int Dp, const uint32_t* __restrict__ keys, const uint32_t* __restrict__ idx,
                          int n, int k, double* __restrict__ sums, int32_t* __restrict__ counts, int32_t* __restrict__ status)
{
    if (status[0] != ST_RUN) return;
    const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (j >= k) return;
    auto lower = [&](uint32_t key) {
        int lo = 0, hi = n;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (keys[mid] < key) lo = mid + 1;
            else hi = mid;
        }
        return lo;
    };
    const int lo = lower((uint32_t)j), hi = lower((uint32_t)j + 1);
    double acc[KM_DMAX / 32];
#pragma unroll
    for (int q = 0; q < KM_DMAX / 32; ++q) acc[q] = 0.0;
    int m = lo;
    for (; m + 4 <= hi; m += 4) {                        // four rows in flight, added in order
        double v[4][KM_DMAX / 32];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const double* x = xp + (size_t)idx[m + u] * Dp;
#pragma unroll
            for (int q = 0; q < KM_DMAX / 32; ++q) v[u][q] = (lane + 32 * q < Dp) ? x[lane + 32 * q] : 0.0;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int q = 0; q < KM_DMAX / 32; ++q) acc[q] += v[u][q];
    }
    for (; m < hi; ++m) {
        const double* x = xp + (size_t)idx[m] * Dp;
#pragma unroll
        for (int q = 0; q < KM_DMAX / 32; ++q)
            if (lane + 32 * q < Dp) acc[q] += x[lane + 32 * q];
    }
#pragma unroll
    for (int q = 0; q < KM_DMAX / 32; ++q)
        if (lane + 32 * q < D) sums[(size_t)j * D + lane + 32 * q] = acc[q];
    if (lane == 0) {
        counts[j] = hi - lo;
        if (hi == lo) atomicAdd(status + 3, 1);
    }
}

// centre = sum * (1 / count) (scikit-learn's _average_centers) and shift_j = |new - old|, one warp per cluster; a sweep with an
// empty cluster stops the run for the host instead
__global__ void k_km_update(double* __restrict__ cp, int D, int Dp, const double* __restrict__ sums, const int32_t* __restrict__ counts,
                            int k, double* __restrict__ shift, int32_t* __restrict__ status)
{
    if (status[0] != ST_RUN) return;
    if (status[3] != 0) {
        if (blockIdx.x == 0 && threadIdx.x == 0) status[0] = ST_EMPTY;
        return;
    }
    const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (j >= k) return;
    const double alpha = 1.0 / (double)counts[j];
    double ss = 0.0;
    for (int d = lane; d < D; d += 32) {
        const double nv = sums[(size_t)j * D + d] * alpha;
        const double diff = nv - cp[(size_t)j * Dp + d];
        ss = __fma_rn(diff, diff, ss);
        cp[(size_t)j * Dp + d] = nv;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if (lane == 0) shift[j] = sqrt(ss);
}

// fixed-order block sum (blockDim.x == R_THREADS)
__device__ double block_sum(double v)
{
    __shared__ double red[R_THREADS];
    red[threadIdx.x] = v;
    __syncthreads();
    for (int s = R_THREADS / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    return red[0];
}

__global__ void k_km_converge(const double* __restrict__ shift, int k, double tol, int max_iter, int32_t* __restrict__ status)
{
    if (status[0] != ST_RUN) return;
    double v = 0.0;
    for (int j = threadIdx.x; j < k; j += R_THREADS) v = __fma_rn(shift[j], shift[j], v);
    const double tot = block_sum(v);
    if (threadIdx.x == 0) {
        int st = ST_RUN;
        if (status[2] == 0) st = ST_STRICT;
        else if (tot <= tol) st = ST_TOL;
        const int sweeps = status[1] + 1;
        if (st == ST_RUN && sweeps >= max_iter) st = ST_MAXITER;
        status[0] = st;
        status[1] = sweeps;
        status[2] = 0;
        status[3] = 0;
    }
}

// inertia = sum_i |x_i - c_{label_i}|^2: per-block partial sums, then one block adds them in order
__global__ void k_km_inertia_part(const double* __restrict__ xp, int n, int D, int Dp, const double* __restrict__ cp,
                                  const int32_t* __restrict__ labels, double* __restrict__ partial, const int32_t* __restrict__ status)
{
    const int st = status[0];
    if (st == ST_RUN || st == ST_EMPTY) return;
    const int i = blockIdx.x * R_THREADS + threadIdx.x;
    double s = 0.0;
    if (i < n) {
        const double* x = xp + (size_t)i * Dp;
        const double* c = cp + (size_t)labels[i] * Dp;
        for (int d = 0; d < D; ++d) {
            const double diff = x[d] - c[d];
            s = __fma_rn(diff, diff, s);
        }
    }
    const double tot = block_sum(s);
    if (threadIdx.x == 0) partial[blockIdx.x] = tot;
}

__global__ void k_km_inertia_final(const double* __restrict__ partial, int n_part, double* __restrict__ inertia,
                                   const int32_t* __restrict__ status)
{
    const int st = status[0];
    if (st == ST_RUN || st == ST_EMPTY) return;
    double v = 0.0;
    for (int q = threadIdx.x; q < n_part; q += R_THREADS) v += partial[q];
    const double tot = block_sum(v);
    if (threadIdx.x == 0) inertia[0] = tot;
}

// exact squared distances of a 64-sample x 64-centre tile, features added in order; pass 0 lowers dmin[j] to the least distance of
// centre j, pass 1 lowers nearest[j] to the least sample index at that distance
template <int pass>
__global__ void __launch_bounds__(N_THREADS)
k_km_nearest(const double* __restrict__ xp, int n, const double* __restrict__ cp, int k, int D, int Dp,
             unsigned long long* __restrict__ dmin, int32_t* __restrict__ nearest)
{
    __shared__ double sx[NB][AK + 1], sc[NB][AK + 1];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int i0 = blockIdx.x * NB, j0 = blockIdx.y * NB;
    double acc[4][4] = {};
    for (int kc = 0; kc < D; kc += AK) {
        for (int q = threadIdx.x; q < NB * AK; q += N_THREADS) {
            const int r = q / AK, c = q % AK;
            sx[r][c] = xp[(size_t)(i0 + r) * Dp + kc + c];   // rows padded to AM (a multiple of NB), columns to Dp
            sc[r][c] = cp[(size_t)(j0 + r) * Dp + kc + c];
        }
        __syncthreads();
        const int kn = min(AK, D - kc);
        for (int c = 0; c < kn; ++c) {
            double xv[4], cv[4];
#pragma unroll
            for (int a = 0; a < 4; ++a) xv[a] = sx[ty + 16 * a][c];
#pragma unroll
            for (int b = 0; b < 4; ++b) cv[b] = sc[tx + 16 * b][c];
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    const double diff = xv[a] - cv[b];
                    acc[a][b] = __fma_rn(diff, diff, acc[a][b]);
                }
        }
        __syncthreads();
    }
#pragma unroll
    for (int b = 0; b < 4; ++b) {
        const int j = j0 + tx + 16 * b;
        if (j >= k) continue;
        if (pass == 0) {
            unsigned long long m = ~0ull;
#pragma unroll
            for (int a = 0; a < 4; ++a)
                if (i0 + ty + 16 * a < n) m = min(m, f64_ordered(acc[a][b]));
            if (m != ~0ull) atomicMin(dmin + j, m);
        } else {
            const unsigned long long m = dmin[j];
            int best = 0x7fffffff;
#pragma unroll
            for (int a = 0; a < 4; ++a) {
                const int i = i0 + ty + 16 * a;
                if (i < n && f64_ordered(acc[a][b]) == m) best = min(best, i);
            }
            if (best != 0x7fffffff) atomicMin(nearest + j, best);
        }
    }
}

__global__ void k_km_nearest_init(unsigned long long* __restrict__ dmin, int32_t* __restrict__ nearest, int k)
{
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < k; j += gridDim.x * blockDim.x) {
        dmin[j] = ~0ull;
        nearest[j] = 0x7fffffff;
    }
}

int check_sizes(int n, int k, int D)
{
    ISB_REQUIRE(n >= 1 && k >= 1 && k <= n && D >= 1, "need n >= k >= 1 and D >= 1");
    if (D > KM_DMAX || n > (1 << 30) || k > NB * 65535) {
        isb_set_error("k-means of %d centres over %d samples of %d features: at most %d features, 2^30 samples and %d centres", k, n, D,
                      KM_DMAX, NB * 65535);
        return ISB_ERR_UNSUPPORTED;
    }
    return ISB_OK;
}

int grid_of(size_t work, int threads)
{
    const size_t g = (work + threads - 1) / threads;
    return (int)(g < (1u << 16) ? g : (1u << 16));
}

} // namespace

extern "C" size_t isb_kmeans_workspace_bytes(int n, int k, int D)
{
    if (check_sizes(n, k, D) != ISB_OK) return 0;
    return carve(nullptr, n, k, D).need;
}

extern "C" int isb_kmeans_lloyd(const double* X, int n, int D, int k, int max_iter, int sweeps, double tol, double* centres, int32_t* labels,
                                int32_t* status, double* sums, int32_t* counts, double* inertia, void* ws, size_t ws_bytes,
                                isb_stream_t stream)
{
    if (int s = check_sizes(n, k, D)) return s;
    ISB_REQUIRE(X && centres && labels && status && sums && counts && inertia && ws, "null pointer");
    ISB_REQUIRE(max_iter >= 1, "max_iter must be >= 1");
    ISB_REQUIRE(sweeps >= 0 && sweeps <= max_iter, "sweeps must be in [0, max_iter]");
    ISB_REQUIRE(ws_bytes >= isb_kmeans_workspace_bytes(n, k, D), "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const KmWs w = carve(ws, n, k, D);
    const int n_pad = round_up(n, AM), k_pad = round_up(k, AN), Dp = round_up(D, AK);
    k_km_pad<<<grid_of((size_t)n_pad * Dp, 256), 256, 0, st>>>(X, n, D, n_pad, Dp, w.xp);
    ISB_LAUNCH_CHECK();
    k_km_pad<<<grid_of((size_t)k_pad * Dp, 256), 256, 0, st>>>(centres, k, D, k_pad, Dp, w.cp);
    ISB_LAUNCH_CHECK();
    k_km_iota<<<grid_of(n, 256), 256, 0, st>>>(w.idx_in, n);
    ISB_LAUNCH_CHECK();
    ISB_CUDA_CHECK(cudaFuncSetAttribute(k_km_assign<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)A_SMEM));
    ISB_CUDA_CHECK(cudaFuncSetAttribute(k_km_assign<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)A_SMEM));
    const int warp_blocks = (int)(((size_t)k * 32 + 255) / 256);
    // the radix sort does not read the status: a sweep enqueued after the run has stopped still sorts the n pairs (its other
    // kernels return at once), so the caller enqueues only the sweeps the run can still do
    for (int it = 0; it < sweeps; ++it) {
        k_km_norms<false><<<(k + 255) / 256, 256, 0, st>>>(w.cp, k, D, Dp, w.cnorm, status);
        ISB_LAUNCH_CHECK();
        k_km_assign<false><<<n_pad / AM, A_THREADS, A_SMEM, st>>>(w.xp, n, w.cp, w.cnorm, k, Dp, labels, status);
        ISB_LAUNCH_CHECK();
        size_t sort_bytes = w.sort_bytes;
        ISB_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(w.sort_tmp, sort_bytes, (const uint32_t*)labels, w.keys, w.idx_in, w.idx_sorted, n, 0,
                                                       sort_bits(k), st));
        ISB_LAUNCH_CHECK();
        k_km_sums<<<warp_blocks, 256, 0, st>>>(w.xp, D, Dp, w.keys, w.idx_sorted, n, k, sums, counts, status);
        ISB_LAUNCH_CHECK();
        k_km_update<<<warp_blocks, 256, 0, st>>>(w.cp, D, Dp, sums, counts, k, w.shift, status);
        ISB_LAUNCH_CHECK();
        k_km_converge<<<1, R_THREADS, 0, st>>>(w.shift, k, tol, max_iter, status);
        ISB_LAUNCH_CHECK();
    }
    k_km_norms<true><<<(k + 255) / 256, 256, 0, st>>>(w.cp, k, D, Dp, w.cnorm, status);
    ISB_LAUNCH_CHECK();
    k_km_assign<true><<<n_pad / AM, A_THREADS, A_SMEM, st>>>(w.xp, n, w.cp, w.cnorm, k, Dp, labels, status);
    ISB_LAUNCH_CHECK();
    const int n_part = (n + R_THREADS - 1) / R_THREADS;
    k_km_inertia_part<<<n_part, R_THREADS, 0, st>>>(w.xp, n, D, Dp, w.cp, labels, w.partial, status);
    ISB_LAUNCH_CHECK();
    k_km_inertia_final<<<1, R_THREADS, 0, st>>>(w.partial, n_part, inertia, status);
    ISB_LAUNCH_CHECK();
    k_km_unpad<<<grid_of((size_t)k * D, 256), 256, 0, st>>>(w.cp, k, D, Dp, centres);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_kmeans_nearest(const double* X, int n, int D, const double* centres, int k, int32_t* nearest, void* ws, size_t ws_bytes,
                                  isb_stream_t stream)
{
    if (int s = check_sizes(n, k, D)) return s;
    ISB_REQUIRE(X && centres && nearest && ws, "null pointer");
    ISB_REQUIRE(ws_bytes >= isb_kmeans_workspace_bytes(n, k, D), "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const KmWs w = carve(ws, n, k, D);
    const int n_pad = round_up(n, AM), k_pad = round_up(k, AN), Dp = round_up(D, AK);
    k_km_pad<<<grid_of((size_t)n_pad * Dp, 256), 256, 0, st>>>(X, n, D, n_pad, Dp, w.xp);
    ISB_LAUNCH_CHECK();
    k_km_pad<<<grid_of((size_t)k_pad * Dp, 256), 256, 0, st>>>(centres, k, D, k_pad, Dp, w.cp);
    ISB_LAUNCH_CHECK();
    k_km_nearest_init<<<grid_of(k, 256), 256, 0, st>>>(w.dmin, nearest, k);
    ISB_LAUNCH_CHECK();
    const dim3 grid((n + NB - 1) / NB, (k + NB - 1) / NB);
    k_km_nearest<0><<<grid, N_THREADS, 0, st>>>(w.xp, n, w.cp, k, D, Dp, w.dmin, nearest);
    ISB_LAUNCH_CHECK();
    k_km_nearest<1><<<grid, N_THREADS, 0, st>>>(w.xp, n, w.cp, k, D, Dp, w.dmin, nearest);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
