// class_models.cu -- predict_proba of a caller-fitted class model on the device (the shared-model entry point of the reference,
// imsegm/pipelines.py:160-241, with a model from estim_model_classes_group or a trained classifier): the feature transform of the
// model's Pipeline (NaN -> 0, StandardScaler, PCA) and the decision-tree / random-forest, k-nearest-neighbour and logistic-regression
// evaluations.  The tables are compiled on the
// host by pyimsegm_b200/class_models.py.  The mixture evaluation lives in gmm.cu, next to the FP64 GEMM it shares with the fit.
// Nothing here synchronises with the host or allocates, so the calls can be captured in a CUDA graph.
#include <climits>
#include <math_constants.h>

#include "common.cuh"

namespace {

constexpr int FOREST_KMAX = 64;   // classes of a tree model (the alpha-expansion limit)

inline int grid_for(size_t n, int threads)
{
    const size_t b = (n + threads - 1) / threads;
    return (int)(b < 4096 ? (b > 0 ? b : 1) : 4096);
}

// NaN -> 0 (pipelines.py: features[np.isnan(features)] = 0), then StandardScaler.transform: x -= mean_; x /= scale_ (either optional)
__global__ void k_cm_scale(const double* __restrict__ feat, int N_in, const int* n_dev, int D, int ld, const double* __restrict__ mean,
                           const double* __restrict__ scale, double* __restrict__ out)
{
    const int N = n_dev ? min(*n_dev, N_in) : N_in;
    const size_t total = (size_t)N * D;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t n = i / D;
        const int d = (int)(i % D);
        double v = feat[n * ld + d];
        if (isnan(v)) v = 0.0;
        if (mean) v = v - mean[d];
        if (scale) v = v / scale[d];
        out[i] = v;
    }
}

// PCA.transform as scikit-learn orders it: X C^T - (mean_ C^T), then / max(sqrt(explained_variance_), eps) when whitening.
// One thread per (sample, component); the host passes mean_ C^T and the clipped scale.
__global__ void k_cm_pca(const double* __restrict__ xs, int N_in, const int* n_dev, int D_in, int D_out, const double* __restrict__ comp,
                         const double* __restrict__ pmean, const double* __restrict__ pscale, double* __restrict__ out)
{
    const int N = n_dev ? min(*n_dev, N_in) : N_in;
    const size_t total = (size_t)N * D_out;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t n = i / D_out;
        const int j = (int)(i % D_out);
        const double* x = xs + n * D_in;
        const double* c = comp + (size_t)j * D_in;
        double acc = 0.0;
        for (int k = 0; k < D_in; ++k) acc = fma(x[k], c[k], acc);
        acc = acc - pmean[j];
        if (pscale) acc = acc / pscale[j];
        out[i] = acc;
    }
}

// one thread per (sample, tree): the leaf the sample reaches.  sklearn casts X to float32 before the trees see it
// (_validate_X_predict) and compares that value, widened, against the float64 threshold: x <= t goes left.
__global__ void k_forest_leaves(const double* __restrict__ x, int N_in, const int* n_dev, int D, int T, const int* __restrict__ roots,
                                const int* __restrict__ feature, const double* __restrict__ thr, const int* __restrict__ left,
                                const int* __restrict__ right, int n_nodes, int* __restrict__ leaf)
{
    const int N = n_dev ? min(*n_dev, N_in) : N_in;
    const size_t total = (size_t)N * T;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t n = i / T;
        const double* xr = x + n * D;
        int node = roots[i % T];
        for (int step = 0; step < n_nodes && left[node] >= 0; ++step) {
            const double v = (double)(float)xr[feature[node]];
            node = v <= thr[node] ? left[node] : right[node];
        }
        leaf[i] = node;
    }
}

// one thread per (sample, class): ForestClassifier.predict_proba with n_jobs=None -- the per-tree leaf values added in estimator order
// onto zeros, then ONE division by the number of trees (average = 0: a single DecisionTreeClassifier, the leaf value itself)
__global__ void k_forest_sum(const int* __restrict__ leaf, int N_in, const int* n_dev, int T, int K, const double* __restrict__ value,
                             int average, double* __restrict__ proba)
{
    const int N = n_dev ? min(*n_dev, N_in) : N_in;
    const size_t total = (size_t)N * K;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t n = i / K;
        const int c = (int)(i % K);
        const int* lf = leaf + n * T;
        double s = 0.0;
        for (int e = 0; e < T; ++e) s = s + value[(size_t)lf[e] * K + c];
        if (average) s = s / (double)T;
        proba[i] = s;
    }
}

} // namespace

extern "C" size_t isb_class_transform_workspace_bytes(int N, int D_in, int has_pca)
{
    return has_pca ? isb_align(sizeof(double) * (size_t)(N > 0 ? N : 0) * (D_in > 0 ? D_in : 0)) : 0;
}

extern "C" int isb_class_transform(const double* feat, int N, int ld, const int32_t* n_dev, int D_in, const double* sc_mean,
                                   const double* sc_scale, const double* pca_comp, const double* pca_mean, const double* pca_scale, int D_out,
                                   double* out, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(feat && out, "null pointer");
    ISB_REQUIRE(N > 0 && D_in > 0 && ld >= D_in && D_out > 0, "bad sizes");
    if (pca_comp) {
        ISB_REQUIRE(pca_mean && ws, "null pointer");
        ISB_REQUIRE(ws_bytes >= isb_class_transform_workspace_bytes(N, D_in, 1), "workspace too small");
    } else {
        ISB_REQUIRE(D_out == D_in, "without PCA the output has the input's dimensions");
    }
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_GMM, st);
    double* xs = pca_comp ? (double*)ws : out;
    k_cm_scale<<<grid_for((size_t)N * D_in, 256), 256, 0, st>>>(feat, N, n_dev, D_in, ld, sc_mean, sc_scale, xs);
    ISB_LAUNCH_CHECK();
    if (pca_comp) {
        k_cm_pca<<<grid_for((size_t)N * D_out, 256), 256, 0, st>>>(xs, N, n_dev, D_in, D_out, pca_comp, pca_mean, pca_scale, out);
        ISB_LAUNCH_CHECK();
    }
    return ISB_OK;
}

extern "C" size_t isb_forest_predict_workspace_bytes(int N, int n_trees)
{
    return isb_align(sizeof(int32_t) * (size_t)(N > 0 ? N : 0) * (n_trees > 0 ? n_trees : 0));
}

extern "C" int isb_forest_predict_proba(const double* x, int N, const int32_t* n_dev, int D, int n_trees, const int32_t* roots,
                                        const int32_t* feature, const double* threshold, const int32_t* left, const int32_t* right, int n_nodes,
                                        const double* value, int K, int average, double* proba, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(x && roots && feature && threshold && left && right && value && proba && ws, "null pointer");
    ISB_REQUIRE(N > 0 && D > 0 && n_trees > 0 && n_nodes > 0 && K > 0, "bad sizes");
    if (K > FOREST_KMAX) { isb_set_error("device forest handles K <= %d classes (got K=%d)", FOREST_KMAX, K); return ISB_ERR_UNSUPPORTED; }
    ISB_REQUIRE(ws_bytes >= isb_forest_predict_workspace_bytes(N, n_trees), "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_GMM, st);
    int* leaf = (int*)ws;
    k_forest_leaves<<<grid_for((size_t)N * n_trees, 256), 256, 0, st>>>(x, N, n_dev, D, n_trees, roots, feature, threshold, left, right,
                                                                        n_nodes, leaf);
    ISB_LAUNCH_CHECK();
    k_forest_sum<<<grid_for((size_t)N * K, 256), 256, 0, st>>>(leaf, N, n_dev, n_trees, K, value, average, proba);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// k-nearest neighbours (KNeighborsClassifier, Euclidean).  Kernel 1 (k_knn_partial): a CTA takes KNN_QT queries and one split of the
// training rows; chunks of KNN_DC dimensions of the queries and of KNN_TT training rows stream through a double-buffered cp.async
// ring, each thread accumulates a 4x4 register tile of squared distances in feature order, and once a training tile is complete its
// distances go to shared memory, where one warp per query inserts the ones that beat the query's k-th best into a sorted list.
// The lists of every split go to the workspace.  Kernel 2 (k_knn_vote): one warp per query merges the split lists and votes.
// Every list is ordered by (squared distance, training index), so the result does not depend on the split count.
namespace {

constexpr int KNN_QT = 64, KNN_TT = 64, KNN_DC = 16, KNN_THREADS = 256, KNN_KMAX = 64, KNN_MAX_SPLITS = 32;
constexpr int KNN_LD = KNN_DC + 1;           // padded row of a staged chunk: the 16 rows a warp reads per dimension hit distinct banks
constexpr int KNN_TARGET_CTAS = 2 * 132;

struct KnnPlan {
    int splits, rows_per_split;
};

// the training set is split so that a few thousand queries still fill the GPU; rows_per_split is a whole number of tiles
inline KnnPlan knn_plan(int N, int N_t)
{
    const long q_tiles = (N + KNN_QT - 1) / KNN_QT;
    const long t_tiles = (N_t + KNN_TT - 1) / KNN_TT;
    long s = (KNN_TARGET_CTAS + q_tiles - 1) / q_tiles;
    s = s < 1 ? 1 : (s > KNN_MAX_SPLITS ? KNN_MAX_SPLITS : s);
    if (s > t_tiles) s = t_tiles;
    const long tiles_per_split = (t_tiles + s - 1) / s;
    KnnPlan p;
    p.rows_per_split = (int)(tiles_per_split * KNN_TT);
    p.splits = (int)((t_tiles + tiles_per_split - 1) / tiles_per_split);
    return p;
}

inline size_t knn_smem_bytes(int k)
{
    return sizeof(double) * (2 * (KNN_QT + KNN_TT) * KNN_LD + KNN_QT * (KNN_TT + 1)) + (sizeof(double) + sizeof(int)) * KNN_QT * k;
}

__device__ __forceinline__ void cp_async8(void* smem, const void* gmem, bool valid)
{
    const unsigned dst = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(gmem), "r"(valid ? 8 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
__device__ __forceinline__ void cp_async_wait1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

// (d, i) < (e, j) in the neighbour order
__device__ __forceinline__ bool knn_less(double d, int i, double e, int j) { return d < e || (d == e && i < j); }

__global__ void __launch_bounds__(KNN_THREADS) k_knn_partial(const double* __restrict__ x, int N_in, const int* n_dev, int D,
                                                             const double* __restrict__ fit_x, int N_t, int k, int rows_per_split,
                                                             double* __restrict__ part_d, int* __restrict__ part_i)
{
    extern __shared__ __align__(16) unsigned char knn_smem[];
    double* stage = (double*)knn_smem;                                  // [2][KNN_QT + KNN_TT][KNN_LD]
    double* dist = stage + 2 * (KNN_QT + KNN_TT) * KNN_LD;              // [KNN_QT][KNN_TT + 1]
    double* list_d = dist + KNN_QT * (KNN_TT + 1);                      // [KNN_QT][k]
    int* list_i = (int*)(list_d + KNN_QT * k);                          // [KNN_QT][k]

    const int N = n_dev ? min(*n_dev, N_in) : N_in;
    const int q0 = blockIdx.x * KNN_QT;
    if (q0 >= N) return;
    const int t_lo = blockIdx.y * rows_per_split;
    const int t_hi = min(N_t, t_lo + rows_per_split);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int e = tid; e < KNN_QT * k; e += KNN_THREADS) {
        list_d[e] = CUDART_INF;
        list_i[e] = INT_MAX;
    }
    const int n_dc = (D + KNN_DC - 1) / KNN_DC;
    const int n_stages = (t_hi - t_lo + KNN_TT - 1) / KNN_TT * n_dc;

    // stage s: dimensions [c * KNN_DC, +KNN_DC) of the query tile and of training tile s / n_dc; rows past the end read as zeros
    auto load = [&](int s) {
        double* buf = stage + (s & 1) * (KNN_QT + KNN_TT) * KNN_LD;
        const int t0 = t_lo + s / n_dc * KNN_TT, d0 = s % n_dc * KNN_DC;
        for (int e = tid; e < (KNN_QT + KNN_TT) * KNN_DC; e += KNN_THREADS) {
            const int r = e / KNN_DC, dd = e % KNN_DC;
            const bool is_q = r < KNN_QT;
            const long row = is_q ? (long)q0 + r : (long)t0 + (r - KNN_QT);
            const bool ok = d0 + dd < D && row < (is_q ? N : t_hi);
            const double* src = is_q ? x : fit_x;
            cp_async8(buf + r * KNN_LD + dd, ok ? src + row * D + d0 + dd : src, ok);
        }
    };

    const int tq = tid >> 4, tt = tid & 15;           // queries tq + 16 i, training rows tt + 16 j
    double acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;

    if (n_stages > 0) load(0);
    cp_async_commit();
    for (int s = 0; s < n_stages; ++s) {
        if (s + 1 < n_stages) load(s + 1);
        cp_async_commit();
        cp_async_wait1();
        __syncthreads();
        const double* xs = stage + (s & 1) * (KNN_QT + KNN_TT) * KNN_LD;
        const double* ts = xs + KNN_QT * KNN_LD;
        const int c = s % n_dc, dlim = min(KNN_DC, D - c * KNN_DC);
        // sum_d (x_d - t_d)^2 in feature order, each step rounded on its own: the bits of a left-to-right float64 loop
#pragma unroll 4
        for (int d = 0; d < dlim; ++d) {
            double xv[4], tv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) xv[i] = xs[(tq + 16 * i) * KNN_LD + d];
#pragma unroll
            for (int j = 0; j < 4; ++j) tv[j] = ts[(tt + 16 * j) * KNN_LD + d];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const double df = __dsub_rn(xv[i], tv[j]);
                    acc[i][j] = __dadd_rn(acc[i][j], __dmul_rn(df, df));
                }
        }
        if (c == n_dc - 1) {
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    dist[(tq + 16 * i) * (KNN_TT + 1) + tt + 16 * j] = acc[i][j];
                    acc[i][j] = 0.0;
                }
            __syncthreads();
            const int t0 = t_lo + s / n_dc * KNN_TT;
            for (int q = warp; q < KNN_QT && q0 + q < N; q += KNN_THREADS / 32) {
                double* ld = list_d + q * k;
                int* li = list_i + q * k;
                double thr_d = ld[k - 1];
                int thr_i = li[k - 1];
                for (int j = 0; j < KNN_TT / 32; ++j) {
                    const int tcol = lane + 32 * j;
                    const int idx = t0 + tcol;
                    const double d = dist[q * (KNN_TT + 1) + tcol];
                    const bool live = idx < t_hi;
                    unsigned mask = __ballot_sync(0xffffffffu, live && knn_less(d, idx, thr_d, thr_i));
                    while (mask) {
                        const int src = __ffs(mask) - 1;
                        const double cd = __shfl_sync(0xffffffffu, d, src);
                        const int ci = __shfl_sync(0xffffffffu, idx, src);
                        // insert (cd, ci) at its rank among the k sorted entries; the last one drops out
                        const bool in0 = lane < k, in1 = lane + 32 < k;
                        const double e0 = in0 ? ld[lane] : 0.0, e1 = in1 ? ld[lane + 32] : 0.0;
                        const int f0 = in0 ? li[lane] : 0, f1 = in1 ? li[lane + 32] : 0;
                        const int pos = __popc(__ballot_sync(0xffffffffu, in0 && knn_less(e0, f0, cd, ci))) +
                                        __popc(__ballot_sync(0xffffffffu, in1 && knn_less(e1, f1, cd, ci)));
                        const double p0 = __shfl_up_sync(0xffffffffu, e0, 1), p1 = __shfl_up_sync(0xffffffffu, e1, 1);
                        const int g0 = __shfl_up_sync(0xffffffffu, f0, 1), g1 = __shfl_up_sync(0xffffffffu, f1, 1);
                        const double top0 = __shfl_sync(0xffffffffu, e0, 31);
                        const int topi0 = __shfl_sync(0xffffffffu, f0, 31);
                        __syncwarp();
                        if (in0 && lane >= pos) {
                            ld[lane] = lane == pos ? cd : p0;
                            li[lane] = lane == pos ? ci : g0;
                        }
                        if (in1 && lane + 32 >= pos) {
                            const bool at = lane + 32 == pos;
                            ld[lane + 32] = at ? cd : (lane == 0 ? top0 : p1);
                            li[lane + 32] = at ? ci : (lane == 0 ? topi0 : g1);
                        }
                        __syncwarp();
                        thr_d = ld[k - 1];
                        thr_i = li[k - 1];
                        mask &= ~(1u << src);
                        mask &= __ballot_sync(0xffffffffu, live && knn_less(d, idx, thr_d, thr_i));
                    }
                }
            }
        }
        __syncthreads();          // the buffer just read is the one stage s + 2 loads into; dist is rewritten by the next tile
    }
    for (int e = tid; e < KNN_QT * k; e += KNN_THREADS) {
        const int q = e / k;
        if (q0 + q >= N) break;
        const size_t o = ((size_t)blockIdx.y * N_in + q0 + q) * k + e % k;
        part_d[o] = list_d[e];
        part_i[o] = list_i[e];
    }
}

// one warp per query: merge the split lists (lane s holds the head of split s) into the k nearest, in ascending order, and add each
// neighbour's weight to its class -- lane c owns classes c and c + 32, so every class sums its weights in neighbour order, as
// KNeighborsClassifier.predict_proba does -- then divide by the row sum.  distance weights: 1 / sqrt(d^2), or, when the nearest
// neighbour is at distance 0, the indicator d == 0 (_get_weights).
__global__ void k_knn_vote(const double* __restrict__ part_d, const int* __restrict__ part_i, int N_in, const int* n_dev, int splits, int k,
                           const int* __restrict__ y, int N_t, int K, int distance_weights, double* __restrict__ proba)
{
    const int N = n_dev ? min(*n_dev, N_in) : N_in;
    const int lane = threadIdx.x & 31;
    const int warps = gridDim.x * (blockDim.x >> 5);
    for (int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); n < N; n += warps) {
        const size_t base = ((size_t)lane * N_in + n) * k;
        int head = 0;
        double hd = CUDART_INF;
        int hi = INT_MAX;
        if (lane < splits) {
            hd = part_d[base];
            hi = part_i[base];
        }
        double acc0 = 0.0, acc1 = 0.0;
        bool zero_row = false;
        for (int r = 0; r < k; ++r) {
            double bd = hd;
            int bi = hi, bl = lane;
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                const double od = __shfl_xor_sync(0xffffffffu, bd, off);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, off), ol = __shfl_xor_sync(0xffffffffu, bl, off);
                if (knn_less(od, oi, bd, bi) || (od == bd && oi == bi && ol < bl)) {
                    bd = od;
                    bi = oi;
                    bl = ol;
                }
            }
            if (lane == bl) {
                ++head;
                hd = head < k ? part_d[base + head] : CUDART_INF;
                hi = head < k ? part_i[base + head] : INT_MAX;
            }
            if (bi < 0 || bi >= N_t) continue;          // fewer than k finite distances: nothing to add
            double w = 1.0;
            if (distance_weights) {
                if (r == 0) zero_row = bd == 0.0;
                w = zero_row ? (bd == 0.0 ? 1.0 : 0.0) : 1.0 / sqrt(bd);
            }
            const int c = y[bi];
            if (c == lane) acc0 = acc0 + w;
            if (c == lane + 32) acc1 = acc1 + w;
        }
        double sum = 0.0;
        for (int c = 0; c < K; ++c) sum = sum + __shfl_sync(0xffffffffu, c < 32 ? acc0 : acc1, c & 31);
        if (sum == 0.0) sum = 1.0;
        double* out = proba + (size_t)n * K;
        if (lane < K) out[lane] = acc0 / sum;
        if (lane + 32 < K) out[lane + 32] = acc1 / sum;
    }
}

// logistic regression: one thread per row.  decision_c = x . coef_c + intercept_c; one coefficient row (binary) gives
// [1 - expit(d), expit(d)] (_predict_proba_lr), more give the softmax in sklearn.utils.extmath.softmax's order: subtract the row
// maximum, exp, divide by the row sum.
__global__ void k_linear_proba(const double* __restrict__ x, int N_in, const int* n_dev, int D, const double* __restrict__ coef,
                               const double* __restrict__ intercept, int n_coef, double* __restrict__ proba)
{
    const int N = n_dev ? min(*n_dev, N_in) : N_in;
    const int K = n_coef == 1 ? 2 : n_coef;
    for (size_t n = blockIdx.x * (size_t)blockDim.x + threadIdx.x; n < (size_t)N; n += (size_t)gridDim.x * blockDim.x) {
        const double* xr = x + n * D;
        double* out = proba + n * K;
        double mx = -CUDART_INF;
        for (int c = 0; c < n_coef; ++c) {
            const double* w = coef + (size_t)c * D;
            double acc = 0.0;
            for (int d = 0; d < D; ++d) acc = fma(xr[d], w[d], acc);
            acc = acc + intercept[c];
            mx = fmax(mx, acc);
            out[n_coef == 1 ? 1 : c] = acc;
        }
        if (n_coef == 1) {
            const double e = 1.0 / (1.0 + exp(-out[1]));
            out[0] = 1.0 - e;
            out[1] = e;
            continue;
        }
        double sum = 0.0;
        for (int c = 0; c < K; ++c) {
            const double e = exp(out[c] - mx);
            out[c] = e;
            sum = sum + e;
        }
        for (int c = 0; c < K; ++c) out[c] = out[c] / sum;
    }
}

} // namespace

extern "C" size_t isb_knn_predict_workspace_bytes(int N, int N_t, int k)
{
    if (N <= 0 || N_t <= 0 || k <= 0) return 0;
    const KnnPlan p = knn_plan(N, N_t);
    const size_t entries = (size_t)p.splits * N * k;
    return isb_align(sizeof(double) * entries) + isb_align(sizeof(int32_t) * entries);
}

extern "C" int isb_knn_predict_proba(const double* x, int N, const int32_t* n_dev, int D, const double* fit_x, int N_t, const int32_t* y,
                                     int k, int K, int weights, double* proba, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(x && fit_x && y && proba && ws, "null pointer");
    ISB_REQUIRE(N > 0 && D > 0 && N_t > 0 && K > 0, "bad sizes");
    ISB_REQUIRE(k >= 1 && k <= KNN_KMAX, "k must be in [1, 64]");
    ISB_REQUIRE(k <= N_t, "k must not exceed the training rows");
    ISB_REQUIRE(K <= FOREST_KMAX, "K <= 64 classes");
    ISB_REQUIRE(weights == 0 || weights == 1, "weights: 0 uniform, 1 distance");
    ISB_REQUIRE(ws_bytes >= isb_knn_predict_workspace_bytes(N, N_t, k), "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_GMM, st);
    const KnnPlan p = knn_plan(N, N_t);
    const size_t entries = (size_t)p.splits * N * k;
    double* part_d = (double*)ws;
    int* part_i = (int*)((char*)ws + isb_align(sizeof(double) * entries));
    const size_t smem = knn_smem_bytes(k);
    ISB_CUDA_CHECK(cudaFuncSetAttribute(k_knn_partial, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const dim3 grid((N + KNN_QT - 1) / KNN_QT, p.splits);
    k_knn_partial<<<grid, KNN_THREADS, smem, st>>>(x, N, n_dev, D, fit_x, N_t, k, p.rows_per_split, part_d, part_i);
    ISB_LAUNCH_CHECK();
    k_knn_vote<<<grid_for((size_t)N * 32, 256), 256, 0, st>>>(part_d, part_i, N, n_dev, p.splits, k, y, N_t, K, weights, proba);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" size_t isb_linear_predict_workspace_bytes(int N, int n_coef)
{
    (void)N;
    (void)n_coef;
    return 0;
}

extern "C" int isb_linear_predict_proba(const double* x, int N, const int32_t* n_dev, int D, const double* coef, const double* intercept,
                                        int n_coef, double* proba, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    (void)ws;
    ISB_REQUIRE(x && coef && intercept && proba, "null pointer");
    ISB_REQUIRE(N > 0 && D > 0 && n_coef > 0, "bad sizes");
    ISB_REQUIRE(n_coef <= FOREST_KMAX, "K <= 64 classes");
    ISB_REQUIRE(ws_bytes >= isb_linear_predict_workspace_bytes(N, n_coef), "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_GMM, st);
    k_linear_proba<<<grid_for((size_t)N, 128), 128, 0, st>>>(x, N, n_dev, D, coef, intercept, n_coef, proba);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
