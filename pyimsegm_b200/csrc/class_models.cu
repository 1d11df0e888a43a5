// class_models.cu -- predict_proba of a caller-fitted class model on the device (the shared-model entry point of the reference,
// imsegm/pipelines.py:160-241, with a model from estim_model_classes_group or a trained classifier): the feature transform of the
// model's Pipeline (NaN -> 0, StandardScaler, PCA) and the decision-tree / random-forest evaluation.  The tables are compiled on the
// host by pyimsegm_b200/class_models.py.  The mixture evaluation lives in gmm.cu, next to the FP64 GEMM it shares with the fit.
// Nothing here synchronises with the host or allocates, so the calls can be captured in a CUDA graph.
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
