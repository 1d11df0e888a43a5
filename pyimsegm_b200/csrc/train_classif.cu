// train_classif.cu -- the per-image data step of the supervised training (imsegm/pipelines.py:272-290, :293-379):
//   isb_superpixel_train_labels : one training label per superpixel from an annotation (labeling.py:245-278 + the argmax / purity)
//   isb_unique_rows_rounded     : balance_dataset_by_(features, labels, 'unique') of one image (classification.py:1159-1216)
#include <cub/device/device_merge_sort.cuh>
#include "common.cuh"
#include "compact.cuh"

namespace {

// ---- training labels ------------------------------------------------------------------------------------------------------
// Every (superpixel, label) pair with its pixel count goes into an open-addressing table of keys sp << 32 | code, code = the label
// for a known pixel and TL_UNKNOWN for a negative one.  The table holds at most H * W distinct keys, so its size follows the image
// and never the label range.  Pixels are read as row strips of TL_STRIP per thread; the runs a warp flushes together with the same
// key are summed first, so a region of one label costs one insert per warp and strip step.

constexpr unsigned long long TL_EMPTY = ~0ull;
constexpr unsigned TL_UNKNOWN = 0x80000000u;
constexpr int TL_STRIP = 32, TL_THREADS = 256;

inline size_t tl_capacity(int H, int W)
{
    const size_t n = (size_t)H * W;
    return n + n / 2 + 64;      // load factor <= 2/3
}

__device__ __forceinline__ unsigned long long tl_hash(unsigned long long k)
{
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return k;
}

__device__ __forceinline__ void tl_insert(unsigned long long* keys, unsigned* cnt, size_t cap, unsigned long long key, unsigned c)
{
    size_t i = (size_t)__umul64hi(tl_hash(key), (unsigned long long)cap);
    while (true) {
        unsigned long long prev = __ldcg(keys + i);       // a key once written never changes: a stale TL_EMPTY only costs the CAS
        if (prev == TL_EMPTY) prev = atomicCAS(keys + i, TL_EMPTY, key);
        if (prev == TL_EMPTY || prev == key) {
            atomicAdd(cnt + i, c);
            return;
        }
        if (++i == cap) i = 0;
    }
}

// every lane must call this; the flushing lanes' runs of equal keys go in as one insert
__device__ __forceinline__ void tl_flush(bool flush, unsigned long long key, unsigned c, unsigned long long* keys, unsigned* cnt, size_t cap)
{
    const unsigned fl = __ballot_sync(0xffffffffu, flush);
    if (flush) {
        const unsigned peers = __match_any_sync(fl, key);
        const unsigned s = __reduce_add_sync(peers, c);
        if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) tl_insert(keys, cnt, cap, key, s);
    }
}

__device__ __forceinline__ unsigned long long tl_key(const int* __restrict__ slic, const int* __restrict__ annot, size_t p, int nb)
{
    const int s = slic[p];
    if ((unsigned)s >= (unsigned)nb) return TL_EMPTY;               // outside the table: not counted
    const int a = annot[p];
    return ((unsigned long long)s << 32) | (a < 0 ? TL_UNKNOWN : (unsigned)a);
}

__global__ void __launch_bounds__(TL_THREADS) k_train_label_runs(const int* __restrict__ slic, const int* __restrict__ annot, int H, int W,
                                                                 int nb, unsigned long long* __restrict__ keys, unsigned* __restrict__ cnt,
                                                                 size_t cap)
{
    const int strips = (W + TL_STRIP - 1) / TL_STRIP;
    const long long t = (long long)blockIdx.x * TL_THREADS + threadIdx.x;
    const bool row_ok = t < (long long)H * strips;                 // whole warps stay in the loop for the shuffles
    const int y = row_ok ? (int)(t / strips) : 0;
    const int x0 = row_ok ? (int)(t % strips) * TL_STRIP : W;
    const size_t row = (size_t)y * W;
    unsigned long long run = TL_EMPTY;
    unsigned n = 0;
    for (int k = 0; k < TL_STRIP; ++k) {
        const int x = x0 + k;
        const unsigned long long key = x < W ? tl_key(slic, annot, row + x, nb) : TL_EMPTY;
        tl_flush(key != run && n > 0 && run != TL_EMPTY, run, n, keys, cnt, cap);
        if (key != run) {
            run = key;
            n = 0;
        }
        ++n;
    }
    tl_flush(n > 0 && run != TL_EMPTY, run, n, keys, cnt, cap);
}

// every table entry: its pixels to the superpixel's size, the unknown count, or the (count, smallest label) maximum as count << 32 |
// (2^31 - 1 - label), so that atomicMax keeps np.argmax's first maximum
__global__ void __launch_bounds__(256) k_train_label_best(const unsigned long long* __restrict__ keys, const unsigned* __restrict__ cnt,
                                                          size_t cap, unsigned* __restrict__ npx, unsigned* __restrict__ unk,
                                                          unsigned long long* __restrict__ best)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) {
        const unsigned long long key = keys[i];
        if (key == TL_EMPTY) continue;
        const unsigned c = cnt[i];
        const unsigned s = (unsigned)(key >> 32), code = (unsigned)key;
        atomicAdd(npx + s, c);
        if (code == TL_UNKNOWN) unk[s] = c;                           // one entry per superpixel
        else atomicMax(best + s, ((unsigned long long)c << 32) | (0x7fffffffu - code));
    }
}

// the closed form of argmax + purity (pipelines.py:283-290): the smallest label l* of the largest known count c* wins when c* >= u (the
// unknown bin ranks after every label) and c* / n is not below label_purity; -1 otherwise
__global__ void __launch_bounds__(256) k_train_label_pick(const unsigned* __restrict__ npx, const unsigned* __restrict__ unk,
                                                          const unsigned long long* __restrict__ best, int nb, const int* __restrict__ n_dev,
                                                          double purity, long long* __restrict__ labels)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nb) return;
    const int n_real = n_dev ? *n_dev : nb;
    const unsigned n = npx[s], u = unk[s];
    const unsigned c = (unsigned)(best[s] >> 32);
    long long lab = -1;
    if (s < n_real && c > 0 && c >= u && !((double)c / (double)n < purity)) lab = (long long)(0x7fffffffu - (unsigned)best[s]);
    labels[s] = lab;
}

// ---- unique rounded rows per class ----------------------------------------------------------------------------------------
constexpr long long UR_DROP = 0x7fffffffffffffffll;

// rounded = rint(x * 1000) / 1000 (np.round(x, 3)), -0 made +0 so that equal rows compare equal in the sort; key = the row's label, or
// UR_DROP for a row labelled -1 or past the real row count; any NaN of a kept row raises the flag
__global__ void __launch_bounds__(256) k_unique_round(const double* __restrict__ feat, int N, int D, int ld, const int* __restrict__ n_dev,
                                                      const long long* __restrict__ labels, double* __restrict__ rounded,
                                                      long long* __restrict__ key, int* __restrict__ order, int* __restrict__ nan_flag)
{
    const int n_real = n_dev ? min(*n_dev, N) : N;
    const size_t total = (size_t)N * D;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / D), d = (int)(i % D);
        const bool keep = r < n_real && labels[r] != -1;
        if (d == 0) {
            key[r] = keep ? labels[r] : UR_DROP;
            order[r] = r;
        }
        if (!keep) continue;
        const double x = feat[(size_t)r * ld + d];
        if (isnan(x)) atomicOr(nan_flag, 1);
        const double v = rint(x * 1000.0) / 1000.0;
        rounded[(size_t)r * D + d] = v == 0.0 ? 0.0 : v;
    }
}

struct RowLess {
    const double* rows;
    const long long* key;
    int D;
    __device__ bool operator()(int a, int b) const
    {
        const long long ka = key[a], kb = key[b];
        if (ka != kb) return ka < kb;
        if (ka == UR_DROP) return false;
        const double* ra = rows + (size_t)a * D;
        const double* rb = rows + (size_t)b * D;
        for (int d = 0; d < D; ++d)
            if (ra[d] != rb[d]) return ra[d] < rb[d];
        return false;
    }
};

// 1 where the sorted row is kept and differs from the one before it (its class or a column)
__global__ void __launch_bounds__(256) k_unique_flag(const int* __restrict__ order, int N, const long long* __restrict__ key,
                                                     const double* __restrict__ rows, int D, unsigned char* __restrict__ flag)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int a = order[i];
    bool f = key[a] != UR_DROP;
    if (f && i > 0) {
        const int b = order[i - 1];
        f = key[b] != key[a];
        for (int d = 0; d < D && !f; ++d) f = rows[(size_t)a * D + d] != rows[(size_t)b * D + d];
    }
    flag[i] = f;
}

__global__ void __launch_bounds__(CPT_THREADS) k_unique_write(const unsigned char* __restrict__ flag, const int* __restrict__ order, long long n,
                                                              const long long* __restrict__ tile_off, const long long* __restrict__ key,
                                                              int* __restrict__ out_row, long long* __restrict__ labels_out)
{
    const long long beg = (long long)blockIdx.x * CPT_TILE + (long long)threadIdx.x * CPT_PER;
    int total;
    long long o = tile_off[blockIdx.x] + cta_exclusive_sum<CPT_THREADS>(thread_count(flag, beg, n), total);
    for (int k = 0; k < CPT_PER; ++k) {
        const long long i = beg + k;
        if (i < n && flag[i]) {
            const int a = order[i];
            out_row[o] = a;
            labels_out[o] = key[a];
            ++o;
        }
    }
}

// rows_out [n_out, D] from the rounded rows; a NaN seen by k_unique_round turns the count into -1
__global__ void __launch_bounds__(256) k_unique_gather(const double* __restrict__ rows, int N, int D, const int* __restrict__ out_row,
                                                       const long long* __restrict__ n_out, double* __restrict__ rows_out)
{
    const long long n = *n_out;
    const size_t total = (size_t)N * D;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / D), d = (int)(i % D);
        if (r >= n) break;
        rows_out[i] = rows[(size_t)out_row[r] * D + d];
    }
}

__global__ void k_unique_status(const int* __restrict__ nan_flag, long long* __restrict__ n_out)
{
    if (*nan_flag) *n_out = -1;
}

inline unsigned grid_of(size_t n, int threads)
{
    const size_t g = (n + threads - 1) / threads;
    return (unsigned)(g < 1 ? 1 : g > 65536 ? 65536 : g);
}

size_t unique_sort_bytes(int N, int D)
{
    size_t b = 0;
    cub::DeviceMergeSort::SortKeys(nullptr, b, (int*)nullptr, N, RowLess{nullptr, nullptr, D});
    return b;
}

} // namespace

extern "C" size_t isb_train_labels_workspace_bytes(int H, int W, int nb)
{
    if (H <= 0 || W <= 0 || nb <= 0) return 0;
    const size_t cap = tl_capacity(H, W);
    return isb_align(8 * cap) + isb_align(4 * cap) + isb_align(8 * (size_t)nb) + 2 * isb_align(4 * (size_t)nb);
}

extern "C" int isb_superpixel_train_labels(const int32_t* slic, int H, int W, int nb, const int32_t* n_labels_dev, const int32_t* annot,
                                           double label_purity, int64_t* labels, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(slic && annot && labels && ws, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && nb > 0, "bad sizes");
    ISB_REQUIRE((long long)H * W <= (1ll << 31), "more than 2^31 pixels");
    ISB_REQUIRE(ws_bytes >= isb_train_labels_workspace_bytes(H, W, nb), "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t cap = tl_capacity(H, W);
    WsCarver c(ws, ws_bytes);
    unsigned long long* keys = c.take<unsigned long long>(cap);
    unsigned* cnt = c.take<unsigned>(cap);
    unsigned long long* best = c.take<unsigned long long>(nb);
    unsigned* npx = c.take<unsigned>(nb);
    unsigned* unk = c.take<unsigned>(nb);
    ISB_CUDA_CHECK(cudaMemsetAsync(keys, 0xff, 8 * cap, st));
    ISB_CUDA_CHECK(cudaMemsetAsync(cnt, 0, 4 * cap, st));
    ISB_CUDA_CHECK(cudaMemsetAsync(best, 0, 8 * (size_t)nb, st));
    ISB_CUDA_CHECK(cudaMemsetAsync(npx, 0, 4 * (size_t)nb, st));
    ISB_CUDA_CHECK(cudaMemsetAsync(unk, 0, 4 * (size_t)nb, st));
    const long long threads = (long long)H * ((W + TL_STRIP - 1) / TL_STRIP);
    k_train_label_runs<<<(unsigned)((threads + TL_THREADS - 1) / TL_THREADS), TL_THREADS, 0, st>>>(slic, annot, H, W, nb, keys, cnt, cap);
    ISB_LAUNCH_CHECK();
    k_train_label_best<<<grid_of(cap, 256), 256, 0, st>>>(keys, cnt, cap, npx, unk, best);
    ISB_LAUNCH_CHECK();
    k_train_label_pick<<<(nb + 255) / 256, 256, 0, st>>>(npx, unk, best, nb, n_labels_dev, label_purity, (long long*)labels);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" size_t isb_unique_rows_workspace_bytes(int N, int D)
{
    if (N <= 0 || D <= 0) return 0;
    return isb_align(8 * (size_t)N * D) + isb_align(8 * (size_t)N) + 2 * isb_align(4 * (size_t)N) + isb_align((size_t)N) + isb_align(4)
         + compact_workspace_bytes(N) + isb_align(unique_sort_bytes(N, D));
}

extern "C" int isb_unique_rows_rounded(const double* feat, int N, int D, int ld, const int32_t* n_dev, const int64_t* labels, double* rows_out,
                                       int64_t* labels_out, long long* n_out, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(feat && labels && rows_out && labels_out && n_out && ws, "null pointer");
    ISB_REQUIRE(N > 0 && D > 0 && ld >= D, "bad sizes");
    ISB_REQUIRE(ws_bytes >= isb_unique_rows_workspace_bytes(N, D), "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    WsCarver c(ws, ws_bytes);
    double* rounded = c.take<double>((size_t)N * D);
    long long* key = c.take<long long>(N);
    int* order = c.take<int>(N);
    int* out_row = c.take<int>(N);
    unsigned char* flag = c.take<unsigned char>(N);
    int* nan_flag = c.take<int>(1);
    void* cws = c.take<unsigned char>(compact_workspace_bytes(N));
    size_t sort_bytes = unique_sort_bytes(N, D);
    void* sort_ws = c.take<unsigned char>(sort_bytes);
    ISB_CUDA_CHECK(cudaMemsetAsync(nan_flag, 0, sizeof(int), st));
    k_unique_round<<<grid_of((size_t)N * D, 256), 256, 0, st>>>(feat, N, D, ld, n_dev, (const long long*)labels, rounded, key, order, nan_flag);
    ISB_LAUNCH_CHECK();
    ISB_CUDA_CHECK(cub::DeviceMergeSort::SortKeys(sort_ws, sort_bytes, order, N, RowLess{rounded, key, D}, st));
    ++g_isb_launches;
    k_unique_flag<<<(N + 255) / 256, 256, 0, st>>>(order, N, key, rounded, D, flag);
    ISB_LAUNCH_CHECK();
    const int rc = compact_count(flag, (long long)N, cws, st, n_out);
    if (rc != ISB_OK) return rc;
    k_unique_write<<<compact_tiles(N), CPT_THREADS, 0, st>>>(flag, order, N, compact_tile_offsets(cws, N), key, out_row,
                                                            (long long*)labels_out);
    ISB_LAUNCH_CHECK();
    k_unique_gather<<<grid_of((size_t)N * D, 256), 256, 0, st>>>(rounded, N, D, out_row, n_out, rows_out);
    ISB_LAUNCH_CHECK();
    k_unique_status<<<1, 1, 0, st>>>(nan_flag, n_out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
