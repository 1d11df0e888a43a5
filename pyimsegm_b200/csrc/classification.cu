// classification.cu -- the contingency table behind the scoring functions of the reference's imsegm/classification.py
// (compute_classif_metrics :305-371, compute_classif_stat_segm_annot :374-421, compute_tp_tn_fp_fn :1265-1310): the number of
// pixels of every (annotation value, segmentation value) pair, pixels with a value of the drop list in either map left out
// (:404-410).  Three passes over the two maps:
//   1. the least and largest kept value of each map (skipped for dtypes of 16 bits or fewer, whose range the dtype bounds);
//   2. a presence table over [min, max] of each map, compacted (compact.cuh) into the ascending distinct values and, in place, the
//      value -> dense index table;
//   3. the counts of every (dense true, dense pred) cell: per-CTA shared-memory bins for tables of at most SMEM_CELLS cells, global
//      atomics above.  Every lane keeps a run of one cell (run_flush.cuh).
#include <algorithm>

#include "compact.cuh"
#include "run_flush.cuh"

namespace {

constexpr int CT_THREADS = 256;
constexpr int CT_PER = 16;                       // pixels per lane and chunk, 32 apart (consecutive lanes on consecutive pixels)
constexpr long long CT_CHUNK = 32LL * CT_PER;    // pixels of one warp chunk
constexpr long long RANGE_MAX = 1LL << 26;       // widest [min, max] of one map
constexpr long long CELLS_MAX = 1LL << 28;       // largest table
// u32 bins of the shared-memory table: 64 KB, so three 256-thread CTAs share an SM's 228 KB
constexpr int SMEM_CELLS = 16384;
constexpr unsigned NO_CELL = 0xffffffffu;        // a dropped pixel or one past the end (cells are < 2^28)

__device__ __forceinline__ long long load_label(const void* __restrict__ p, int dtype, long long i)
{
    switch (dtype) {
        case ISB_U8:
        case ISB_BOOL: return ((const uint8_t*)p)[i];
        case ISB_I8: return ((const int8_t*)p)[i];
        case ISB_U16: return ((const uint16_t*)p)[i];
        case ISB_I16: return ((const int16_t*)p)[i];
        case ISB_I32: return ((const int32_t*)p)[i];
        case ISB_U32: return ((const uint32_t*)p)[i];
        default: return ((const int64_t*)p)[i];
    }
}

// v is one of the sorted drop values
__device__ __forceinline__ bool in_drop(long long v, const int64_t* __restrict__ drop, int n_drop)
{
    int lo = 0, hi = n_drop;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(drop + mid) < v) lo = mid + 1; else hi = mid;
    }
    return lo < n_drop && __ldg(drop + lo) == v;
}

struct Pair {
    long long a, b;
    bool kept;
};

// the values of both maps at pixel i (i < n), kept unless one of them is dropped
__device__ __forceinline__ Pair load_pair(const void* yt, int dt, const void* yp, int dp, long long i, const int64_t* drop, int n_drop)
{
    Pair q;
    q.a = load_label(yt, dt, i);
    q.b = load_label(yp, dp, i);
    q.kept = n_drop == 0 || !(in_drop(q.a, drop, n_drop) || in_drop(q.b, drop, n_drop));
    return q;
}

__device__ __forceinline__ long long warp_min(long long v)
{
    for (int o = 16; o; o >>= 1) v = min(v, (long long)__shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ long long warp_max(long long v)
{
    for (int o = 16; o; o >>= 1) v = max(v, (long long)__shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__global__ void k_ct_range_init(long long* mm)
{
    mm[0] = mm[2] = LLONG_MAX;
    mm[1] = mm[3] = LLONG_MIN;
}

// pass 1: mm = (min true, max true, min pred, max pred) over the kept pixels; grid-stride over warp chunks
__global__ void __launch_bounds__(CT_THREADS) k_ct_range(const void* __restrict__ yt, int dt, const void* __restrict__ yp, int dp, long long n,
                                                       const int64_t* __restrict__ drop, int n_drop, long long* __restrict__ mm)
{
    const long long warps = (long long)gridDim.x * (CT_THREADS / 32);
    long long lo_a = LLONG_MAX, hi_a = LLONG_MIN, lo_b = LLONG_MAX, hi_b = LLONG_MIN;
    for (long long w = ((long long)blockIdx.x * CT_THREADS + threadIdx.x) >> 5; w * CT_CHUNK < n; w += warps) {
        const long long base = w * CT_CHUNK + (threadIdx.x & 31);
#pragma unroll 4
        for (int k = 0; k < CT_PER; ++k) {
            const long long i = base + 32LL * k;
            if (i >= n) break;
            const Pair q = load_pair(yt, dt, yp, dp, i, drop, n_drop);
            if (q.kept) {
                lo_a = min(lo_a, q.a); hi_a = max(hi_a, q.a);
                lo_b = min(lo_b, q.b); hi_b = max(hi_b, q.b);
            }
        }
    }
    lo_a = warp_min(lo_a); hi_a = warp_max(hi_a);
    lo_b = warp_min(lo_b); hi_b = warp_max(hi_b);
    if ((threadIdx.x & 31) == 0 && lo_a <= hi_a) {
        atomicMin(mm + 0, lo_a); atomicMax(mm + 1, hi_a);
        atomicMin(mm + 2, lo_b); atomicMax(mm + 3, hi_b);
    }
}

// pass 2: pres_x[v - min_x] = 1 for every kept value; a lane writes only when its value changes
__global__ void __launch_bounds__(CT_THREADS) k_ct_mark(const void* __restrict__ yt, int dt, const void* __restrict__ yp, int dp, long long n,
                                                      const int64_t* __restrict__ drop, int n_drop, long long min_a, long long min_b,
                                                      int32_t* __restrict__ pres_a, int32_t* __restrict__ pres_b)
{
    const long long warps = (long long)gridDim.x * (CT_THREADS / 32);
    long long last_a = LLONG_MIN, last_b = LLONG_MIN;     // LLONG_MIN: nothing written yet (min_x >= LLONG_MIN, so v - min_x >= 0)
    bool any = false;
    for (long long w = ((long long)blockIdx.x * CT_THREADS + threadIdx.x) >> 5; w * CT_CHUNK < n; w += warps) {
        const long long base = w * CT_CHUNK + (threadIdx.x & 31);
        for (int k = 0; k < CT_PER; ++k) {
            const long long i = base + 32LL * k;
            if (i >= n) break;
            const Pair q = load_pair(yt, dt, yp, dp, i, drop, n_drop);
            if (!q.kept) continue;
            if (!any || q.a != last_a) pres_a[q.a - min_a] = 1;
            if (!any || q.b != last_b) pres_b[q.b - min_b] = 1;
            last_a = q.a; last_b = q.b; any = true;
        }
    }
}

// the compaction of a presence table: values[o] = min + i and, in place, pres[i] = o (the dense index) for its o-th present entry
__global__ void __launch_bounds__(CPT_THREADS) k_ct_dense(int32_t* __restrict__ pres, long long range, long long min_v,
                                                        const long long* __restrict__ tile_off, int64_t* __restrict__ values)
{
    const long long beg = (long long)blockIdx.x * CPT_TILE + (long long)threadIdx.x * CPT_PER;
    int total;
    long long o = tile_off[blockIdx.x] + cta_exclusive_sum<CPT_THREADS>(thread_count(pres, beg, range), total);
    for (int k = 0; k < CPT_PER; ++k) {
        const long long i = beg + k;
        if (i < range && pres[i]) {
            values[o] = min_v + i;
            pres[i] = (int32_t)o;
            ++o;
        }
    }
}

// pass 3: counts[dense(a) * k_b + dense(b)] += 1 over the kept pixels.  SMEM: the CTA counts into u32 bins in shared memory and adds
// every nonzero bin to the table once at the end; otherwise every flush is a global atomic.
template <bool SMEM>
__global__ void __launch_bounds__(CT_THREADS) k_ct_count(const void* __restrict__ yt, int dt, const void* __restrict__ yp, int dp, long long n,
                                                       const int64_t* __restrict__ drop, int n_drop, long long min_a, long long min_b,
                                                       const int32_t* __restrict__ dense_a, const int32_t* __restrict__ dense_b, int k_b,
                                                       int cells, unsigned long long* __restrict__ counts)
{
    extern __shared__ unsigned bins[];
    if constexpr (SMEM) {
        for (int c = threadIdx.x; c < cells; c += CT_THREADS) bins[c] = 0;
        __syncthreads();
    }
    const auto add = [counts](unsigned cell, unsigned s) {
        if constexpr (SMEM) atomicAdd(bins + cell, s);
        else atomicAdd(counts + cell, (unsigned long long)s);
    };
    const long long warps = (long long)gridDim.x * (CT_THREADS / 32);
    unsigned cur = NO_CELL, cnt = 0;
    long long last_a = 0, last_b = 0;
    unsigned last_cell = NO_CELL;
    for (long long w = ((long long)blockIdx.x * CT_THREADS + threadIdx.x) >> 5; w * CT_CHUNK < n; w += warps) {
        const long long base = w * CT_CHUNK + (threadIdx.x & 31);
        for (int k = 0; k < CT_PER; ++k) {
            const long long i = base + 32LL * k;
            unsigned cell = NO_CELL;
            if (i < n) {
                const Pair q = load_pair(yt, dt, yp, dp, i, drop, n_drop);
                if (q.kept) {
                    if (last_cell == NO_CELL || q.a != last_a || q.b != last_b) {
                        last_cell = (unsigned)__ldg(dense_a + (q.a - min_a)) * (unsigned)k_b + (unsigned)__ldg(dense_b + (q.b - min_b));
                        last_a = q.a; last_b = q.b;
                    }
                    cell = last_cell;
                }
            }
            flush_run(cell != cur && cnt != 0, cur, cnt, add);
            if (cell != cur) { cur = cell; cnt = 0; }
            if (cell != NO_CELL) ++cnt;
        }
    }
    flush_run(cnt != 0, cur, cnt, add);
    if constexpr (SMEM) {
        __syncthreads();
        for (int c = threadIdx.x; c < cells; c += CT_THREADS)
            if (bins[c]) atomicAdd(counts + c, (unsigned long long)bins[c]);
    }
}

bool label_dtype(int d) { return d == ISB_U8 || d == ISB_U16 || (d >= ISB_I8 && d <= ISB_BOOL); }

// [lo, hi] of a dtype of 16 bits or fewer (no range pass); false for the wider ones
bool narrow_bounds(int d, long long* lo, long long* hi)
{
    switch (d) {
        case ISB_BOOL: *lo = 0; *hi = 1; return true;
        case ISB_U8: *lo = 0; *hi = 255; return true;
        case ISB_I8: *lo = -128; *hi = 127; return true;
        case ISB_U16: *lo = 0; *hi = 65535; return true;
        case ISB_I16: *lo = -32768; *hi = 32767; return true;
        default: return false;
    }
}

long long range_cap(int d)
{
    long long lo, hi;
    return narrow_bounds(d, &lo, &hi) ? hi - lo + 1 : RANGE_MAX;
}

unsigned pass_grid(long long n, int ctas_per_sm)
{
    // persistent CTAs; enough of them that one CTA's u32 bins stay below 2^31 pixels
    const long long chunks_per_cta = (long long)(CT_THREADS / 32);
    const long long need = (n + CT_CHUNK * chunks_per_cta - 1) / (CT_CHUNK * chunks_per_cta);
    return (unsigned)std::max<long long>(1, std::min<long long>(need, std::max<long long>(132LL * ctas_per_sm, n >> 30)));
}

struct CtWs {
    long long* mm;     // [4]
    long long* k;      // [2] device counts of the compactions
    int32_t* pres_a;   // [range_cap(dt)]
    int32_t* pres_b;   // [range_cap(dp)]
    void* cws_a;       // compaction workspaces
    void* cws_b;
    size_t need;
};

CtWs carve(void* ws, int dt, int dp)
{
    const long long ca = range_cap(dt), cb = range_cap(dp);
    WsCarver c(ws, 0);
    CtWs w;
    w.mm = c.take<long long>(4);
    w.k = c.take<long long>(2);
    w.pres_a = c.take<int32_t>(ca);
    w.pres_b = c.take<int32_t>(cb);
    w.cws_a = c.take<char>(compact_workspace_bytes(ca));
    w.cws_b = c.take<char>(compact_workspace_bytes(cb));
    w.need = c.off;
    return w;
}

int check_args(const void* yt, int dt, const void* yp, int dp, long long n, const int64_t* drop, int n_drop)
{
    ISB_REQUIRE(yt && yp, "null pointer");
    ISB_REQUIRE(n > 0, "bad sizes");
    ISB_REQUIRE(n_drop >= 0 && (n_drop == 0 || drop), "bad drop list");
    ISB_REQUIRE(label_dtype(dt) && label_dtype(dp), "label maps are bool, u8, i8, u16, i16, i32, u32 or i64");
    return ISB_OK;
}

} // namespace

extern "C" size_t isb_contingency_workspace_bytes(int dtype_true, int dtype_pred)
{
    if (!label_dtype(dtype_true) || !label_dtype(dtype_pred)) return 0;
    return carve(nullptr, dtype_true, dtype_pred).need;
}

extern "C" int isb_contingency_count(const void* y_true, int dtype_true, const void* y_pred, int dtype_pred, long long n, const int64_t* drop,
                                     int n_drop, void* ws, size_t ws_bytes, long long* info, isb_stream_t stream)
{
    if (int s = check_args(y_true, dtype_true, y_pred, dtype_pred, n, drop, n_drop)) return s;
    ISB_REQUIRE(ws && info, "null pointer");
    ISB_REQUIRE(ws_bytes >= isb_contingency_workspace_bytes(dtype_true, dtype_pred), "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const CtWs w = carve(ws, dtype_true, dtype_pred);
    long long mm[4];
    const bool narrow_a = narrow_bounds(dtype_true, mm + 0, mm + 1), narrow_b = narrow_bounds(dtype_pred, mm + 2, mm + 3);
    if (!(narrow_a && narrow_b)) {
        k_ct_range_init<<<1, 1, 0, st>>>(w.mm);
        ISB_LAUNCH_CHECK();
        k_ct_range<<<pass_grid(n, 8), CT_THREADS, 0, st>>>(y_true, dtype_true, y_pred, dtype_pred, n, drop, n_drop, w.mm);
        ISB_LAUNCH_CHECK();
        long long got[4];
        ISB_CUDA_CHECK(cudaMemcpyAsync(got, w.mm, sizeof(got), cudaMemcpyDeviceToHost, st));
        ISB_CUDA_CHECK(cudaStreamSynchronize(st));
        if (got[0] > got[1]) {                       // every pixel dropped
            for (int j = 0; j < 4; ++j) info[j] = 0;
            info[4] = info[5] = 0;
            return ISB_OK;
        }
        if (!narrow_a) { mm[0] = got[0]; mm[1] = got[1]; }
        if (!narrow_b) { mm[2] = got[2]; mm[3] = got[3]; }
        for (int j = 0; j < 2; ++j) {
            if ((unsigned long long)mm[2 * j + 1] - (unsigned long long)mm[2 * j] >= (unsigned long long)RANGE_MAX) {
                isb_set_error("the %s map's values span [%lld, %lld], more than the %lld values the presence table holds",
                              j ? "segmentation" : "annotation", mm[2 * j], mm[2 * j + 1], RANGE_MAX);
                return ISB_ERR_UNSUPPORTED;
            }
        }
    }
    const long long ra = mm[1] - mm[0] + 1, rb = mm[3] - mm[2] + 1;
    ISB_CUDA_CHECK(cudaMemsetAsync(w.pres_a, 0, sizeof(int32_t) * ra, st));
    ISB_CUDA_CHECK(cudaMemsetAsync(w.pres_b, 0, sizeof(int32_t) * rb, st));
    k_ct_mark<<<pass_grid(n, 8), CT_THREADS, 0, st>>>(y_true, dtype_true, y_pred, dtype_pred, n, drop, n_drop, mm[0], mm[2], w.pres_a, w.pres_b);
    ISB_LAUNCH_CHECK();
    if (int s = compact_count(w.pres_a, ra, w.cws_a, st, w.k + 0)) return s;
    if (int s = compact_count(w.pres_b, rb, w.cws_b, st, w.k + 1)) return s;
    long long k[2];
    ISB_CUDA_CHECK(cudaMemcpyAsync(k, w.k, sizeof(k), cudaMemcpyDeviceToHost, st));
    ISB_CUDA_CHECK(cudaStreamSynchronize(st));
    info[0] = k[0];
    info[1] = k[1];
    info[2] = mm[0];
    info[3] = ra;
    info[4] = mm[2];
    info[5] = rb;
    return ISB_OK;
}

extern "C" int isb_contingency_write(const void* y_true, int dtype_true, const void* y_pred, int dtype_pred, long long n, const int64_t* drop,
                                     int n_drop, const long long* info, void* ws, size_t ws_bytes, int64_t* values_true, int64_t* values_pred,
                                     int64_t* counts, isb_stream_t stream)
{
    if (int s = check_args(y_true, dtype_true, y_pred, dtype_pred, n, drop, n_drop)) return s;
    ISB_REQUIRE(ws && info, "null pointer");
    ISB_REQUIRE(ws_bytes >= isb_contingency_workspace_bytes(dtype_true, dtype_pred), "workspace too small");
    const long long ka = info[0], kb = info[1], ra = info[3], rb = info[5];
    ISB_REQUIRE(ka >= 0 && kb >= 0 && ra >= ka && rb >= kb && ra <= range_cap(dtype_true) && rb <= range_cap(dtype_pred),
                "info is not the output of isb_contingency_count");
    if (ka == 0 || kb == 0) return ISB_OK;
    ISB_REQUIRE(values_true && values_pred && counts, "null pointer");
    if (ka * kb > CELLS_MAX) {
        isb_set_error("a table of %lld x %lld cells is above the limit of %lld", ka, kb, CELLS_MAX);
        return ISB_ERR_UNSUPPORTED;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const CtWs w = carve(ws, dtype_true, dtype_pred);
    k_ct_dense<<<compact_tiles(ra), CPT_THREADS, 0, st>>>(w.pres_a, ra, info[2], compact_tile_offsets(w.cws_a, ra), values_true);
    ISB_LAUNCH_CHECK();
    k_ct_dense<<<compact_tiles(rb), CPT_THREADS, 0, st>>>(w.pres_b, rb, info[4], compact_tile_offsets(w.cws_b, rb), values_pred);
    ISB_LAUNCH_CHECK();
    const long long cells = ka * kb;
    ISB_CUDA_CHECK(cudaMemsetAsync(counts, 0, sizeof(int64_t) * cells, st));
    unsigned long long* out = (unsigned long long*)counts;
    if (cells <= SMEM_CELLS) {
        const size_t smem = sizeof(unsigned) * cells;
        if (smem > 48 * 1024) ISB_CUDA_CHECK(cudaFuncSetAttribute(k_ct_count<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_ct_count<true><<<pass_grid(n, 3), CT_THREADS, smem, st>>>(y_true, dtype_true, y_pred, dtype_pred, n, drop, n_drop, info[2], info[4],
                                                                   w.pres_a, w.pres_b, (int)kb, (int)cells, out);
    } else {
        k_ct_count<false><<<pass_grid(n, 8), CT_THREADS, 0, st>>>(y_true, dtype_true, y_pred, dtype_pred, n, drop, n_drop, info[2], info[4],
                                                                  w.pres_a, w.pres_b, (int)kb, (int)cells, out);
    }
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
