// compact.cuh -- order-preserving stream compaction of the nonzero elements of an array: per tile counts, one scan of the tile
// counts, then each tile writes its elements in input order.  Shared by the label-map masks of labeling.cu and the colour
// histogram of annotation.cu; each source keeps its own write kernel (what it writes per element differs).
#pragma once
#include "common.cuh"
#include "block_scan.cuh"

namespace {

constexpr int CPT_THREADS = 256, CPT_PER = 16, CPT_TILE = CPT_THREADS * CPT_PER;

inline int compact_tiles(long long n) { return (int)((n + CPT_TILE - 1) / CPT_TILE); }

template <typename T>
__device__ __forceinline__ int thread_count(const T* __restrict__ v, long long beg, long long n)
{
    int c = 0;
    for (int k = 0; k < CPT_PER; ++k) {
        const long long i = beg + k;
        if (i < n && v[i]) ++c;
    }
    return c;
}

template <typename T>
__global__ void __launch_bounds__(CPT_THREADS) k_compact_count(const T* __restrict__ v, long long n, long long* __restrict__ tile_count)
{
    const long long beg = (long long)blockIdx.x * CPT_TILE + (long long)threadIdx.x * CPT_PER;
    int total;
    cta_exclusive_sum<CPT_THREADS>(thread_count(v, beg, n), total);
    if (threadIdx.x == 0) tile_count[blockIdx.x] = total;
}

// exclusive scan of the tile counts in one CTA (tiles are few: 16 384 for an 8192^2 map); total -> tile_off[n_tiles]
__global__ void __launch_bounds__(1024) k_compact_scan(const long long* __restrict__ tile_count, int n_tiles, long long* __restrict__ tile_off)
{
    const long long total = cta_scan_chunks<1024, long long>(n_tiles, [&](int b) { return tile_count[b]; },
                                                             [&](int b, long long off) { tile_off[b] = off; });
    if (threadIdx.x == 0) tile_off[n_tiles] = total;
}

inline size_t compact_workspace_bytes(long long n)
{
    const int nt = compact_tiles(n);
    return isb_align(sizeof(long long) * (size_t)nt) + isb_align(sizeof(long long) * ((size_t)nt + 1));
}

// the count phase: per-tile counts and their scan into ws, the number of nonzero elements into the DEVICE int64 *total
template <typename T>
int compact_count(const T* v, long long n, void* ws, cudaStream_t st, long long* total)
{
    const int nt = compact_tiles(n);
    WsCarver c(ws, compact_workspace_bytes(n));
    long long* tile_count = c.take<long long>(nt);
    long long* tile_off = c.take<long long>((size_t)nt + 1);
    k_compact_count<T><<<nt, CPT_THREADS, 0, st>>>(v, n, tile_count);
    ISB_LAUNCH_CHECK();
    k_compact_scan<<<1, 1024, 0, st>>>(tile_count, nt, tile_off);
    ISB_LAUNCH_CHECK();
    ISB_CUDA_CHECK(cudaMemcpyAsync(total, tile_off + nt, sizeof(long long), cudaMemcpyDeviceToDevice, st));
    return ISB_OK;
}

// the tile offsets the count phase left in ws
inline const long long* compact_tile_offsets(const void* ws, long long n)
{
    WsCarver c(const_cast<void*>(ws), compact_workspace_bytes(n));
    c.take<long long>(compact_tiles(n));
    return c.take<long long>((size_t)compact_tiles(n) + 1);
}

} // namespace
