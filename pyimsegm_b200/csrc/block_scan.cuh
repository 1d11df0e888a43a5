// block_scan.cuh -- integer exclusive prefix sums over one CTA, on cub::BlockScan.  Kept apart from common.cuh so that only the
// sources that scan pull in CUB.  Every CTA scan ends with a barrier: cub's TempStorage may then be reused by the next call (in a
// loop, or a second scan in the same kernel), and what out() wrote is visible to the whole CTA on return.
#pragma once
#include <cub/block/block_scan.cuh>

namespace {

// the exclusive prefix of v over the CTA's NT threads; total = the CTA's sum, in every thread.  Warp scans rather than cub's default
// raking, whose 1 024-thread int64 scan spills under __launch_bounds__(1024); inclusive minus v (exact over integers) rather than
// ExclusiveSum, which costs the compaction write kernels a spill.
template <int NT, typename T>
__device__ __forceinline__ T cta_exclusive_sum(T v, T& total)
{
    using Scan = cub::BlockScan<T, NT, cub::BLOCK_SCAN_WARP_SCANS>;
    __shared__ typename Scan::TempStorage tmp;
    T incl;
    Scan(tmp).InclusiveSum(v, incl, total);
    __syncthreads();
    return incl - v;
}

// one CTA walks [0, n) in rounds of NT: out(i, sum of val(j) for j < i) for every i; returns the sum over [0, n), in every thread
template <int NT, typename T, typename Val, typename Out>
__device__ __forceinline__ T cta_scan_chunks(int n, Val val, Out out)
{
    T carry = 0;
    for (int base = 0; base < n; base += NT) {
        const int i = base + threadIdx.x;
        T total;
        const T excl = cta_exclusive_sum<NT>(i < n ? val(i) : T(0), total);
        if (i < n) out(i, carry + excl);
        carry += total;
    }
    __syncthreads();
    return carry;
}

} // namespace
