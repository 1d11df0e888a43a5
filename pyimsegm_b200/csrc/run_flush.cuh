// run_flush.cuh -- warp-aggregated flush of per-lane runs into a histogram.  Shared by the colour histogram of annotation.cu and the
// contingency table of classification.cu.
#pragma once
#include "common.cuh"

namespace {

// Every lane keeps a run (key, count) over its pixels and calls this with flush = true when the key changes and at the end; every
// lane of the warp must call it.  The runs of all flushing lanes with the same key are first summed (__match_any_sync,
// __reduce_add_sync), so one add(key, sum) -- one atomic -- serves the whole warp: a constant map issues one per 32 runs.
template <typename Add>
__device__ __forceinline__ void flush_run(bool flush, unsigned key, unsigned cnt, Add add)
{
    const unsigned fl = __ballot_sync(0xffffffffu, flush);
    if (flush) {
        const unsigned peers = __match_any_sync(fl, key);
        const unsigned s = __reduce_add_sync(peers, cnt);
        if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) add(key, s);
    }
}

} // namespace
