// wgmma.cuh -- thin inline-PTX wrappers for the Hopper (sm_90a) asynchronous machinery used by the tensor-core kernels:
// mbarrier, TMA (cp.async.bulk / cp.async.bulk.tensor) and the warpgroup MMA (wgmma.mma_async, TF32 inputs, FP32 accumulators
// in registers).  Descriptor encodings follow the PTX ISA "Matrix Descriptor Format" of wgmma.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace wgmma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- mbarrier -------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity), "r"(0x989680u)   // suspend-time hint: the warp sleeps in hardware instead of spinning
        : "memory");
    return ok != 0;
}
// Wait for the phase with the given parity to complete.  A watchdog turns a protocol bug into a trap (a failed launch the host
// reports) instead of a hung GPU: no wait in these kernels is legitimately longer than a few milliseconds.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    unsigned spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 1023u) == 0 && clock64() - t0 > 4000000000LL) __trap();
    }
}

// generic-proxy writes to shared memory (st.shared) -> visible to the async proxy (TMA, wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- TMA ------------------------------------------------------------
// 1-D bulk copy global -> shared, completion counted in bytes on an mbarrier (size and addresses multiples of 16 B)
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src_gmem, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
                 "l"(src_gmem), "r"(bytes), "r"(bar)
                 : "memory");
}
// 2-D tiled tensor-map load: box (c0.., c1..) of the tensor described by `tmap` -> shared
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const CUtensorMap* tmap, int c0, int c1, uint32_t bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst_smem),
                 "l"(tmap), "r"(c0), "r"(c1), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst_smem, const CUtensorMap* tmap, int c0, int c1, int c2, uint32_t bar)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(dst_smem),
                 "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* tmap)
{
    asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}

// ---------------------------------------------------------------- warpgroup MMA ------------------------------------------------
// A warpgroup is four consecutive warps (warp w of the group owns rows 16 w .. 16 w + 15 of the M = 64 tile).  wgmma.mma_async reads
// its register operands asynchronously: wg_fence() before the first MMA that uses registers written since, wg_commit() closes a group,
// wg_wait<n>() returns once at most n groups are pending -- only then may the accumulators or the A fragments be touched again.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// ---------------------------------------------------------------- descriptors ----------------------------------------------------
// Shared-memory matrix descriptor, K-major operand WITHOUT swizzle.  The operand is stored as "core matrices" of 8 rows (M or N)
// x 16 bytes (4 tf32 along K), each core matrix 128 contiguous bytes:
//   element (row, k) at  start + (row % 8) * 16 + (row / 8) * SBO + (k_bytes % 16) + (k_bytes / 16) * LBO
// bits [0,14) start >> 4 | [16,30) LBO >> 4 | [32,46) SBO >> 4 | [49,52) base offset = 0 | [62,64) layout = 0 (no swizzle)
__device__ __forceinline__ uint64_t smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes)
{
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, TF32 inputs, FP32 accumulators in registers; scale_d = 0 overwrites D.  Issued by all 128
// threads of the warpgroup.  Accumulator register i of a thread holds row 16 (warp % 4) + lane / 4 + 8 ((i / 2) % 2), column
// 8 (i / 4) + 2 (lane % 4) + i % 2.  B comes from shared memory through its descriptor, A from four registers per thread: rows
// lane / 4 and lane / 4 + 8 of the warp's 16, columns lane % 4 and lane % 4 + 4, as {(r, c), (r + 8, c), (r, c + 4), (r + 8, c + 4)}.
// Only the two widths the Leung-Malik contraction issues are spelled out: N = 48 (short bank) and N = 80 (full bank).
__device__ __forceinline__ void mma_tf32_rs(float (&d)[24], const uint32_t (&a)[4], uint64_t bdesc, int scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        "%16, %17, %18, %19, %20, %21, %22, %23}, {%24, %25, %26, %27}, %28, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void mma_tf32_rs(float (&d)[40], const uint32_t (&a)[4], uint64_t bdesc, int scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %45, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n80k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        "%32, %33, %34, %35, %36, %37, %38, %39}, {%40, %41, %42, %43}, %44, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}

// ---------------------------------------------------------------- host: tensor maps ----------------------------------------------
// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda); nullptr when unavailable
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static inline EncodeTiledFn encode_tiled_fn()
{
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

} // namespace wgmma
