// wgmma_selftest.cu -- known-answer test of the wgmma plumbing in wgmma.cuh (descriptor encoding of B, the register fragments of
// A, the accumulator layout): D[128, N] = A[128, K] * B[N, K]^T in one CTA of two warpgroups (rows 0..63 and 64..127) with TF32
// inputs and FP32 accumulators in registers.  Test infrastructure for tests/test_gpu_umma.py; the Leung-Malik contraction
// (lm_texture.cu) feeds its operands in exactly these layouts: A from registers, B from K-major shared memory.
#include "common.cuh"
#include "wgmma.cuh"

namespace {

using namespace wgmma;

// one warpgroup's 64 x N product; K % 8 == 0.  A from registers, straight from global memory
template <int N>
__device__ void selftest_rows(const float* __restrict__ A, uint32_t sB, int K, float* __restrict__ D)
{
    const int wg = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
    const uint32_t b_lbo = (uint32_t)(N >> 3) * 128, sbo = 128;
    const int r0 = 64 * wg + 16 * w + (lane >> 2), c0 = lane & 3;
    wg_fence();
    for (int kk = 0; kk < K / 8; ++kk) {
        const uint64_t bd = smem_desc(sB + kk * 2 * b_lbo, b_lbo, sbo);
        const float* a = A + (size_t)r0 * K + 8 * kk + c0;
        const uint32_t af[4] = { __float_as_uint(a[0]), __float_as_uint(a[8 * K]), __float_as_uint(a[4]), __float_as_uint(a[8 * K + 4]) };
        wg_fence();
        mma_tf32_rs(d, af, bd, kk > 0);
        wg_commit();
        wg_wait<0>();
    }
#pragma unroll
    for (int i = 0; i < N / 2; ++i)
        D[(size_t)(r0 + 8 * ((i >> 1) & 1)) * N + 8 * (i >> 2) + 2 * c0 + (i & 1)] = d[i];
}

// A [128][K] and B [N][K] row-major f32 in global memory (values already representable in tf32)
__global__ void __launch_bounds__(256) k_wgmma_selftest(const float* __restrict__ A, const float* __restrict__ B, int N, int K,
                                                        float* __restrict__ D)
{
    extern __shared__ __align__(128) unsigned char sm[];
    float* sB = (float*)sm;                 // [K/4][N/8][8][4]
    for (int i = threadIdx.x; i < N * K; i += blockDim.x) {
        const int n = i / K, k = i - n * K;
        sB[(k >> 2) * ((N >> 3) * 32) + (n >> 3) * 32 + (n & 7) * 4 + (k & 3)] = B[i];
    }
    fence_proxy_async();
    __syncthreads();
    if (N == 48) selftest_rows<48>(A, smem_u32(sB), K, D);
    else selftest_rows<80>(A, smem_u32(sB), K, D);
}

} // namespace

extern "C" int isb_wgmma_selftest(const float* A, const float* B, int N, int K, int variant, float* D, isb_stream_t stream)
{
    ISB_REQUIRE(A && B && D, "null pointer");
    ISB_REQUIRE((N == 48 || N == 80) && K >= 8 && K <= 64 && K % 8 == 0, "N must be 48 or 80, K a multiple of 8 <= 64");
    ISB_REQUIRE(variant == 2, "variant must be 2 (A from registers)");
    const size_t smem = sizeof(float) * (size_t)N * K;
    k_wgmma_selftest<<<1, 256, smem, (cudaStream_t)stream>>>(A, B, N, K, D);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
