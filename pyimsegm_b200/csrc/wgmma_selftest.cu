// wgmma_selftest.cu -- known-answer test of the wgmma plumbing in wgmma.cuh (descriptor encodings, the register fragments of A,
// the accumulator layout): D[128, N] = A[128, K] * B[N, K]^T in one CTA of two warpgroups (rows 0..63 and 64..127) with TF32
// inputs and FP32 accumulators in registers.  Test infrastructure for tests/test_gpu_umma.py; the Leung-Malik contraction
// (lm_texture.cu) uses exactly these operand layouts.
#include "common.cuh"
#include "wgmma.cuh"

namespace {

using namespace wgmma;

// one warpgroup's 64 x N product; K % 8 == 0.  variant 0 / 1: A from shared memory (1 swaps the LBO / SBO fields, a diagnostic),
// variant 2: A from registers, straight from global memory
template <int N>
__device__ void selftest_rows(const float* __restrict__ A, uint32_t sA, uint32_t sB, int K, int variant, float* __restrict__ D)
{
    const int wg = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
    const uint32_t a_lbo = 16 * 128, b_lbo = (uint32_t)(N >> 3) * 128, sbo = 128;
    const int r0 = 64 * wg + 16 * w + (lane >> 2), c0 = lane & 3;
    wg_fence();
    for (int kk = 0; kk < K / 8; ++kk) {
        const uint32_t b_addr = sB + kk * 2 * b_lbo;
        const uint64_t bd = variant == 1 ? smem_desc(b_addr, sbo, b_lbo) : smem_desc(b_addr, b_lbo, sbo);
        if (variant == 2) {
            const float* a = A + (size_t)r0 * K + 8 * kk + c0;
            const uint32_t af[4] = { __float_as_uint(a[0]), __float_as_uint(a[8 * K]), __float_as_uint(a[4]), __float_as_uint(a[8 * K + 4]) };
            wg_fence();
            mma_tf32_rs(d, af, bd, kk > 0);
        } else {
            // this warpgroup's 64 rows start 8 core matrices (8 x 128 bytes) into every k-chunk of A
            const uint32_t a_addr = sA + kk * 2 * a_lbo + wg * 8 * 128;
            const uint64_t ad = variant ? smem_desc(a_addr, sbo, a_lbo) : smem_desc(a_addr, a_lbo, sbo);
            mma_tf32_ss(d, ad, bd, kk > 0);
        }
        wg_commit();
        wg_wait<0>();
    }
#pragma unroll
    for (int i = 0; i < N / 2; ++i)
        D[(size_t)(r0 + 8 * ((i >> 1) & 1)) * N + 8 * (i >> 2) + 2 * c0 + (i & 1)] = d[i];
}

// A [128][K] and B [N][K] row-major f32 in global memory (values already representable in tf32)
__global__ void __launch_bounds__(256) k_wgmma_selftest(const float* __restrict__ A, const float* __restrict__ B, int N, int K, int variant,
                                                        float* __restrict__ D)
{
    extern __shared__ __align__(128) unsigned char sm[];
    float* sA = (float*)sm;                 // [K/4][16][8][4]
    float* sB = sA + 128 * K;               // [K/4][N/8][8][4]
    const int tid = threadIdx.x;
    for (int i = tid; i < 128 * K; i += blockDim.x) {
        const int m = i / K, k = i - m * K;
        sA[(k >> 2) * (16 * 32) + (m >> 3) * 32 + (m & 7) * 4 + (k & 3)] = A[i];
    }
    for (int i = tid; i < N * K; i += blockDim.x) {
        const int n = i / K, k = i - n * K;
        sB[(k >> 2) * ((N >> 3) * 32) + (n >> 3) * 32 + (n & 7) * 4 + (k & 3)] = B[i];
    }
    fence_proxy_async();
    __syncthreads();
    const uint32_t a = smem_u32(sA), b = smem_u32(sB);
    switch (N) {
    case 16: selftest_rows<16>(A, a, b, K, variant, D); break;
    case 48: selftest_rows<48>(A, a, b, K, variant, D); break;
    case 80: selftest_rows<80>(A, a, b, K, variant, D); break;
    case 240: selftest_rows<240>(A, a, b, K, variant, D); break;
    default: selftest_rows<256>(A, a, b, K, variant, D); break;
    }
}

// dependent-issue latency of the FP64 pipe: one warp, chains of n dependent operations; out[0..2] = clocks per DADD, DMUL, DFMA, out[3] = sink
__global__ void k_fp64_latency(int n, double seed, double* out)
{
    double a = seed, b = seed * 0.5, c = seed * 0.25;
    long long t0 = clock64();
    for (int i = 0; i < n; ++i) a = __dadd_rn(a, seed);
    long long t1 = clock64();
    for (int i = 0; i < n; ++i) b = __dmul_rn(b, seed);
    long long t2 = clock64();
    for (int i = 0; i < n; ++i) c = __fma_rn(c, seed, seed);
    long long t3 = clock64();
    if (threadIdx.x == 0) {
        out[0] = (double)(t1 - t0) / n; out[1] = (double)(t2 - t1) / n; out[2] = (double)(t3 - t2) / n; out[3] = a + b + c;
    }
}

} // namespace

extern "C" int isb_fp64_latency(int n, double* out, isb_stream_t stream)
{
    ISB_REQUIRE(out && n > 0, "bad arguments");
    k_fp64_latency<<<1, 32, 0, (cudaStream_t)stream>>>(n, 1.0000001, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_wgmma_selftest(const float* A, const float* B, int N, int K, int variant, float* D, isb_stream_t stream)
{
    ISB_REQUIRE(A && B && D, "null pointer");
    ISB_REQUIRE((N == 16 || N == 48 || N == 80 || N == 240 || N == 256) && K >= 8 && K <= 64 && K % 8 == 0,
                "N must be 16, 48, 80, 240 or 256, K a multiple of 8 <= 64");
    ISB_REQUIRE(variant >= 0 && variant <= 2, "variant: 0 / 1 = A from shared memory (descriptor field order), 2 = A from registers");
    const size_t smem = sizeof(float) * (size_t)(128 + N) * K;
    ISB_CUDA_CHECK(cudaFuncSetAttribute(k_wgmma_selftest, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_wgmma_selftest<<<1, 256, smem, (cudaStream_t)stream>>>(A, B, N, K, variant, D);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
