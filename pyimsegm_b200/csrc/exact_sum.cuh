// exact_sum.cuh -- order-free f64 sums for the per-segment statistics (segment_stats.cu, native_misc.cu).
//
// The statistics kernels flush per-run partial sums of f32 values (or of f32 products) into one total per label from many warps
// at once.  Added with f64 atomics, those totals depend on the order in which the flushes arrive, so two launches on the same input
// could differ in the last bits.  Here every flushed partial is added EXACTLY into a fixed-point accumulator with integer atomics,
// and the total is rounded to f64 once (round to nearest, ties to even): the result is the correctly rounded sum of the partials,
// which does not depend on the order of the flushes (Python's math.fsum of the same partials gives the same bits).
//
// Why a fixed point fits: every partial is a sum of f32 values, hence a multiple of 2^-149 (the least f32 subnormal), and below
// 2^137 in magnitude (at most 512 values below 2^128); the total of 2^31 of them stays below 2^168.  Bits [-149, 171) in XS_DIGITS
// digits of 32 bits, each kept in a signed 64-bit word so that carries can wait: a partial adds less than 2^32 to at most three
// words, so a word takes 2^31 partials before it could overflow -- callers bound the flushes by the pixel count, <= 2^31.
// Infinite and NaN partials set flag bits instead (3 per sum: +inf, -inf, NaN) and round as IEEE summation in any order would.
#pragma once
#include "common.cuh"

namespace {

constexpr int XS_DIGITS = 10;
constexpr int XS_LSB = -149;

// add the partial t into sum j of a label: digits w [XS_DIGITS], flag word *flag (bits 3j .. 3j+2)
__device__ __forceinline__ void xs_add(long long* w, unsigned* flag, int j, double t)
{
    if (t == 0.0) return;
    if (!isfinite(t)) {
        atomicOr(flag, (isnan(t) ? 4u : (t > 0 ? 1u : 2u)) << (3 * j));
        return;
    }
    const unsigned long long u = (unsigned long long)__double_as_longlong(t);
    const int ex = (int)((u >> 52) & 0x7ff);
    unsigned long long mant = u & ((1ull << 52) - 1);
    int sh = (ex ? ex - 1075 : -1074) - XS_LSB;     // bit position of mant's lsb above 2^-149
    if (ex) mant |= 1ull << 52;
    if (sh < 0) { mant = sh > -64 ? mant >> -sh : 0; sh = 0; }   // the bits shifted out are zero (the f32 grid)
    const int k = sh >> 5, r = sh & 31;
    const unsigned long long lo = mant << r, hi = r ? mant >> (64 - r) : 0;
    const unsigned long long d[3] = {lo & 0xffffffffull, lo >> 32, hi};
    const bool neg = u >> 63;
#pragma unroll
    for (int i = 0; i < 3; ++i)
        if (d[i] && k + i < XS_DIGITS) atomicAdd((unsigned long long*)&w[k + i], neg ? 0ull - d[i] : d[i]);
}

// the correctly rounded f64 value of sum j: w [XS_DIGITS] digits, fl the label's flag word
__device__ __forceinline__ double xs_round(const long long* w, unsigned fl, int j)
{
    const unsigned f = (fl >> (3 * j)) & 7u;
    if ((f & 4u) || f == 3u) return __longlong_as_double(0x7ff8000000000000ll);
    if (f) return f == 1u ? __longlong_as_double(0x7ff0000000000000ll) : __longlong_as_double((long long)0xfff0000000000000ull);
    unsigned dig[XS_DIGITS];
    long long carry = 0;
#pragma unroll
    for (int i = 0; i < XS_DIGITS; ++i) {    // propagate the carries: dig = 32-bit two's-complement digits of the total
        const long long v = w[i];
        const unsigned long long lo = (unsigned long long)(v & 0xffffffffll) + (unsigned long long)(carry & 0xffffffffll);
        dig[i] = (unsigned)lo;
        carry = (v >> 32) + (carry >> 32) + (long long)(lo >> 32);
    }
    const bool neg = carry < 0;
    if (neg) {                               // magnitude of a negative total
        unsigned long long c = 1;
#pragma unroll
        for (int i = 0; i < XS_DIGITS; ++i) { c += (unsigned long long)(~dig[i]); dig[i] = (unsigned)c; c >>= 32; }
    }
    int kt = XS_DIGITS - 1;
    while (kt >= 0 && dig[kt] == 0) --kt;
    if (kt < 0) return 0.0;
    // the 64 bits below and at the top bit, with every lower bit folded into bit 0 (sticky): __ull2double_rn then rounds as the
    // exact value would round
    const unsigned long long top = dig[kt];
    const unsigned long long mid = ((unsigned long long)(kt >= 1 ? dig[kt - 1] : 0u) << 32) | (kt >= 2 ? dig[kt - 2] : 0u);
    const int s = 32 - __clzll(top << 32);   // top bit of digit kt at 63 + s of the 96 bits (top, mid), 1 <= s <= 32
    unsigned long long T = (top << (64 - s)) | (mid >> s);
    bool sticky = (mid & ((1ull << s) - 1)) != 0;
    for (int i = 0; i < kt - 2; ++i) sticky |= dig[i] != 0;
    T |= sticky ? 1ull : 0ull;
    const double m = ldexp(__ull2double_rn(T), 32 * (kt - 2) + s + XS_LSB);
    return neg ? -m : m;
}

// the exact sums of nsums values per label for nb labels, digits then flag words, carved from base (nullptr: the size only)
static size_t xs_carve(void* base, int nb, int nsums, long long** x, unsigned** flag)
{
    WsCarver c(base, 0);
    *x = c.take<long long>((size_t)nsums * XS_DIGITS * nb);
    *flag = c.take<unsigned>(nb);
    return isb_align(c.off);
}

// device memory for one call of an entry whose caller passes no workspace, allocated and freed in the order of its stream
struct StreamScratch {
    void* p = nullptr;
    cudaStream_t st;
    explicit StreamScratch(cudaStream_t s) : st(s) {}
    ~StreamScratch() { if (p) cudaFreeAsync(p, st); }
};

// out[i] += the rounded sum i, i = label * nsums + sum: x [nb * nsums][XS_DIGITS], flag [nb]
__global__ void k_exact_fold(int nb, int nsums, const long long* __restrict__ x, const unsigned* __restrict__ flag, double* out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)nb * nsums) return;
    out[i] += xs_round(x + i * XS_DIGITS, flag[i / nsums], (int)(i % nsums));
}

} // namespace
