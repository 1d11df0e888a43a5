// common.cuh -- shared helpers for the imsegm_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/imsegm_b200.h"

void isb_set_error(const char* fmt, ...);
extern long long g_isb_launches;

// stage timers (capi.cu): no-ops unless isb_profile_enable(1)
enum {
    ISB_PROF_PREPARE = 0, ISB_PROF_ASSIGN, ISB_PROF_UPDATE, ISB_PROF_FINALIZE, ISB_PROF_CONN, ISB_PROF_STATS, ISB_PROF_ADJ,
    ISB_PROF_ENERGY, ISB_PROF_GC, ISB_PROF_GATHER, ISB_PROF_GMM, ISB_PROF_LM, ISB_PROF_COUNT
};
int isb_prof_begin(int id, cudaStream_t st);
void isb_prof_end(int handle, cudaStream_t st);
struct ProfScope {
    int h; cudaStream_t st;
    ProfScope(int id, cudaStream_t s) : h(isb_prof_begin(id, s)), st(s) {}
    ~ProfScope() { if (h >= 0) isb_prof_end(h, st); }
};

#define ISB_CUDA_CHECK(call)                                                                      \
    do {                                                                                          \
        cudaError_t e__ = (call);                                                                 \
        if (e__ != cudaSuccess) {                                                                 \
            isb_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__));  \
            return ISB_ERR_CUDA;                                                                  \
        }                                                                                         \
    } while (0)

#define ISB_LAUNCH_CHECK()                                                                        \
    do {                                                                                          \
        ++g_isb_launches;                                                                         \
        cudaError_t e__ = cudaGetLastError();                                                     \
        if (e__ != cudaSuccess) {                                                                 \
            isb_set_error("%s:%d kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
            return ISB_ERR_CUDA;                                                                  \
        }                                                                                         \
    } while (0)

#define ISB_REQUIRE(cond, msg)                                          \
    do {                                                                \
        if (!(cond)) {                                                  \
            isb_set_error("%s:%d %s", __FILE__, __LINE__, msg);         \
            return ISB_ERR_ARG;                                         \
        }                                                               \
    } while (0)

static inline size_t isb_align(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// bump allocator over a caller-provided workspace
struct WsCarver {
    char* base;
    size_t off, cap;
    WsCarver(void* p, size_t bytes) : base((char*)p), off(0), cap(bytes) {}
    template <typename T> T* take(size_t n)
    {
        size_t o = isb_align(off);
        off = o + n * sizeof(T);
        return (T*)(base + o);
    }
    bool ok() const { return off <= cap; }
};

__device__ __forceinline__ double load_as_f64(const void* p, int dtype, size_t i)
{
    switch (dtype) {
        case ISB_U8: return (double)((const unsigned char*)p)[i];
        case ISB_U16: return (double)((const unsigned short*)p)[i];
        case ISB_F32: return (double)((const float*)p)[i];
        default: return ((const double*)p)[i];
    }
}

__device__ __forceinline__ float load_as_f32(const void* p, int dtype, size_t i)
{
    switch (dtype) {
        case ISB_U8: return (float)((const unsigned char*)p)[i];
        case ISB_U16: return (float)((const unsigned short*)p)[i];
        case ISB_F32: return ((const float*)p)[i];
        default: return (float)((const double*)p)[i]; // round-to-nearest-even, same as numpy astype(float32)
    }
}

// order-preserving map double <-> uint64 (for atomicMin/atomicMax on doubles)
__device__ __forceinline__ unsigned long long f64_ordered(double d)
{
    unsigned long long u = (unsigned long long)__double_as_longlong(d);
    return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double f64_unordered(unsigned long long u)
{
    u = (u & 0x8000000000000000ull) ? (u & 0x7FFFFFFFFFFFFFFFull) : ~u;
    return __longlong_as_double((long long)u);
}
