// emu_shims/cuda_runtime.h -- TEST INFRASTRUCTURE: stands in for <cuda_runtime.h> when a libsis3d source is compiled for
// the host (tools/cuda_host_emu.py); see host_emu.h.
#pragma once
#include <cstddef>
#include <cstring>
#include "host_emu.h"
typedef int cudaError_t;
enum { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
template <class F> inline int cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }
inline int cudaMemsetAsync(void *p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }

// ---- single-rounding float intrinsics (the emulation is compiled with -ffp-contract=off, so a*b and a+b round once each)
#include <cmath>
#include <cstdlib>
inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
inline float __fmaf_rn(float a, float b, float c) { return std::fmaf(a, b, c); }
inline float __uint_as_float(unsigned u) { float f; std::memcpy(&f, &u, 4); return f; }
inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
inline int __ffsll(long long v) { return __builtin_ffsll(v); }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline void __trap() { std::abort(); }
// atomics: relaxed RMW on plain objects, visible to ThreadSanitizer as atomic accesses
template <class T> inline T atomicAdd(T *p, T v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
template <class T> inline T atomicOr(T *p, T v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
template <class T> inline T atomicMax(T *p, T v) {
    T old = __atomic_load_n(p, __ATOMIC_RELAXED);
    while (old < v && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
    return old;
}
template <class T> inline T atomicMin(T *p, T v) {
    T old = __atomic_load_n(p, __ATOMIC_RELAXED);
    while (v < old && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
    return old;
}
inline long long __double_as_longlong(double d) { long long u; std::memcpy(&u, &d, 8); return u; }
inline double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }
inline double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }
