// frz_hd.cuh — FRZ_HD, the qualifier of functions that are compiled both for the device and, by the g++ harnesses under
// tests/harness/, for the CPU: inlined device and host code under nvcc, a plain inline function otherwise.
#pragma once

#if defined(__CUDACC__)
#define FRZ_HD __host__ __device__ __forceinline__
#else
#define FRZ_HD inline
#endif
