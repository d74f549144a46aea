// Shared host/device helpers for libgifb200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "gifb200.h"

namespace gifb200 {

extern thread_local char g_err[512];
extern long long g_launches;

inline int fail(int code, const char* what, const char* detail = nullptr) {
    snprintf(g_err, sizeof(g_err), "%s%s%s", what, detail ? ": " : "", detail ? detail : "");
    return code;
}

inline int check_launch(const char* kernel) {
    ++g_launches;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(GIFB200_E_CUDA, kernel, cudaGetErrorString(e));
    return GIFB200_OK;
}

#define GIFB200_LAUNCH_CHECK(name)                      \
    do {                                                \
        int _rc = ::gifb200::check_launch(name);        \
        if (_rc != GIFB200_OK) return _rc;              \
    } while (0)

#define GIFB200_REQUIRE(cond, code, msg)                 \
    do {                                                 \
        if (!(cond)) return ::gifb200::fail(code, msg);  \
    } while (0)

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
inline int cdiv(long long a, long long b) { return static_cast<int>((a + b - 1) / b); }

constexpr int kNumSMs = 132;  // H100 SXM

// Deterministic cross-block sums.  A float atomicAdd per block adds the partial sums in whatever order the blocks finish, so
// the result changes in its last bits from run to run, and an optimiser step turns that into visibly different weights.
// Instead every block writes its partial sum to its own slot, part[slot * n + i]: slots_take points the kernel's output
// pointer at a stream-ordered buffer (cudaMallocAsync, so it also works inside a CUDA graph), slots_reduce adds the slots
// in slot order into the original output and frees the buffer.
struct Slots {
    float* part = nullptr;
    float* out = nullptr;
    int count = 0;
    long long n = 0;
};
int slots_take(Slots& s, float*& out, int count, long long n, cudaStream_t st);
int slots_reduce(Slots& s, cudaStream_t st);

__device__ __forceinline__ float round_tf32(float v) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return __uint_as_float(r);
}

// fused convolution epilogue: y = lrelu(acc + bias[o]) * gain (optionally tf32-rounded); act == 0: identity
struct ConvEpilogue {
    int act;
    const float* bias;
    float slope, gain;
    int rtf32;
};
__device__ __forceinline__ float apply_epilogue(const ConvEpilogue& e, float acc, int o) {
    if (!e.act) return acc;
    float t = acc + (e.bias ? __ldg(e.bias + o) : 0.f);
    t = (t > 0.f ? t : t * e.slope) * e.gain;
    return e.rtf32 ? round_tf32(t) : t;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace gifb200
