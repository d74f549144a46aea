// Memory-bound elementwise / reduction kernels of the StyleGAN2 hot path (channels-last fp32).
// Roofline for all of them is HBM: algorithmic bytes = inputs read once + outputs written once.
#include <cuda_bf16.h>

#include <mutex>

#include "common.cuh"

namespace gifb200 {

thread_local char g_err[512] = "";
long long g_launches = 0;

// ------------------------------------------------------------------------------------------------ bias_act
// t = x*rowscale[b,c] + add + bias[c]; y = lrelu(t)*gain.  One float4 (4 channels) per thread-iteration,
// grid-stride over rows so that the grid is a multiple of the SM count.
template <bool VEC>
__global__ void __launch_bounds__(256) bias_act_kernel(const float* __restrict__ x, const float* __restrict__ rowscale,
                                                       const float* __restrict__ add, const float* __restrict__ bias,
                                                       float* __restrict__ y, long long total, int P, int C, float slope,
                                                       float gain, int rtf32) {
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    if (VEC) {
        const long long nvec = total >> 2;
        const int c4n = C >> 2;
        for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec; v += stride) {
            const int c = static_cast<int>(v % c4n) << 2;
            float4 t = __ldcs(reinterpret_cast<const float4*>(x) + v);
            if (rowscale) {
                const long long b = (v / c4n) / P;
                const float4 s = *reinterpret_cast<const float4*>(rowscale + b * C + c);
                t.x *= s.x; t.y *= s.y; t.z *= s.z; t.w *= s.w;
            }
            if (add) {
                const float4 a = __ldcs(reinterpret_cast<const float4*>(add) + v);
                t.x += a.x; t.y += a.y; t.z += a.z; t.w += a.w;
            }
            if (bias) {
                const float4 bb = *reinterpret_cast<const float4*>(bias + c);
                t.x += bb.x; t.y += bb.y; t.z += bb.z; t.w += bb.w;
            }
            t.x = (t.x > 0.f ? t.x : t.x * slope) * gain;
            t.y = (t.y > 0.f ? t.y : t.y * slope) * gain;
            t.z = (t.z > 0.f ? t.z : t.z * slope) * gain;
            t.w = (t.w > 0.f ? t.w : t.w * slope) * gain;
            if (rtf32) { t.x = round_tf32(t.x); t.y = round_tf32(t.y); t.z = round_tf32(t.z); t.w = round_tf32(t.w); }
            reinterpret_cast<float4*>(y)[v] = t;
        }
    } else {
        for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
            const int c = static_cast<int>(i % C);
            float t = x[i];
            if (rowscale) t *= rowscale[((i / C) / P) * C + c];
            if (add) t += add[i];
            if (bias) t += bias[c];
            t = (t > 0.f ? t : t * slope) * gain;
            y[i] = rtf32 ? round_tf32(t) : t;
        }
    }
}

template <bool VEC>
__global__ void __launch_bounds__(256) act_bwd_kernel(const float* __restrict__ gy, const float* __restrict__ y,
                                                      float* __restrict__ gx, long long n, float slope, float gain,
                                                      int rtf32) {
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    if (VEC) {
        const long long nvec = n >> 2;
        for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec; v += stride) {
            const float4 g = __ldcs(reinterpret_cast<const float4*>(gy) + v);
            const float4 o = __ldcs(reinterpret_cast<const float4*>(y) + v);
            float4 r;
            r.x = g.x * gain * (o.x > 0.f ? 1.f : slope);
            r.y = g.y * gain * (o.y > 0.f ? 1.f : slope);
            r.z = g.z * gain * (o.z > 0.f ? 1.f : slope);
            r.w = g.w * gain * (o.w > 0.f ? 1.f : slope);
            if (rtf32) { r.x = round_tf32(r.x); r.y = round_tf32(r.y); r.z = round_tf32(r.z); r.w = round_tf32(r.w); }
            reinterpret_cast<float4*>(gx)[v] = r;
        }
    } else {
        for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        {
            const float r = gy[i] * gain * (y[i] > 0.f ? 1.f : slope);
            gx[i] = rtf32 ? round_tf32(r) : r;
        }
    }
}

// ------------------------------------------------------------------------------------------------ reductions
// out[g,c] = sum_r x[g,r,c].  Block = 32 (channels) x 8 (row lanes); grid = (C/32, row chunks, G).  The reductions below
// store one partial sum per (row chunk, output element) in a Slots buffer (common.cuh): slot = blockIdx.y, G*C floats per
// slot (the bias gradient of the tail kernels: slot = (b, row chunk), C floats per slot).
__global__ void __launch_bounds__(256) rows_sum_kernel(const float* __restrict__ x, float* __restrict__ out, int rows,
                                                       int C, int rows_per_block) {
    __shared__ float sm[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const int g = blockIdx.z;
    const int r0 = blockIdx.y * rows_per_block;
    const int r1 = min(rows, r0 + rows_per_block);
    float acc = 0.f;
    if (c < C) {
        const float* base = x + (static_cast<long long>(g) * rows) * C + c;
        for (int r = r0 + threadIdx.y; r < r1; r += 8) acc += base[static_cast<long long>(r) * C];
    }
    sm[threadIdx.y][threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
        float t = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) t += sm[j][threadIdx.x];
        out[(static_cast<long long>(blockIdx.y) * gridDim.z + g) * C + c] = t;
    }
}

// out[b,c] = sum_p a[b,p,c]*b2[b,p,c]  (same decomposition)
__global__ void __launch_bounds__(256) spatial_dot_kernel(const float* __restrict__ a, const float* __restrict__ b2,
                                                          float* __restrict__ out, int rows, int C, int rows_per_block) {
    __shared__ float sm[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const int g = blockIdx.z;
    const int r0 = blockIdx.y * rows_per_block;
    const int r1 = min(rows, r0 + rows_per_block);
    float acc = 0.f;
    if (c < C) {
        const long long base = (static_cast<long long>(g) * rows) * C + c;
        for (int r = r0 + threadIdx.y; r < r1; r += 8) {
            const long long i = base + static_cast<long long>(r) * C;
            acc += a[i] * b2[i];
        }
    }
    sm[threadIdx.y][threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
        float t = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) t += sm[j][threadIdx.x];
        out[(static_cast<long long>(blockIdx.y) * gridDim.z + g) * C + c] = t;
    }
}

// ------------------------------------------------------------------------------------------------ fused backward passes
// Backward of the StyledConv tail y = lrelu(acc*d[b,c] + noise + bias[c])*gain in ONE pass over (gy, y, acc):
//   gt = gy*gain*(y>0 ? 1 : slope)   (gradient of the pre-activation: goes to the noise branch)      -> written
//   gacc = gt*d[b,c]                 (gradient of the convolution accumulator)                       -> written
//   gb[c] += sum gt ;  gd[b,c] += sum gt*acc                                                          -> reduced
// instead of four kernels (act_bwd, chan_scale, spatial_dot, rows_sum) that read gt three more times.
__global__ void __launch_bounds__(256) tail_bwd_kernel(const float* __restrict__ gy, const float* __restrict__ y,
                                                       const float* __restrict__ acc, const float* __restrict__ d,
                                                       float* __restrict__ gt, float* __restrict__ gacc,
                                                       float* __restrict__ gb, float* __restrict__ gd, int rows, int C,
                                                       int rows_per_block, float slope, float gain, int rtf32) {
    __shared__ float sm[2][8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * rows_per_block;
    const int r1 = min(rows, r0 + rows_per_block);
    float sb = 0.f, sd = 0.f;
    if (c < C) {
        const float dv = d ? d[static_cast<long long>(b) * C + c] : 1.f;
        const long long base = (static_cast<long long>(b) * rows) * C + c;
        for (int r = r0 + threadIdx.y; r < r1; r += 8) {
            const long long i = base + static_cast<long long>(r) * C;
            float g = __ldcs(gy + i) * gain * (__ldcs(y + i) > 0.f ? 1.f : slope);
            float ga = g * dv;
            sb += g;
            if (gd) sd += g * __ldcs(acc + i);
            if (rtf32) { g = round_tf32(g); ga = round_tf32(ga); }
            if (gt) gt[i] = g;
            if (gacc) gacc[i] = ga;
        }
    }
    sm[0][threadIdx.y][threadIdx.x] = sb;
    sm[1][threadIdx.y][threadIdx.x] = sd;
    __syncthreads();
    if (threadIdx.y < 2 && c < C) {
        float t = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) t += sm[threadIdx.y][j][threadIdx.x];
        if (threadIdx.y == 0) { if (gb) gb[(static_cast<long long>(b) * gridDim.y + blockIdx.y) * C + c] = t; }
        else if (gd) gd[(static_cast<long long>(blockIdx.y) * gridDim.z + b) * C + c] = t;
    }
}

// Backward of y = x*s[b,c] in one pass over (gy, x):  gx = gy*s (written),  gs[b,c] += sum gy*x (reduced).
__global__ void __launch_bounds__(256) scale_bwd_kernel(const float* __restrict__ gy, const float* __restrict__ x,
                                                        const float* __restrict__ s, float* __restrict__ gx,
                                                        float* __restrict__ gs, int rows, int C, int rows_per_block,
                                                        int rtf32) {
    __shared__ float sm[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * rows_per_block;
    const int r1 = min(rows, r0 + rows_per_block);
    float acc = 0.f;
    if (c < C) {
        const float sv = s[static_cast<long long>(b) * C + c];
        const long long base = (static_cast<long long>(b) * rows) * C + c;
        for (int r = r0 + threadIdx.y; r < r1; r += 8) {
            const long long i = base + static_cast<long long>(r) * C;
            const float g = __ldcs(gy + i);
            acc += g * __ldcs(x + i);
            const float o = g * sv;
            gx[i] = rtf32 ? round_tf32(o) : o;
        }
    }
    sm[threadIdx.y][threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
        float t = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) t += sm[j][threadIdx.x];
        gs[(static_cast<long long>(blockIdx.y) * gridDim.z + b) * C + c] = t;
    }
}


// 16-byte-per-lane variants of the two kernels above for C % 32 == 0 (every layer of the model): a thread owns 4
// channels, TX lanes span TX*4 channels of one pixel row, 256/TX rows per block step; the row loop is unrolled so
// that 8-12 independent 16-byte loads are in flight per thread (a scalar kernel keeps too few bytes in flight to reach the HBM rate).
// four consecutive elements of the two-term bf16 expansion (hi plane at planes[e], lo plane at planes[total + e])
__device__ __forceinline__ void store_planes4(__nv_bfloat16* __restrict__ planes, long long total, long long e, const float4& t) {
    const __nv_bfloat16 h0 = __float2bfloat16_rn(t.x), h1 = __float2bfloat16_rn(t.y), h2 = __float2bfloat16_rn(t.z),
                        h3 = __float2bfloat16_rn(t.w);
    const __nv_bfloat16 l0 = __float2bfloat16_rn(t.x - __bfloat162float(h0)), l1 = __float2bfloat16_rn(t.y - __bfloat162float(h1)),
                        l2 = __float2bfloat16_rn(t.z - __bfloat162float(h2)), l3 = __float2bfloat16_rn(t.w - __bfloat162float(h3));
    uint2 ph, pl;
    ph.x = static_cast<uint32_t>(__bfloat16_as_ushort(h0)) | (static_cast<uint32_t>(__bfloat16_as_ushort(h1)) << 16);
    ph.y = static_cast<uint32_t>(__bfloat16_as_ushort(h2)) | (static_cast<uint32_t>(__bfloat16_as_ushort(h3)) << 16);
    pl.x = static_cast<uint32_t>(__bfloat16_as_ushort(l0)) | (static_cast<uint32_t>(__bfloat16_as_ushort(l1)) << 16);
    pl.y = static_cast<uint32_t>(__bfloat16_as_ushort(l2)) | (static_cast<uint32_t>(__bfloat16_as_ushort(l3)) << 16);
    *reinterpret_cast<uint2*>(planes + e) = ph;
    *reinterpret_cast<uint2*>(planes + total + e) = pl;
}

__device__ __forceinline__ float4 f4_zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void f4_add(float4& a, const float4& b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
__device__ __forceinline__ float4 f4_round(float4 v) {
    return make_float4(round_tf32(v.x), round_tf32(v.y), round_tf32(v.z), round_tf32(v.w));
}
__device__ __forceinline__ void f4_store(float* p, const float4& v) { *reinterpret_cast<float4*>(p) = v; }

template <int TX>
__global__ void __launch_bounds__(256) tail_bwd_vec_kernel(const float* __restrict__ gy, const float* __restrict__ y,
                                                           const float* __restrict__ acc, const float* __restrict__ d,
                                                           float* __restrict__ gt, float* __restrict__ gacc,
                                                           float* __restrict__ gb, float* __restrict__ gd, int rows, int C,
                                                           int rows_per_block, float slope, float gain, int rtf32,
                                                           __nv_bfloat16* __restrict__ gt_planes,
                                                           __nv_bfloat16* __restrict__ gacc_planes, long long total) {
    constexpr int TY = 256 / TX;
    __shared__ float4 sm[2][TY][TX];
    const int tx = threadIdx.x % TX, ty = threadIdx.x / TX;
    const int c = (blockIdx.x * TX + tx) * 4;          // first of this thread's 4 channels (C % (4*TX) == 0)
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * rows_per_block;
    const int r1 = min(rows, r0 + rows_per_block);
    float4 sb = f4_zero(), sd = f4_zero();
    const float4 dv = d ? *reinterpret_cast<const float4*>(d + static_cast<long long>(b) * C + c) : make_float4(1.f, 1.f, 1.f, 1.f);
    const long long base = (static_cast<long long>(b) * rows) * C + c;
    const bool has_acc = gd != nullptr;
#pragma unroll 4
    for (int r = r0 + ty; r < r1; r += TY) {
        const long long i = base + static_cast<long long>(r) * C;
        const float4 g0 = __ldcs(reinterpret_cast<const float4*>(gy + i));
        const float4 yv = __ldcs(reinterpret_cast<const float4*>(y + i));
        float4 g = make_float4(g0.x * gain * (yv.x > 0.f ? 1.f : slope), g0.y * gain * (yv.y > 0.f ? 1.f : slope),
                               g0.z * gain * (yv.z > 0.f ? 1.f : slope), g0.w * gain * (yv.w > 0.f ? 1.f : slope));
        f4_add(sb, g);
        if (has_acc) {
            const float4 a = __ldcs(reinterpret_cast<const float4*>(acc + i));
            sd.x += g.x * a.x; sd.y += g.y * a.y; sd.z += g.z * a.z; sd.w += g.w * a.w;
        }
        float4 ga = make_float4(g.x * dv.x, g.y * dv.y, g.z * dv.z, g.w * dv.w);
        if (rtf32) { g = f4_round(g); ga = f4_round(ga); }
        if (gt) *reinterpret_cast<float4*>(gt + i) = g;
        if (gacc) *reinterpret_cast<float4*>(gacc + i) = ga;
        if (gt_planes) store_planes4(gt_planes, total, i, g);          // bf16x3 operands of the consuming dgrad / wgrad
        if (gacc_planes) store_planes4(gacc_planes, total, i, ga);
    }
    sm[0][ty][tx] = sb;
    sm[1][ty][tx] = sd;
    __syncthreads();
    if (ty < 2) {
        float4 t = f4_zero();
#pragma unroll
        for (int j = 0; j < TY; ++j) f4_add(t, sm[ty][j][tx]);
        if (ty == 0) { if (gb) f4_store(gb + (static_cast<long long>(b) * gridDim.y + blockIdx.y) * C + c, t); }
        else if (gd) f4_store(gd + (static_cast<long long>(blockIdx.y) * gridDim.z + b) * C + c, t);
    }
}

template <int TX>
__global__ void __launch_bounds__(256) scale_bwd_vec_kernel(const float* __restrict__ gy, const float* __restrict__ x,
                                                            const float* __restrict__ s, float* __restrict__ gx,
                                                            float* __restrict__ gs, int rows, int C, int rows_per_block,
                                                            int rtf32) {
    constexpr int TY = 256 / TX;
    __shared__ float4 sm[TY][TX];
    const int tx = threadIdx.x % TX, ty = threadIdx.x / TX;
    const int c = (blockIdx.x * TX + tx) * 4;
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * rows_per_block;
    const int r1 = min(rows, r0 + rows_per_block);
    float4 a = f4_zero();
    const float4 sv = *reinterpret_cast<const float4*>(s + static_cast<long long>(b) * C + c);
    const long long base = (static_cast<long long>(b) * rows) * C + c;
#pragma unroll 4
    for (int r = r0 + ty; r < r1; r += TY) {
        const long long i = base + static_cast<long long>(r) * C;
        const float4 g = __ldcs(reinterpret_cast<const float4*>(gy + i));
        const float4 xv = __ldcs(reinterpret_cast<const float4*>(x + i));
        a.x += g.x * xv.x; a.y += g.y * xv.y; a.z += g.z * xv.z; a.w += g.w * xv.w;
        float4 o = make_float4(g.x * sv.x, g.y * sv.y, g.z * sv.z, g.w * sv.w);
        if (rtf32) o = f4_round(o);
        *reinterpret_cast<float4*>(gx + i) = o;
    }
    sm[ty][tx] = a;
    __syncthreads();
    if (ty == 0) {
        float4 t = f4_zero();
#pragma unroll
        for (int j = 0; j < TY; ++j) f4_add(t, sm[j][tx]);
        f4_store(gs + (static_cast<long long>(blockIdx.y) * gridDim.z + b) * C + c, t);
    }
}


// Second-order pass of the two kernels above (path-length regulariser: the derivative of a first-order backward that was
// recorded with create_graph).  The first-order map is, with m = gain*(y>0 ? 1 : slope) (m = 1 when y is null: the
// modulation variant), per (b, pixel, c):   gacc = gy*m*d[b,c]      gd[b,c] = sum_pixels gy*m*acc
// and given the upstream pair (gg = dL/dgacc, ggd = dL/dgd) this writes, in ONE pass over (gg, gy, y, acc):
//   ggy = m*(gg*d + ggd*acc)   (dL/dgy)      gx2 = gy*m*ggd   (dL/dacc)      gdd[b,c] += sum gg*gy*m   (dL/dd)
// instead of the closed-set composition (act_bwd, chan_scale x3, spatial_dot, and autograd's gradient-sum adds).
__global__ void __launch_bounds__(256) tail_bwd2_kernel(const float* __restrict__ gg, const float* __restrict__ ggd,
                                                        const float* __restrict__ gy, const float* __restrict__ y,
                                                        const float* __restrict__ acc, const float* __restrict__ d,
                                                        float* __restrict__ ggy, float* __restrict__ gx2,
                                                        float* __restrict__ gdd, int rows, int C, int rows_per_block,
                                                        float slope, float gain) {
    __shared__ float sm[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * rows_per_block;
    const int r1 = min(rows, r0 + rows_per_block);
    float sd = 0.f;
    if (c < C) {
        const float dv = d ? d[static_cast<long long>(b) * C + c] : 1.f;
        const float qv = ggd ? ggd[static_cast<long long>(b) * C + c] : 0.f;
        const long long base = (static_cast<long long>(b) * rows) * C + c;
        for (int r = r0 + threadIdx.y; r < r1; r += 8) {
            const long long i = base + static_cast<long long>(r) * C;
            const float m = y ? gain * (__ldcs(y + i) > 0.f ? 1.f : slope) : 1.f;
            const float gm = __ldcs(gy + i) * m;
            float u = 0.f;
            if (gg) { const float G = __ldcs(gg + i); u = G * dv; sd += G * gm; }
            if (ggd) { u += qv * __ldcs(acc + i); if (gx2) gx2[i] = gm * qv; }
            if (ggy) ggy[i] = m * u;
        }
    }
    sm[threadIdx.y][threadIdx.x] = sd;
    __syncthreads();
    if (threadIdx.y == 0 && c < C && gdd && gg) {
        float t = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) t += sm[j][threadIdx.x];
        gdd[(static_cast<long long>(blockIdx.y) * gridDim.z + b) * C + c] = t;
    }
}

template <int TX>
__global__ void __launch_bounds__(256) tail_bwd2_vec_kernel(const float* __restrict__ gg, const float* __restrict__ ggd,
                                                            const float* __restrict__ gy, const float* __restrict__ y,
                                                            const float* __restrict__ acc, const float* __restrict__ d,
                                                            float* __restrict__ ggy, float* __restrict__ gx2,
                                                            float* __restrict__ gdd, int rows, int C, int rows_per_block,
                                                            float slope, float gain, __nv_bfloat16* __restrict__ ggy_planes,
                                                            long long total) {
    constexpr int TY = 256 / TX;
    __shared__ float4 sm[TY][TX];
    const int tx = threadIdx.x % TX, ty = threadIdx.x / TX;
    const int c = (blockIdx.x * TX + tx) * 4;
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * rows_per_block;
    const int r1 = min(rows, r0 + rows_per_block);
    float4 sd = f4_zero();
    const float4 dv = d ? *reinterpret_cast<const float4*>(d + static_cast<long long>(b) * C + c) : make_float4(1.f, 1.f, 1.f, 1.f);
    const float4 qv = ggd ? *reinterpret_cast<const float4*>(ggd + static_cast<long long>(b) * C + c) : f4_zero();
    const long long base = (static_cast<long long>(b) * rows) * C + c;
    const float neg = gain * slope;
#pragma unroll 4
    for (int r = r0 + ty; r < r1; r += TY) {
        const long long i = base + static_cast<long long>(r) * C;
        const float4 g0 = __ldcs(reinterpret_cast<const float4*>(gy + i));
        float4 m = make_float4(1.f, 1.f, 1.f, 1.f);
        if (y) {
            const float4 yv = __ldcs(reinterpret_cast<const float4*>(y + i));
            m = make_float4(yv.x > 0.f ? gain : neg, yv.y > 0.f ? gain : neg, yv.z > 0.f ? gain : neg, yv.w > 0.f ? gain : neg);
        }
        const float4 gm = make_float4(g0.x * m.x, g0.y * m.y, g0.z * m.z, g0.w * m.w);
        float4 u = f4_zero();
        if (gg) {
            const float4 G = __ldcs(reinterpret_cast<const float4*>(gg + i));
            u = make_float4(G.x * dv.x, G.y * dv.y, G.z * dv.z, G.w * dv.w);
            sd.x += G.x * gm.x; sd.y += G.y * gm.y; sd.z += G.z * gm.z; sd.w += G.w * gm.w;
        }
        if (ggd) {
            const float4 a = __ldcs(reinterpret_cast<const float4*>(acc + i));
            u.x += qv.x * a.x; u.y += qv.y * a.y; u.z += qv.z * a.z; u.w += qv.w * a.w;
            if (gx2) *reinterpret_cast<float4*>(gx2 + i) = make_float4(gm.x * qv.x, gm.y * qv.y, gm.z * qv.z, gm.w * qv.w);
        }
        const float4 o = make_float4(m.x * u.x, m.y * u.y, m.z * u.z, m.w * u.w);
        if (ggy) *reinterpret_cast<float4*>(ggy + i) = o;
        if (ggy_planes) store_planes4(ggy_planes, total, i, o);
    }
    sm[ty][tx] = sd;
    __syncthreads();
    if (ty == 0 && gdd && gg) {
        float4 t = f4_zero();
#pragma unroll
        for (int j = 0; j < TY; ++j) f4_add(t, sm[j][tx]);
        f4_store(gdd + (static_cast<long long>(blockIdx.y) * gridDim.z + b) * C + c, t);
    }
}

// ------------------------------------------------------------------------------------------------ chan_scale
template <bool VEC>
__global__ void __launch_bounds__(256) chan_scale_kernel(const float* __restrict__ x, const float* __restrict__ s,
                                                         float* __restrict__ y, long long total, int P, int C,
                                                         int rtf32) {
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    if (VEC) {
        const long long nvec = total >> 2;
        const int c4n = C >> 2;
        for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec; v += stride) {
            const int c = static_cast<int>(v % c4n) << 2;
            const long long b = (v / c4n) / P;
            float4 t = __ldcs(reinterpret_cast<const float4*>(x) + v);
            const float4 sc = *reinterpret_cast<const float4*>(s + b * C + c);
            t.x *= sc.x; t.y *= sc.y; t.z *= sc.z; t.w *= sc.w;
            if (rtf32) { t.x = round_tf32(t.x); t.y = round_tf32(t.y); t.z = round_tf32(t.z); t.w = round_tf32(t.w); }
            reinterpret_cast<float4*>(y)[v] = t;
        }
    } else {
        for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
            float t = x[i] * s[((i / C) / P) * C + (i % C)];
            y[i] = rtf32 ? round_tf32(t) : t;
        }
    }
}


// ------------------------------------------------------------------------------------------------ split (bf16x3 operands)
// planes[0][e] = bf16_rn(v), planes[1][e] = bf16_rn(v - planes[0][e]) with v = x[e] * (s ? s[b,c] : 1): the two-term bf16
// expansion (16 significant bits) the compensated tensor-core contraction reads (conv_tc.cu / conv_wgrad_tc.cu, X3 mode).
// One pass: 4 B in, 2 x 2 B out per element; with s it also IS the modulation pass (no fp32 copy of the modulated input).
__global__ void __launch_bounds__(256) split_bf16_kernel(const float* __restrict__ x, const float* __restrict__ s,
                                                         __nv_bfloat16* __restrict__ planes, long long total, int P, int C) {
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    const long long nvec = total >> 2;
    const int c4n = C >> 2;
    __nv_bfloat16* hi = planes;
    __nv_bfloat16* lo = planes + total;
    for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec; v += stride) {
        float4 t = __ldcs(reinterpret_cast<const float4*>(x) + v);
        if (s) {
            const int c = static_cast<int>(v % c4n) << 2;
            const long long b = (v / c4n) / P;
            const float4 sc = *reinterpret_cast<const float4*>(s + b * C + c);
            t.x *= sc.x; t.y *= sc.y; t.z *= sc.z; t.w *= sc.w;
        }
        const __nv_bfloat16 h0 = __float2bfloat16_rn(t.x), h1 = __float2bfloat16_rn(t.y), h2 = __float2bfloat16_rn(t.z),
                            h3 = __float2bfloat16_rn(t.w);
        const __nv_bfloat16 l0 = __float2bfloat16_rn(t.x - __bfloat162float(h0)), l1 = __float2bfloat16_rn(t.y - __bfloat162float(h1)),
                            l2 = __float2bfloat16_rn(t.z - __bfloat162float(h2)), l3 = __float2bfloat16_rn(t.w - __bfloat162float(h3));
        uint2 ph, pl;
        ph.x = static_cast<uint32_t>(__bfloat16_as_ushort(h0)) | (static_cast<uint32_t>(__bfloat16_as_ushort(h1)) << 16);
        ph.y = static_cast<uint32_t>(__bfloat16_as_ushort(h2)) | (static_cast<uint32_t>(__bfloat16_as_ushort(h3)) << 16);
        pl.x = static_cast<uint32_t>(__bfloat16_as_ushort(l0)) | (static_cast<uint32_t>(__bfloat16_as_ushort(l1)) << 16);
        pl.y = static_cast<uint32_t>(__bfloat16_as_ushort(l2)) | (static_cast<uint32_t>(__bfloat16_as_ushort(l3)) << 16);
        reinterpret_cast<uint2*>(hi)[v] = ph;
        reinterpret_cast<uint2*>(lo)[v] = pl;
    }
}

template <bool VEC>
__global__ void __launch_bounds__(256) axpby_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                    float* __restrict__ y, long long n, float alpha, float beta,
                                                    int rtf32) {
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    if (VEC) {
        const long long nvec = n >> 2;
        for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec; v += stride) {
            float4 t = __ldcs(reinterpret_cast<const float4*>(a) + v);
            t.x *= alpha; t.y *= alpha; t.z *= alpha; t.w *= alpha;
            if (b) {
                const float4 u = __ldcs(reinterpret_cast<const float4*>(b) + v);
                t.x += beta * u.x; t.y += beta * u.y; t.z += beta * u.z; t.w += beta * u.w;
            }
            if (rtf32) { t.x = round_tf32(t.x); t.y = round_tf32(t.y); t.z = round_tf32(t.z); t.w = round_tf32(t.w); }
            reinterpret_cast<float4*>(y)[v] = t;
        }
    } else {
        for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
        {
            const float t = alpha * a[i] + (b ? beta * b[i] : 0.f);
            y[i] = rtf32 ? round_tf32(t) : t;
        }
    }
}

// ------------------------------------------------------------------------------------------------ demod
// One warp per (b,o): lanes stride over i, shuffle-reduce sum_i s[b,i]^2 q[o,i].
__global__ void __launch_bounds__(256) demod_kernel(const float* __restrict__ s, const float* __restrict__ q,
                                                    float* __restrict__ d, int B, int Ci, int Co, float eps) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= B * Co) return;
    const int b = warp / Co, o = warp % Co;
    const float* sr = s + static_cast<long long>(b) * Ci;
    const float* qr = q + static_cast<long long>(o) * Ci;
    float acc = 0.f;
    for (int i = lane; i < Ci; i += 32) {
        const float sv = sr[i];
        acc += sv * sv * qr[i];
    }
    acc = warp_sum(acc);
    if (lane == 0) d[warp] = rsqrtf(acc + eps);
}

// ------------------------------------------------------------------------------------------------ ToRGB
// y[b,p,0..2] = sum_i x[b,p,i]*ws[b,k,i].  One warp per pixel group: each lane strides the channel dim with float4,
// three shuffle reductions per pixel.  x is read exactly once (HBM-bound: C*4 bytes/pixel in, 12 out).
__global__ void __launch_bounds__(256) torgb_fwd_kernel(const float* __restrict__ x, const float* __restrict__ ws,
                                                        float* __restrict__ y, int B, int P, int C) {
    extern __shared__ float sw[];  // 3*C weights of this sample
    const int b = blockIdx.y;
    const float* wsb = ws + static_cast<long long>(b) * 3 * C;
    for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) sw[i] = wsb[i];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
    for (int p = blockIdx.x * nwarp + warp; p < P; p += gridDim.x * nwarp) {
        const float* xr = x + (static_cast<long long>(b) * P + p) * C;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        if ((C & 3) == 0) {
            for (int i = lane * 4; i < C; i += 128) {
                const float4 v = __ldcs(reinterpret_cast<const float4*>(xr + i));
                a0 += v.x * sw[i] + v.y * sw[i + 1] + v.z * sw[i + 2] + v.w * sw[i + 3];
                a1 += v.x * sw[C + i] + v.y * sw[C + i + 1] + v.z * sw[C + i + 2] + v.w * sw[C + i + 3];
                a2 += v.x * sw[2 * C + i] + v.y * sw[2 * C + i + 1] + v.z * sw[2 * C + i + 2] + v.w * sw[2 * C + i + 3];
            }
        } else {
            for (int i = lane; i < C; i += 32) {
                const float v = xr[i];
                a0 += v * sw[i]; a1 += v * sw[C + i]; a2 += v * sw[2 * C + i];
            }
        }
        a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2);
        if (lane == 0) {
            float* yr = y + (static_cast<long long>(b) * P + p) * 3;
            yr[0] = a0; yr[1] = a1; yr[2] = a2;
        }
    }
}

// gx[b,p,i] = sum_k gy[b,p,k]*ws[b,k,i]
__global__ void __launch_bounds__(256) torgb_bwd_x_kernel(const float* __restrict__ gy, const float* __restrict__ ws,
                                                          float* __restrict__ gx, int B, int P, int C) {
    extern __shared__ float sw[];
    const int b = blockIdx.y;
    const float* wsb = ws + static_cast<long long>(b) * 3 * C;
    for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) sw[i] = wsb[i];
    __syncthreads();
    const long long total = static_cast<long long>(P) * C;
    for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int p = static_cast<int>(e / C), i = static_cast<int>(e % C);
        const float* g = gy + (static_cast<long long>(b) * P + p) * 3;
        gx[static_cast<long long>(b) * total + e] = g[0] * sw[i] + g[1] * sw[C + i] + g[2] * sw[2 * C + i];
    }
}

// gws[b,k,i] = sum_p gy[b,p,k]*x[b,p,i]   (block: 32 channels x 8 row lanes, partial sums into slots)
__global__ void __launch_bounds__(256) torgb_bwd_w_kernel(const float* __restrict__ gy, const float* __restrict__ x,
                                                          float* __restrict__ gws, int P, int C, int rows_per_block) {
    __shared__ float sm[3][8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * rows_per_block;
    const int r1 = min(P, r0 + rows_per_block);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    if (c < C) {
        for (int p = r0 + threadIdx.y; p < r1; p += 8) {
            const long long row = static_cast<long long>(b) * P + p;
            const float v = x[row * C + c];
            const float* g = gy + row * 3;
            a0 += v * g[0]; a1 += v * g[1]; a2 += v * g[2];
        }
    }
    sm[0][threadIdx.y][threadIdx.x] = a0;
    sm[1][threadIdx.y][threadIdx.x] = a1;
    sm[2][threadIdx.y][threadIdx.x] = a2;
    __syncthreads();
    if (threadIdx.y < 3 && c < C) {
        float t = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) t += sm[threadIdx.y][j][threadIdx.x];
        gws[((static_cast<long long>(blockIdx.y) * gridDim.z + b) * 3 + threadIdx.y) * C + c] = t;
    }
}


// 16-byte variants of the three ToRGB kernels for C % 32 == 0 (same lane layout as tail_bwd_vec_kernel: a thread owns 4
// channels, TX lanes span a pixel's channel chunk, 256/TX pixels per block step, rows unrolled for loads in flight).
// The scalar versions kept one 16-byte load in flight per lane and spent 15 shuffles per pixel in the forward.
template <int TX>
__global__ void __launch_bounds__(256) torgb_fwd_vec_kernel(const float* __restrict__ x, const float* __restrict__ ws,
                                                            float* __restrict__ y, int P, int C, int rows_per_block) {
    constexpr int TY = 256 / TX;
    const int tx = threadIdx.x % TX, ty = threadIdx.x / TX;
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * rows_per_block;
    const int r1 = min(P, r0 + rows_per_block);
    const float* wsb = ws + static_cast<long long>(b) * 3 * C;
    const int nchunk = C / (4 * TX);          // channel chunks a lane walks (C = 128: 1 with TX = 32)
    // the first chunk's weights stay in registers (the only chunk for C <= 128, the HBM-heavy resolutions)
    const float4 w0f = *reinterpret_cast<const float4*>(wsb + tx * 4);
    const float4 w1f = *reinterpret_cast<const float4*>(wsb + C + tx * 4);
    const float4 w2f = *reinterpret_cast<const float4*>(wsb + 2 * C + tx * 4);
#pragma unroll 4
    for (int pb = r0; pb < r1; pb += TY) {     // uniform trip count per warp: the shuffles below need every lane
        const int p = pb + ty;
        const bool live = p < r1;
        const float* xr = x + (static_cast<long long>(b) * P + (live ? p : r0)) * C;
        const float4 v0 = __ldcs(reinterpret_cast<const float4*>(xr + tx * 4));
        float a0 = v0.x * w0f.x + v0.y * w0f.y + v0.z * w0f.z + v0.w * w0f.w;
        float a1 = v0.x * w1f.x + v0.y * w1f.y + v0.z * w1f.z + v0.w * w1f.w;
        float a2 = v0.x * w2f.x + v0.y * w2f.y + v0.z * w2f.z + v0.w * w2f.w;
        for (int ch = 1; ch < nchunk; ++ch) {
            const int c = (ch * TX + tx) * 4;
            const float4 v = __ldcs(reinterpret_cast<const float4*>(xr + c));
            const float4 w0 = *reinterpret_cast<const float4*>(wsb + c);
            const float4 w1 = *reinterpret_cast<const float4*>(wsb + C + c);
            const float4 w2 = *reinterpret_cast<const float4*>(wsb + 2 * C + c);
            a0 += v.x * w0.x + v.y * w0.y + v.z * w0.z + v.w * w0.w;
            a1 += v.x * w1.x + v.y * w1.y + v.z * w1.z + v.w * w1.w;
            a2 += v.x * w2.x + v.y * w2.y + v.z * w2.z + v.w * w2.w;
        }
#pragma unroll
        for (int o = TX / 2; o > 0; o >>= 1) {
            a0 += __shfl_xor_sync(0xffffffffu, a0, o);
            a1 += __shfl_xor_sync(0xffffffffu, a1, o);
            a2 += __shfl_xor_sync(0xffffffffu, a2, o);
        }
        if (tx == 0 && live) {
            float* yr = y + (static_cast<long long>(b) * P + p) * 3;
            yr[0] = a0; yr[1] = a1; yr[2] = a2;
        }
    }
}

__global__ void __launch_bounds__(256) torgb_bwd_x_vec_kernel(const float* __restrict__ gy, const float* __restrict__ ws,
                                                              float* __restrict__ gx, int P, int C) {
    const int b = blockIdx.y;
    const float* wsb = ws + static_cast<long long>(b) * 3 * C;
    const int cv = C >> 2;
    const long long total = static_cast<long long>(P) * cv;
    for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int p = static_cast<int>(e / cv), c = static_cast<int>(e % cv) * 4;
        const float* g = gy + (static_cast<long long>(b) * P + p) * 3;
        const float g0 = g[0], g1 = g[1], g2 = g[2];
        const float4 w0 = *reinterpret_cast<const float4*>(wsb + c);
        const float4 w1 = *reinterpret_cast<const float4*>(wsb + C + c);
        const float4 w2 = *reinterpret_cast<const float4*>(wsb + 2 * C + c);
        float4 o;
        o.x = g0 * w0.x + g1 * w1.x + g2 * w2.x; o.y = g0 * w0.y + g1 * w1.y + g2 * w2.y;
        o.z = g0 * w0.z + g1 * w1.z + g2 * w2.z; o.w = g0 * w0.w + g1 * w1.w + g2 * w2.w;
        reinterpret_cast<float4*>(gx + static_cast<long long>(b) * P * C)[e] = o;
    }
}

template <int TX>
__global__ void __launch_bounds__(256) torgb_bwd_w_vec_kernel(const float* __restrict__ gy, const float* __restrict__ x,
                                                              float* __restrict__ gws, int P, int C, int rows_per_block) {
    constexpr int TY = 256 / TX;
    __shared__ float4 sm[3][TY][TX];
    const int tx = threadIdx.x % TX, ty = threadIdx.x / TX;
    const int c = (blockIdx.x * TX + tx) * 4;
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * rows_per_block;
    const int r1 = min(P, r0 + rows_per_block);
    float4 a0 = f4_zero(), a1 = f4_zero(), a2 = f4_zero();
#pragma unroll 4
    for (int p = r0 + ty; p < r1; p += TY) {
        const long long row = static_cast<long long>(b) * P + p;
        const float4 v = __ldcs(reinterpret_cast<const float4*>(x + row * C + c));
        const float* g = gy + row * 3;
        const float g0 = g[0], g1 = g[1], g2 = g[2];
        a0.x += v.x * g0; a0.y += v.y * g0; a0.z += v.z * g0; a0.w += v.w * g0;
        a1.x += v.x * g1; a1.y += v.y * g1; a1.z += v.z * g1; a1.w += v.w * g1;
        a2.x += v.x * g2; a2.y += v.y * g2; a2.z += v.z * g2; a2.w += v.w * g2;
    }
    sm[0][ty][tx] = a0; sm[1][ty][tx] = a1; sm[2][ty][tx] = a2;
    __syncthreads();
    if (ty < 3) {
        float4 t = f4_zero();
#pragma unroll
        for (int j = 0; j < TY; ++j) f4_add(t, sm[ty][j][tx]);
        f4_store(gws + ((static_cast<long long>(blockIdx.y) * gridDim.z + b) * 3 + ty) * C + c, t);
    }
}

// ------------------------------------------------------------------------------------------------ cond pyramid
// y[b,yo,xo,c] = mean of x[b, s*yo + s/2 - {1,0}, s*xo + s/2 - {1,0}, c]   (s >= 2, power of two); adjoint scatters.
__global__ void __launch_bounds__(256) cond_down_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H,
                                                        int W, int C, int s) {
    const int Ho = H / s, Wo = W / s;
    const long long total = static_cast<long long>(B) * Ho * Wo * C;
    for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c = static_cast<int>(e % C);
        long long r = e / C;
        const int xo = static_cast<int>(r % Wo); r /= Wo;
        const int yo = static_cast<int>(r % Ho);
        const int b = static_cast<int>(r / Ho);
        const int y0 = s * yo + s / 2 - 1, x0 = s * xo + s / 2 - 1;
        const float* base = x + ((static_cast<long long>(b) * H + y0) * W + x0) * C + c;
        const long long rs = static_cast<long long>(W) * C;
        y[e] = 0.25f * (base[0] + base[C] + base[rs] + base[rs + C]);
    }
}

__global__ void __launch_bounds__(256) cond_down_adj_kernel(float* __restrict__ gx, const float* __restrict__ gy, int B,
                                                            int H, int W, int C, int s) {
    const int Ho = H / s, Wo = W / s;
    const long long total = static_cast<long long>(B) * H * W * C;
    for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c = static_cast<int>(e % C);
        long long r = e / C;
        const int xi = static_cast<int>(r % W); r /= W;
        const int yi = static_cast<int>(r % H);
        const int b = static_cast<int>(r / H);
        const int ry = yi % s, rx = xi % s;
        const bool hit = (ry == s / 2 - 1 || ry == s / 2) && (rx == s / 2 - 1 || rx == s / 2);
        gx[e] = hit ? 0.25f * gy[((static_cast<long long>(b) * Ho + yi / s) * Wo + xi / s) * C + c] : 0.f;
    }
}

static inline int grid_for(long long work_items, int per_block) {
    long long blocks = (work_items + per_block - 1) / per_block;
    const long long cap = static_cast<long long>(kNumSMs) * 16;  // multiple of the SM count; grid-stride beyond
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return static_cast<int>(blocks);
}

}  // namespace gifb200

using namespace gifb200;

namespace gifb200 {

__global__ void __launch_bounds__(256) slots_reduce_kernel(const float* __restrict__ part, float* __restrict__ out, int slots,
                                                           long long n) {
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        float t = 0.f;
        for (int k = 0; k < slots; ++k) t += part[k * n + i];
        out[i] = t;
    }
}

int slots_take(Slots& s, float*& out, int count, long long n, cudaStream_t st) {
    // keep freed slot buffers in the stream-ordered pool instead of returning them to the driver at every synchronisation
    static std::once_flag keep;
    std::call_once(keep, [] {
        int dev = 0;
        cudaMemPool_t pool;
        if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
            uint64_t keep_all = UINT64_MAX;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep_all);
        }
    });
    cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&s.part), sizeof(float) * static_cast<size_t>(count) * n, st);
    if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "partial-sum buffer", cudaGetErrorString(e));
    s.out = out;
    s.count = count;
    s.n = n;
    out = s.part;
    return GIFB200_OK;
}

int slots_reduce(Slots& s, cudaStream_t st) {
    int blocks = cdiv(s.n, 256);
    if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
    slots_reduce_kernel<<<blocks, 256, 0, st>>>(s.part, s.out, s.count, s.n);
    const int rc = check_launch("slots_reduce_kernel");
    cudaError_t e = cudaFreeAsync(s.part, st);
    s.part = nullptr;
    if (rc != GIFB200_OK) return rc;
    return e == cudaSuccess ? GIFB200_OK : fail(GIFB200_E_CUDA, "partial-sum buffer", cudaGetErrorString(e));
}

}  // namespace gifb200

extern "C" {

int gifb200_version(void) { return 100; }
const char* gifb200_last_error(void) { return g_err; }
long long gifb200_launch_count(void) { return g_launches; }

int gifb200_bias_act(const float* x, const float* rowscale, const float* add, const float* bias, float* y, int B, int P,
                     int C, float slope, float gain, int rtf32, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && P >= 0 && C > 0, GIFB200_E_SHAPE, "bias_act: bad shape");
    const long long total = static_cast<long long>(B) * P * C;
    if (total == 0) return GIFB200_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool vec = (C % 4 == 0) && aligned16(x) && aligned16(y) && (!add || aligned16(add)) &&
                     (!bias || aligned16(bias)) && (!rowscale || aligned16(rowscale));
    if (vec)
        bias_act_kernel<true><<<grid_for(total / 4, 256), 256, 0, st>>>(x, rowscale, add, bias, y, total, P, C, slope, gain, rtf32);
    else
        bias_act_kernel<false><<<grid_for(total, 256), 256, 0, st>>>(x, rowscale, add, bias, y, total, P, C, slope, gain, rtf32);
    GIFB200_LAUNCH_CHECK("bias_act_kernel");
    return GIFB200_OK;
}

int gifb200_act_bwd(const float* gy, const float* y, float* gx, long long n, float slope, float gain, int rtf32,
                    gifb200_stream_t stream) {
    if (n <= 0) return GIFB200_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n % 4 == 0 && aligned16(gy) && aligned16(y) && aligned16(gx))
        act_bwd_kernel<true><<<grid_for(n / 4, 256), 256, 0, st>>>(gy, y, gx, n, slope, gain, rtf32);
    else
        act_bwd_kernel<false><<<grid_for(n, 256), 256, 0, st>>>(gy, y, gx, n, slope, gain, rtf32);
    GIFB200_LAUNCH_CHECK("act_bwd_kernel");
    return GIFB200_OK;
}

static int rows_split(int rows, int cblocks, int G, int* rows_per_block) {
    // aim for ~4 blocks per SM in total
    long long want = (static_cast<long long>(kNumSMs) * 4 + static_cast<long long>(cblocks) * G - 1) /
                     (static_cast<long long>(cblocks) * G);
    if (want < 1) want = 1;
    int rpb = static_cast<int>((rows + want - 1) / want);
    if (rpb < 64) rpb = 64;
    *rows_per_block = rpb;
    return (rows + rpb - 1) / rpb;
}

// lanes along the channel dimension for the 16-byte kernels: the largest of 32/16/8 such that C % (4*lanes) == 0
static int vec_lanes(int C) { return (C % 128 == 0) ? 32 : (C % 64 == 0) ? 16 : 8; }

static int rows_split_vec(int rows, int cblocks, int G, int ty, int* rows_per_block) {
    // ~8 blocks of 256 threads per SM in total; at least 4 unrolled row steps per block
    long long want = (static_cast<long long>(kNumSMs) * 8 + static_cast<long long>(cblocks) * G - 1) /
                     (static_cast<long long>(cblocks) * G);
    if (want < 1) want = 1;
    int rpb = static_cast<int>((rows + want - 1) / want);
    if (rpb < 4 * ty) rpb = 4 * ty;
    *rows_per_block = rpb;
    return (rows + rpb - 1) / rpb;
}

int gifb200_rows_sum(const float* x, float* out, int G, int rows, int C, gifb200_stream_t stream) {
    GIFB200_REQUIRE(G >= 0 && rows >= 0 && C > 0, GIFB200_E_SHAPE, "rows_sum: bad shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (G == 0) return GIFB200_OK;
    cudaError_t e = cudaMemsetAsync(out, 0, sizeof(float) * static_cast<size_t>(G) * C, st);
    if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "rows_sum memset", cudaGetErrorString(e));
    if (rows == 0) return GIFB200_OK;
    const int cb = cdiv(C, 32);
    int rpb;
    const int rb = rows_split(rows, cb, G, &rpb);
    GIFB200_REQUIRE(G <= 65535 && rb <= 65535, GIFB200_E_SHAPE, "rows_sum: grid too large");
    Slots sl;
    if (int rc = slots_take(sl, out, rb, static_cast<long long>(G) * C, st)) return rc;
    rows_sum_kernel<<<dim3(cb, rb, G), dim3(32, 8), 0, st>>>(x, out, rows, C, rpb);
    GIFB200_LAUNCH_CHECK("rows_sum_kernel");
    return slots_reduce(sl, st);
}

int gifb200_spatial_dot(const float* a, const float* b2, float* out, int B, int P, int C, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && P >= 0 && C > 0, GIFB200_E_SHAPE, "spatial_dot: bad shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (B == 0) return GIFB200_OK;
    cudaError_t e = cudaMemsetAsync(out, 0, sizeof(float) * static_cast<size_t>(B) * C, st);
    if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "spatial_dot memset", cudaGetErrorString(e));
    if (P == 0) return GIFB200_OK;
    const int cb = cdiv(C, 32);
    int rpb;
    const int rb = rows_split(P, cb, B, &rpb);
    GIFB200_REQUIRE(B <= 65535 && rb <= 65535, GIFB200_E_SHAPE, "spatial_dot: grid too large");
    Slots sl;
    if (int rc = slots_take(sl, out, rb, static_cast<long long>(B) * C, st)) return rc;
    spatial_dot_kernel<<<dim3(cb, rb, B), dim3(32, 8), 0, st>>>(a, b2, out, P, C, rpb);
    GIFB200_LAUNCH_CHECK("spatial_dot_kernel");
    return slots_reduce(sl, st);
}

// gb: one slot per (b, row chunk); gd: one per row chunk (either may be absent)
static int tail_slots(Slots& sb, Slots& sd, float*& gb, float*& gd, int B, int rb, int C, cudaStream_t st) {
    int rc = gb ? slots_take(sb, gb, B * rb, C, st) : GIFB200_OK;
    return rc == GIFB200_OK && gd ? slots_take(sd, gd, rb, static_cast<long long>(B) * C, st) : rc;
}

static int tail_reduce(Slots& sb, Slots& sd, cudaStream_t st) {
    int rc = sb.part ? slots_reduce(sb, st) : GIFB200_OK;
    return rc == GIFB200_OK && sd.part ? slots_reduce(sd, st) : rc;
}

static int tail_bwd_impl(const float* gy, const float* y, const float* acc, const float* d, float* gt, float* gacc,
                         float* gb, float* gd, int B, int P, int C, float slope, float gain, int rtf32, void* gt_planes,
                         void* gacc_planes, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && P >= 0 && C > 0, GIFB200_E_SHAPE, "tail_bwd: bad shape");
    GIFB200_REQUIRE(gt || gt_planes || gacc, GIFB200_E_SHAPE, "tail_bwd: gt, gt_planes or gacc is required");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (B == 0) return GIFB200_OK;
    if (gb) {
        cudaError_t e = cudaMemsetAsync(gb, 0, sizeof(float) * C, st);
        if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "tail_bwd memset", cudaGetErrorString(e));
    }
    if (gd) {
        cudaError_t e = cudaMemsetAsync(gd, 0, sizeof(float) * static_cast<size_t>(B) * C, st);
        if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "tail_bwd memset", cudaGetErrorString(e));
    }
    if (P == 0) return GIFB200_OK;
    const bool planes = gt_planes || gacc_planes;
    if (C % 32 == 0 && aligned16(gy) && aligned16(y) && (!gt || aligned16(gt)) && (!gd || aligned16(acc)) && (!gacc || aligned16(gacc)) &&
        (!d || aligned16(d)) && (!gt_planes || aligned16(gt_planes)) && (!gacc_planes || aligned16(gacc_planes))) {
        const int tx = vec_lanes(C);
        int rpb;
        const int cbv = C / (4 * tx);
        const int rb = rows_split_vec(P, cbv, B, 256 / tx, &rpb);
        GIFB200_REQUIRE(B <= 65535 && rb <= 65535, GIFB200_E_SHAPE, "tail_bwd: grid too large");
        const dim3 grid(cbv, rb, B);
        Slots sb, sd;
        if (int rc = tail_slots(sb, sd, gb, gd, B, rb, C, st)) return rc;
        __nv_bfloat16* p1 = static_cast<__nv_bfloat16*>(gt_planes);
        __nv_bfloat16* p2 = static_cast<__nv_bfloat16*>(gacc_planes);
        const long long total = static_cast<long long>(B) * P * C;
        if (tx == 32) tail_bwd_vec_kernel<32><<<grid, 256, 0, st>>>(gy, y, acc, d, gt, gacc, gb, gd, P, C, rpb, slope, gain, rtf32, p1, p2, total);
        else if (tx == 16) tail_bwd_vec_kernel<16><<<grid, 256, 0, st>>>(gy, y, acc, d, gt, gacc, gb, gd, P, C, rpb, slope, gain, rtf32, p1, p2, total);
        else tail_bwd_vec_kernel<8><<<grid, 256, 0, st>>>(gy, y, acc, d, gt, gacc, gb, gd, P, C, rpb, slope, gain, rtf32, p1, p2, total);
        GIFB200_LAUNCH_CHECK("tail_bwd_vec_kernel");
        return tail_reduce(sb, sd, st);
    }
    GIFB200_REQUIRE(!planes, GIFB200_E_ALIGN, "tail_bwd: the planes outputs need C % 32 == 0 and 16-byte aligned pointers");
    const int cb = cdiv(C, 32);
    int rpb;
    const int rb = rows_split(P, cb, B, &rpb);
    GIFB200_REQUIRE(B <= 65535 && rb <= 65535, GIFB200_E_SHAPE, "tail_bwd: grid too large");
    Slots sb, sd;
    if (int rc = tail_slots(sb, sd, gb, gd, B, rb, C, st)) return rc;
    tail_bwd_kernel<<<dim3(cb, rb, B), dim3(32, 8), 0, st>>>(gy, y, acc, d, gt, gacc, gb, gd, P, C, rpb, slope, gain, rtf32);
    GIFB200_LAUNCH_CHECK("tail_bwd_kernel");
    return tail_reduce(sb, sd, st);
}

int gifb200_tail_bwd(const float* gy, const float* y, const float* acc, const float* d, float* gt, float* gacc,
                     float* gb, float* gd, int B, int P, int C, float slope, float gain, int rtf32, gifb200_stream_t stream) {
    return tail_bwd_impl(gy, y, acc, d, gt, gacc, gb, gd, B, P, C, slope, gain, rtf32, nullptr, nullptr, stream);
}

int gifb200_tail_bwd_planes(const float* gy, const float* y, const float* acc, const float* d, float* gt, float* gacc,
                            float* gb, float* gd, int B, int P, int C, float slope, float gain, void* gt_planes,
                            void* gacc_planes, gifb200_stream_t stream) {
    return tail_bwd_impl(gy, y, acc, d, gt, gacc, gb, gd, B, P, C, slope, gain, 0, gt_planes, gacc_planes, stream);
}

int gifb200_scale_bwd(const float* gy, const float* x, const float* s, float* gx, float* gs, int B, int P, int C, int rtf32,
                      gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && P >= 0 && C > 0, GIFB200_E_SHAPE, "scale_bwd: bad shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (B == 0) return GIFB200_OK;
    cudaError_t e = cudaMemsetAsync(gs, 0, sizeof(float) * static_cast<size_t>(B) * C, st);
    if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "scale_bwd memset", cudaGetErrorString(e));
    if (P == 0) return GIFB200_OK;
    if (C % 32 == 0 && aligned16(gy) && aligned16(x) && aligned16(gx) && aligned16(s)) {
        const int tx = vec_lanes(C);
        int rpb;
        const int cbv = C / (4 * tx);
        const int rb = rows_split_vec(P, cbv, B, 256 / tx, &rpb);
        GIFB200_REQUIRE(B <= 65535 && rb <= 65535, GIFB200_E_SHAPE, "scale_bwd: grid too large");
        const dim3 grid(cbv, rb, B);
        Slots sl;
        if (int rc = slots_take(sl, gs, rb, static_cast<long long>(B) * C, st)) return rc;
        if (tx == 32) scale_bwd_vec_kernel<32><<<grid, 256, 0, st>>>(gy, x, s, gx, gs, P, C, rpb, rtf32);
        else if (tx == 16) scale_bwd_vec_kernel<16><<<grid, 256, 0, st>>>(gy, x, s, gx, gs, P, C, rpb, rtf32);
        else scale_bwd_vec_kernel<8><<<grid, 256, 0, st>>>(gy, x, s, gx, gs, P, C, rpb, rtf32);
        GIFB200_LAUNCH_CHECK("scale_bwd_vec_kernel");
        return slots_reduce(sl, st);
    }
    const int cb = cdiv(C, 32);
    int rpb;
    const int rb = rows_split(P, cb, B, &rpb);
    GIFB200_REQUIRE(B <= 65535 && rb <= 65535, GIFB200_E_SHAPE, "scale_bwd: grid too large");
    Slots sl;
    if (int rc = slots_take(sl, gs, rb, static_cast<long long>(B) * C, st)) return rc;
    scale_bwd_kernel<<<dim3(cb, rb, B), dim3(32, 8), 0, st>>>(gy, x, s, gx, gs, P, C, rpb, rtf32);
    GIFB200_LAUNCH_CHECK("scale_bwd_kernel");
    return slots_reduce(sl, st);
}

int gifb200_tail_bwd2(const float* gg, const float* ggd, const float* gy, const float* y, const float* acc, const float* d,
                      float* ggy, float* gx2, float* gdd, int B, int P, int C, float slope, float gain, void* ggy_planes,
                      gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && P >= 0 && C > 0, GIFB200_E_SHAPE, "tail_bwd2: bad shape");
    GIFB200_REQUIRE(gy && (gg || ggd), GIFB200_E_SHAPE, "tail_bwd2: gy and at least one upstream gradient are required");
    GIFB200_REQUIRE(!ggd || acc, GIFB200_E_SHAPE, "tail_bwd2: ggd needs acc");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (B == 0) return GIFB200_OK;
    if (gdd) {
        cudaError_t e = cudaMemsetAsync(gdd, 0, sizeof(float) * static_cast<size_t>(B) * C, st);
        if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "tail_bwd2 memset", cudaGetErrorString(e));
    }
    if (P == 0) return GIFB200_OK;
    if (C % 32 == 0 && aligned16(gy) && (!gg || aligned16(gg)) && (!ggd || (aligned16(ggd) && aligned16(acc))) && (!y || aligned16(y)) &&
        (!d || aligned16(d)) && (!ggy || aligned16(ggy)) && (!gx2 || aligned16(gx2)) && (!gdd || aligned16(gdd)) &&
        (!ggy_planes || aligned16(ggy_planes))) {
        const int tx = vec_lanes(C);
        int rpb;
        const int cbv = C / (4 * tx);
        const int rb = rows_split_vec(P, cbv, B, 256 / tx, &rpb);
        GIFB200_REQUIRE(B <= 65535 && rb <= 65535, GIFB200_E_SHAPE, "tail_bwd2: grid too large");
        const dim3 grid(cbv, rb, B);
        Slots sl;
        if (int rc = gdd && gg ? slots_take(sl, gdd, rb, static_cast<long long>(B) * C, st) : GIFB200_OK) return rc;
        __nv_bfloat16* pp = static_cast<__nv_bfloat16*>(ggy_planes);
        const long long total = static_cast<long long>(B) * P * C;
        if (tx == 32) tail_bwd2_vec_kernel<32><<<grid, 256, 0, st>>>(gg, ggd, gy, y, acc, d, ggy, gx2, gdd, P, C, rpb, slope, gain, pp, total);
        else if (tx == 16) tail_bwd2_vec_kernel<16><<<grid, 256, 0, st>>>(gg, ggd, gy, y, acc, d, ggy, gx2, gdd, P, C, rpb, slope, gain, pp, total);
        else tail_bwd2_vec_kernel<8><<<grid, 256, 0, st>>>(gg, ggd, gy, y, acc, d, ggy, gx2, gdd, P, C, rpb, slope, gain, pp, total);
        GIFB200_LAUNCH_CHECK("tail_bwd2_vec_kernel");
        return sl.part ? slots_reduce(sl, st) : GIFB200_OK;
    }
    GIFB200_REQUIRE(!ggy_planes, GIFB200_E_ALIGN, "tail_bwd2: the planes output needs C % 32 == 0 and 16-byte aligned pointers");
    const int cb = cdiv(C, 32);
    int rpb;
    const int rb = rows_split(P, cb, B, &rpb);
    GIFB200_REQUIRE(B <= 65535 && rb <= 65535, GIFB200_E_SHAPE, "tail_bwd2: grid too large");
    Slots sl;
    if (int rc = gdd && gg ? slots_take(sl, gdd, rb, static_cast<long long>(B) * C, st) : GIFB200_OK) return rc;
    tail_bwd2_kernel<<<dim3(cb, rb, B), dim3(32, 8), 0, st>>>(gg, ggd, gy, y, acc, d, ggy, gx2, gdd, P, C, rpb, slope, gain);
    GIFB200_LAUNCH_CHECK("tail_bwd2_kernel");
    return sl.part ? slots_reduce(sl, st) : GIFB200_OK;
}

int gifb200_chan_scale(const float* x, const float* s, float* y, int B, int P, int C, int rtf32,
                       gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && P >= 0 && C > 0, GIFB200_E_SHAPE, "chan_scale: bad shape");
    const long long total = static_cast<long long>(B) * P * C;
    if (total == 0) return GIFB200_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (C % 4 == 0 && aligned16(x) && aligned16(y) && aligned16(s))
        chan_scale_kernel<true><<<grid_for(total / 4, 256), 256, 0, st>>>(x, s, y, total, P, C, rtf32);
    else
        chan_scale_kernel<false><<<grid_for(total, 256), 256, 0, st>>>(x, s, y, total, P, C, rtf32);
    GIFB200_LAUNCH_CHECK("chan_scale_kernel");
    return GIFB200_OK;
}

int gifb200_split_bf16(const float* x, const float* s, void* planes, int B, int P, int C, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && P >= 0 && C > 0 && C % 4 == 0, GIFB200_E_SHAPE, "split_bf16: C must be a positive multiple of 4");
    const long long total = static_cast<long long>(B) * P * C;
    if (total == 0) return GIFB200_OK;
    GIFB200_REQUIRE(aligned16(x) && aligned16(planes) && (!s || aligned16(s)), GIFB200_E_ALIGN, "split_bf16: pointers must be 16-byte aligned");
    split_bf16_kernel<<<grid_for(total / 4, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, s, static_cast<__nv_bfloat16*>(planes), total, P, C);
    GIFB200_LAUNCH_CHECK("split_bf16_kernel");
    return GIFB200_OK;
}

int gifb200_axpby(const float* a, const float* b, float* y, long long n, float alpha, float beta, int rtf32,
                  gifb200_stream_t stream) {
    if (n <= 0) return GIFB200_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n % 4 == 0 && aligned16(a) && aligned16(y) && (!b || aligned16(b)))
        axpby_kernel<true><<<grid_for(n / 4, 256), 256, 0, st>>>(a, b, y, n, alpha, beta, rtf32);
    else
        axpby_kernel<false><<<grid_for(n, 256), 256, 0, st>>>(a, b, y, n, alpha, beta, rtf32);
    GIFB200_LAUNCH_CHECK("axpby_kernel");
    return GIFB200_OK;
}

int gifb200_demod(const float* s, const float* q, float* d, int B, int Ci, int Co, float eps, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && Ci > 0 && Co > 0, GIFB200_E_SHAPE, "demod: bad shape");
    if (B == 0) return GIFB200_OK;
    const long long warps = static_cast<long long>(B) * Co;
    demod_kernel<<<cdiv(warps * 32, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(s, q, d, B, Ci, Co, eps);
    GIFB200_LAUNCH_CHECK("demod_kernel");
    return GIFB200_OK;
}

int gifb200_torgb_fwd(const float* x, const float* ws, float* y, int B, int P, int C, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && P >= 0 && C > 0 && C <= 4096, GIFB200_E_SHAPE, "torgb_fwd: bad shape");
    GIFB200_REQUIRE(B <= 65535, GIFB200_E_SHAPE, "torgb_fwd: batch too large");
    if (B == 0 || P == 0) return GIFB200_OK;
    GIFB200_REQUIRE(C % 4 != 0 || aligned16(x), GIFB200_E_ALIGN, "torgb_fwd: x not 16B aligned");
    if (C % 32 == 0 && aligned16(x) && aligned16(ws)) {
        const int tx = vec_lanes(C);
        int rpb;
        const int rb = rows_split_vec(P, 1, B, 256 / tx, &rpb);
        GIFB200_REQUIRE(rb <= 65535, GIFB200_E_SHAPE, "torgb_fwd: grid too large");
        const dim3 grid(1, rb, B);
        cudaStream_t st = static_cast<cudaStream_t>(stream);
        if (tx == 32) torgb_fwd_vec_kernel<32><<<grid, 256, 0, st>>>(x, ws, y, P, C, rpb);
        else if (tx == 16) torgb_fwd_vec_kernel<16><<<grid, 256, 0, st>>>(x, ws, y, P, C, rpb);
        else torgb_fwd_vec_kernel<8><<<grid, 256, 0, st>>>(x, ws, y, P, C, rpb);
        GIFB200_LAUNCH_CHECK("torgb_fwd_vec_kernel");
        return GIFB200_OK;
    }
    int gx = cdiv(P, 8 * 4);
    const int cap = max(1, kNumSMs * 8 / B);
    if (gx > cap) gx = cap;
    torgb_fwd_kernel<<<dim3(gx, B), 256, 3 * C * sizeof(float), static_cast<cudaStream_t>(stream)>>>(x, ws, y, B, P, C);
    GIFB200_LAUNCH_CHECK("torgb_fwd_kernel");
    return GIFB200_OK;
}

int gifb200_torgb_bwd_x(const float* gy, const float* ws, float* gx, int B, int P, int C, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && P >= 0 && C > 0 && C <= 4096, GIFB200_E_SHAPE, "torgb_bwd_x: bad shape");
    GIFB200_REQUIRE(B <= 65535, GIFB200_E_SHAPE, "torgb_bwd_x: batch too large");
    if (B == 0 || P == 0) return GIFB200_OK;
    if (C % 4 == 0 && aligned16(gx) && aligned16(ws)) {
        int gv = cdiv(static_cast<long long>(P) * (C / 4), 256 * 4);
        const int capv = max(1, kNumSMs * 16 / B);
        if (gv > capv) gv = capv;
        torgb_bwd_x_vec_kernel<<<dim3(gv, B), 256, 0, static_cast<cudaStream_t>(stream)>>>(gy, ws, gx, P, C);
        GIFB200_LAUNCH_CHECK("torgb_bwd_x_vec_kernel");
        return GIFB200_OK;
    }
    int g = cdiv(static_cast<long long>(P) * C, 256 * 4);
    const int cap = max(1, kNumSMs * 8 / B);
    if (g > cap) g = cap;
    torgb_bwd_x_kernel<<<dim3(g, B), 256, 3 * C * sizeof(float), static_cast<cudaStream_t>(stream)>>>(gy, ws, gx, B, P, C);
    GIFB200_LAUNCH_CHECK("torgb_bwd_x_kernel");
    return GIFB200_OK;
}

int gifb200_torgb_bwd_w(const float* gy, const float* x, float* gws, int B, int P, int C, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && P >= 0 && C > 0, GIFB200_E_SHAPE, "torgb_bwd_w: bad shape");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (B == 0) return GIFB200_OK;
    cudaError_t e = cudaMemsetAsync(gws, 0, sizeof(float) * static_cast<size_t>(B) * 3 * C, st);
    if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "torgb_bwd_w memset", cudaGetErrorString(e));
    if (P == 0) return GIFB200_OK;
    if (C % 32 == 0 && aligned16(x) && aligned16(gws)) {
        const int tx = vec_lanes(C);
        int rpbv;
        const int cbv = C / (4 * tx);
        const int rbv = rows_split_vec(P, cbv, B, 256 / tx, &rpbv);
        GIFB200_REQUIRE(B <= 65535 && rbv <= 65535, GIFB200_E_SHAPE, "torgb_bwd_w: grid too large");
        const dim3 grid(cbv, rbv, B);
        Slots sl;
        if (int rc = slots_take(sl, gws, rbv, static_cast<long long>(B) * 3 * C, st)) return rc;
        if (tx == 32) torgb_bwd_w_vec_kernel<32><<<grid, 256, 0, st>>>(gy, x, gws, P, C, rpbv);
        else if (tx == 16) torgb_bwd_w_vec_kernel<16><<<grid, 256, 0, st>>>(gy, x, gws, P, C, rpbv);
        else torgb_bwd_w_vec_kernel<8><<<grid, 256, 0, st>>>(gy, x, gws, P, C, rpbv);
        GIFB200_LAUNCH_CHECK("torgb_bwd_w_vec_kernel");
        return slots_reduce(sl, st);
    }
    const int cb = cdiv(C, 32);
    int rpb;
    const int rb = rows_split(P, cb, B, &rpb);
    GIFB200_REQUIRE(B <= 65535 && rb <= 65535, GIFB200_E_SHAPE, "torgb_bwd_w: grid too large");
    Slots sl;
    if (int rc = slots_take(sl, gws, rb, static_cast<long long>(B) * 3 * C, st)) return rc;
    torgb_bwd_w_kernel<<<dim3(cb, rb, B), dim3(32, 8), 0, st>>>(gy, x, gws, P, C, rpb);
    GIFB200_LAUNCH_CHECK("torgb_bwd_w_kernel");
    return slots_reduce(sl, st);
}

int gifb200_cond_down(float* x, float* y, int B, int H, int W, int C, int s, int adjoint, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && H > 0 && W > 0 && C > 0, GIFB200_E_SHAPE, "cond_down: bad shape");
    GIFB200_REQUIRE(s >= 2 && (s & (s - 1)) == 0 && H % s == 0 && W % s == 0, GIFB200_E_SHAPE,
                    "cond_down: s must be a power of two >= 2 dividing H and W");
    if (B == 0) return GIFB200_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!adjoint) {
        const long long total = static_cast<long long>(B) * (H / s) * (W / s) * C;
        cond_down_kernel<<<grid_for(total, 256), 256, 0, st>>>(x, y, B, H, W, C, s);
        GIFB200_LAUNCH_CHECK("cond_down_kernel");
    } else {
        const long long total = static_cast<long long>(B) * H * W * C;
        cond_down_adj_kernel<<<grid_for(total, 256), 256, 0, st>>>(x, y, B, H, W, C, s);
        GIFB200_LAUNCH_CHECK("cond_down_adj_kernel");
    }
    return GIFB200_OK;
}

}  // extern "C"
