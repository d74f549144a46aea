// upfirdn2d: zero-insert upsample, pad/crop, small FIR, decimate -- one pass, channels-last.
// HBM-bound: algorithmic bytes = input + output (taps are re-read from L1/L2, never from HBM).
#include "common.cuh"

namespace gifb200 {

struct UpfirdnParams {
    int B, Hi, Wi, C, Ho, Wo, kh, kw, up, down, py0, px0, flip, rtf32;
};

// VEC: 4 channels per thread (C % 4 == 0).  Thread -> (pixel, channel group); consecutive threads walk the channel
// dimension first, so every tap is a fully coalesced 16B-per-lane read.
template <bool VEC>
__global__ void __launch_bounds__(256) upfirdn2d_kernel(const float* __restrict__ x, const float* __restrict__ kernel,
                                                        float* __restrict__ y, UpfirdnParams p) {
    __shared__ float sk[64];
    if (threadIdx.x < p.kh * p.kw) {
        const int a = threadIdx.x / p.kw, b = threadIdx.x % p.kw;
        // K[a][b] = flip ? kernel[kh-1-a][kw-1-b] : kernel[a][b]
        sk[threadIdx.x] = p.flip ? kernel[(p.kh - 1 - a) * p.kw + (p.kw - 1 - b)] : kernel[threadIdx.x];
    }
    __syncthreads();
    const int cg = VEC ? (p.C >> 2) : p.C;
    const long long total = static_cast<long long>(p.B) * p.Ho * p.Wo * cg;
    for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c = static_cast<int>(e % cg);
        long long r = e / cg;
        const int xo = static_cast<int>(r % p.Wo); r /= p.Wo;
        const int yo = static_cast<int>(r % p.Ho);
        const int b = static_cast<int>(r / p.Ho);
        // position in the zero-inserted grid touched by tap a: uy = yo*down + (kh-1-a) - py0
        const int uy_hi = yo * p.down + (p.kh - 1) - p.py0;  // a = 0
        const int ux_hi = xo * p.down + (p.kw - 1) - p.px0;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int a = 0; a < p.kh; ++a) {
            const int uy = uy_hi - a;
            if (uy < 0 || uy % p.up != 0) continue;
            const int iy = uy / p.up;
            if (iy >= p.Hi) continue;
            for (int bb = 0; bb < p.kw; ++bb) {
                const int ux = ux_hi - bb;
                if (ux < 0 || ux % p.up != 0) continue;
                const int ix = ux / p.up;
                if (ix >= p.Wi) continue;
                const float kv = sk[a * p.kw + bb];
                const long long off = ((static_cast<long long>(b) * p.Hi + iy) * p.Wi + ix) * p.C;
                if (VEC) {
                    const float4 v = __ldg(reinterpret_cast<const float4*>(x + off) + c);
                    acc.x += kv * v.x; acc.y += kv * v.y; acc.z += kv * v.z; acc.w += kv * v.w;
                } else {
                    acc.x += kv * __ldg(x + off + c);
                }
            }
        }
        if (p.rtf32) { acc.x = round_tf32(acc.x); acc.y = round_tf32(acc.y); acc.z = round_tf32(acc.z); acc.w = round_tf32(acc.w); }
        if (VEC) reinterpret_cast<float4*>(y)[e] = acc;
        else y[e] = acc.x;
    }
}

// Specialisation for the hot case (4x4 FIR, up = down = 1: every Blur of the generator / discriminator and their
// adjoints): each thread produces a column of R vertically adjacent outputs for 4 channels.  The R+3 input rows it
// needs are loaded ONCE (4 horizontal taps each) and scattered into the R accumulators, instead of 16 loads per output:
// (R+3)*4 / (16*R) = 44% of the load instructions / L1-L2 traffic at R = 4.
template <int R>
__global__ void __launch_bounds__(256) upfirdn2d_blur4_kernel(const float* __restrict__ x, const float* __restrict__ kernel,
                                                              float* __restrict__ y, UpfirdnParams p) {
    __shared__ float sk[16];
    if (threadIdx.x < 16) {
        const int a = threadIdx.x >> 2, b = threadIdx.x & 3;
        sk[threadIdx.x] = p.flip ? kernel[(3 - a) * 4 + (3 - b)] : kernel[threadIdx.x];
    }
    __syncthreads();
    const int cg = p.C >> 2;
    const int yblocks = (p.Ho + R - 1) / R;
    const long long total = static_cast<long long>(p.B) * yblocks * p.Wo * cg;
    for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c = static_cast<int>(e % cg);
        long long r = e / cg;
        const int xo = static_cast<int>(r % p.Wo); r /= p.Wo;
        const int yb = static_cast<int>(r % yblocks);
        const int b = static_cast<int>(r / yblocks);
        const int y0 = yb * R;
        float4 acc[R];
#pragma unroll
        for (int i = 0; i < R; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        // output row y0+i, tap a reads input row (y0+i) + (3-a) - py0;  input row index j = iy - (y0 - py0) in [0, R+3)
#pragma unroll
        for (int j = 0; j < R + 3; ++j) {
            const int iy = y0 - p.py0 + j;
            if (iy < 0 || iy >= p.Hi) continue;
            const float* row = x + ((static_cast<long long>(b) * p.Hi + iy) * p.Wi) * p.C;
#pragma unroll
            for (int bb = 0; bb < 4; ++bb) {
                const int ix = xo + (3 - bb) - p.px0;
                if (ix < 0 || ix >= p.Wi) continue;
                const float4 v = __ldg(reinterpret_cast<const float4*>(row + static_cast<long long>(ix) * p.C) + c);
#pragma unroll
                for (int i = 0; i < R; ++i) {
                    const int a = 3 - (j - i);          // j = i + (3 - a)
                    if (a < 0 || a > 3) continue;
                    const float kv = sk[a * 4 + bb];
                    acc[i].x += kv * v.x; acc[i].y += kv * v.y; acc[i].z += kv * v.z; acc[i].w += kv * v.w;
                }
            }
        }
#pragma unroll
        for (int i = 0; i < R; ++i) {
            const int yo = y0 + i;
            if (yo >= p.Ho) break;
            float4 o = acc[i];
            if (p.rtf32) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
            reinterpret_cast<float4*>(y + ((static_cast<long long>(b) * p.Ho + yo) * p.Wo + xo) * p.C)[c] = o;
        }
    }
}

// Tile geometry of the shared-memory FIR kernels below (C % 32 == 0): 16 x 16 outputs from (16+3)^2 input pixels x 32
// channels (46 KB; read amplification 1.41x instead of 16x through L1/L2) for up = down = 1.
constexpr int kBT = 16;                 // output tile edge
constexpr int kBTI = kBT + 3;           // input tile edge
// Decimation by 2 (D's blur -> 1x1 stride-2 skip evaluated as upfirdn2d(down=2), adjoints of up=2): 8 x 8 outputs from
// (2*8+2)^2 input pixels x 32 channels (41 KB; read amplification 1.27x instead of 4x).
constexpr int kDT = 8;                  // output tile edge
constexpr int kDTI = 2 * kDT + 2;       // input tile edge
// ------------------------------------------------------------------------------------------------ pipelined 4x4 FIR
// Persistent, double-buffered shared-memory FIR (C % 32 == 0, 4x4 kernel, up = 1, down = 1 or 2).
// A single-buffered blur moves only the algorithmic DRAM bytes but stalls on `long_scoreboard` -- a CTA loads its tile,
// waits, computes, and 4 CTAs per SM (register + smem limit) do not keep enough bytes in flight.  Here a CTA walks a list of
// tiles and issues the cp.async (LDGSTS, zero-fill for the padding) loads of tile i+1 before it computes tile i, so
// every SM always has 2 x 41-46 KB of reads in flight underneath the FMAs and stores.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, int src_bytes) {
    const unsigned d = static_cast<unsigned>(__cvta_generic_to_shared(smem_dst));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

template <int DOWN>
__global__ void __launch_bounds__(256, 2) upfirdn2d_fir4_pipe_kernel(const float* __restrict__ x,
                                                                     const float* __restrict__ kernel,
                                                                     float* __restrict__ y, UpfirdnParams p, int tiles_x,
                                                                     int tiles_y, int total_tiles) {
    constexpr int TO = DOWN == 1 ? kBT : kDT;          // output tile edge
    constexpr int TI = DOWN == 1 ? kBTI : kDTI;        // input tile edge
    constexpr int TILE_F4 = TI * TI * 8;
    extern __shared__ float4 fir_smem[];
    float kreg[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) kreg[i] = p.flip ? __ldg(kernel + 15 - i) : __ldg(kernel + i);
    // rank-1 kernel (every Blur of the model: outer([1,3,3,1]) * gain / 64)?  Exact test, uniform across the grid.
    bool separable = DOWN == 1 && kreg[0] != 0.f;
    float kcol[4], krow[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        kcol[a] = kreg[a * 4];
        krow[a] = separable ? kreg[a] / kreg[0] : 0.f;
    }
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) separable = separable && (kcol[a] * krow[b] == kreg[a * 4 + b]);
    const int cchunks = p.C >> 5;

    auto decode = [&](int t, int& b, int& y0, int& x0, int& cc) {
        cc = t % cchunks; t /= cchunks;
        x0 = (t % tiles_x) * TO; t /= tiles_x;
        y0 = (t % tiles_y) * TO;
        b = t / tiles_y;
    };
    // per-thread tile coordinates of its first element; the k-th element is 32 pixels further (256 threads / 8 lanes)
    const int c4l = threadIdx.x & 7;
    const int pix0 = threadIdx.x >> 3;
    const int py_first = pix0 / TI, px_first = pix0 - py_first * TI;
    auto issue = [&](int t, int buf) {
        int b, y0, x0, cc;
        decode(t, b, y0, x0, cc);
        const int ix0 = DOWN * x0 - p.px0, iy0 = DOWN * y0 - p.py0;
        const float* xb = x + static_cast<long long>(b) * p.Hi * p.Wi * p.C + cc * 32 + c4l * 4;
        float4* dst = fir_smem + buf * TILE_F4 + threadIdx.x;
        int px = px_first, py = py_first;
#pragma unroll
        for (int k = 0; k < (TILE_F4 + 255) / 256; ++k) {
            if (k * 256 + static_cast<int>(threadIdx.x) < TILE_F4) {
                const int gx = ix0 + px, gy = iy0 + py;
                const bool ok = static_cast<unsigned>(gx) < static_cast<unsigned>(p.Wi) &&
                                static_cast<unsigned>(gy) < static_cast<unsigned>(p.Hi);
                const float* src = ok ? xb + (static_cast<long long>(gy) * p.Wi + gx) * p.C : x;
                cp_async16(dst + k * 256, src, ok ? 16 : 0);
            }
            px += 32 - TI; py += 1;                       // +32 pixels, TI < 32 < 2*TI
            if (px >= TI) { px -= TI; py += 1; }
        }
        cp_async_commit();
    };

    int t = blockIdx.x, buf = 0;
    if (t < total_tiles) issue(t, 0);
    for (; t < total_tiles; t += gridDim.x, buf ^= 1) {
        const int tn = t + gridDim.x;
        if (tn < total_tiles) { issue(tn, buf ^ 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
        __syncthreads();
        const float4* tile = fir_smem + buf * TILE_F4;
        int b, y0, x0, cc;
        decode(t, b, y0, x0, cc);
        const int c4 = threadIdx.x & 7;
        if (DOWN == 1) {
            const int lx = (threadIdx.x >> 3) & 15, half = threadIdx.x >> 7;
            constexpr int R = 8;
            float4 acc[R];
#pragma unroll
            for (int i = 0; i < R; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (separable) {
                // K[a][b] = kcol[a] * krow[b]: one horizontal 4-tap pass per input row, then the vertical taps
                // (11*16 + 32*4 = 304 FMAs per thread instead of 512)
#pragma unroll
                for (int j = 0; j < R + 3; ++j) {
                    const int row = half * R + j;
                    float4 h = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int bb = 0; bb < 4; ++bb) {
                        const float4 v = tile[(row * TI + lx + 3 - bb) * 8 + c4];
                        h.x += krow[bb] * v.x; h.y += krow[bb] * v.y; h.z += krow[bb] * v.z; h.w += krow[bb] * v.w;
                    }
#pragma unroll
                    for (int i = 0; i < R; ++i) {
                        const int a = 3 - (j - i);
                        if (a < 0 || a > 3) continue;
                        acc[i].x += kcol[a] * h.x; acc[i].y += kcol[a] * h.y; acc[i].z += kcol[a] * h.z; acc[i].w += kcol[a] * h.w;
                    }
                }
            } else {
#pragma unroll
                for (int j = 0; j < R + 3; ++j) {
                    const int row = half * R + j;
#pragma unroll
                    for (int bb = 0; bb < 4; ++bb) {
                        const float4 v = tile[(row * TI + lx + 3 - bb) * 8 + c4];
#pragma unroll
                        for (int i = 0; i < R; ++i) {
                            const int a = 3 - (j - i);
                            if (a < 0 || a > 3) continue;
                            const float kv = kreg[a * 4 + bb];
                            acc[i].x += kv * v.x; acc[i].y += kv * v.y; acc[i].z += kv * v.z; acc[i].w += kv * v.w;
                        }
                    }
                }
            }
            const int xo = x0 + lx;
            if (xo < p.Wo) {
#pragma unroll
                for (int i = 0; i < R; ++i) {
                    const int yo = y0 + half * R + i;
                    if (yo < p.Ho) {
                        float4 o = acc[i];
                        if (p.rtf32) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
                        reinterpret_cast<float4*>(y + ((static_cast<long long>(b) * p.Ho + yo) * p.Wo + xo) * p.C + cc * 32)[c4] = o;
                    }
                }
            }
        } else {
            const int lx = (threadIdx.x >> 3) & 7, rp = threadIdx.x >> 6;
            float4 acc0 = make_float4(0.f, 0.f, 0.f, 0.f), acc1 = acc0;
#pragma unroll
            for (int j = 0; j < 6; ++j) {
                const int row = 4 * rp + j;
#pragma unroll
                for (int bb = 0; bb < 4; ++bb) {
                    const float4 v = tile[(row * TI + 2 * lx + 3 - bb) * 8 + c4];
                    if (j <= 3) {
                        const float kv = kreg[(3 - j) * 4 + bb];
                        acc0.x += kv * v.x; acc0.y += kv * v.y; acc0.z += kv * v.z; acc0.w += kv * v.w;
                    }
                    if (j >= 2) {
                        const float kv = kreg[(5 - j) * 4 + bb];
                        acc1.x += kv * v.x; acc1.y += kv * v.y; acc1.z += kv * v.z; acc1.w += kv * v.w;
                    }
                }
            }
            const int xo = x0 + lx;
            if (xo < p.Wo) {
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int yo = y0 + 2 * rp + i;
                    if (yo < p.Ho) {
                        float4 o = i ? acc1 : acc0;
                        if (p.rtf32) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
                        reinterpret_cast<float4*>(y + ((static_cast<long long>(b) * p.Ho + yo) * p.Wo + xo) * p.C + cc * 32)[c4] = o;
                    }
                }
            }
        }
        __syncthreads();      // everyone is done with `buf` before the next iteration's loads overwrite it
    }
}

// Zero-insert x2 upsampling + 4x4 FIR (the adjoint of every decimating call: D's skip / blur backward) for C % 32 == 0,
// same persistent cp.async double-buffered scheme.  An output pixel sees only the 2 x 2 taps whose zero-inserted
// position is even, so a 16 x 16 output tile needs a 10 x 10 input tile (12.5 KB); which taps apply depends on the
// output row / column parity: the 16 kernel values are permuted once per thread into kk[row parity][s][t] (the column
// parity is fixed per thread), everything else is compile-time indexed.
constexpr int kUT = 16;                 // output tile edge
constexpr int kUTI = kUT / 2 + 2;       // input tile edge
__global__ void __launch_bounds__(256, 4) upfirdn2d_up2_pipe_kernel(const float* __restrict__ x,
                                                                    const float* __restrict__ kernel,
                                                                    float* __restrict__ y, UpfirdnParams p, int tiles_x,
                                                                    int tiles_y, int total_tiles) {
    constexpr int TI = kUTI, TILE_F4 = TI * TI * 8;
    __shared__ float4 tiles[2][TILE_F4];
    float kreg[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) kreg[i] = p.flip ? __ldg(kernel + 15 - i) : __ldg(kernel + i);
    const int cchunks = p.C >> 5;
    const int c4 = threadIdx.x & 7, lx = (threadIdx.x >> 3) & 15, half = threadIdx.x >> 7;
    const int q = lx & 1, mx = lx >> 1;
    // tile origins are multiples of 16, so parities depend on (py0, px0) only.  Output row Y = y0 + 8*half + 2m + r uses
    // kernel rows a(r,s) = ((r + 3 - py0) & 1) + 2s at input row (Y + 3 - py0 - a)/2; same for columns with (q, t).
    int ar[2][2], bt[2], offy[2][2], offx[2];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int sl = 0; sl < 2; ++sl) {
            ar[r][sl] = ((r + 3 - p.py0) & 1) + 2 * sl;
            offy[r][sl] = ((3 - p.py0 + r - ar[r][sl]) >> 1) - ((-p.py0) >> 1);      // relative to the tile's first input row
        }
#pragma unroll
    for (int t = 0; t < 2; ++t) {
        bt[t] = ((q + 3 - p.px0) & 1) + 2 * t;
        offx[t] = ((3 - p.px0 + q - bt[t]) >> 1) - ((-p.px0) >> 1);
    }
    float kk[2][2][2];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int sl = 0; sl < 2; ++sl)
#pragma unroll
            for (int t = 0; t < 2; ++t) {
                const int idx = ar[r][sl] * 4 + bt[t];
                float v = 0.f;
#pragma unroll
                for (int i = 0; i < 16; ++i) v = (i == idx) ? kreg[i] : v;
                kk[r][sl][t] = v;
            }

    auto decode = [&](int t, int& b, int& y0, int& x0, int& cc) {
        cc = t % cchunks; t /= cchunks;
        x0 = (t % tiles_x) * kUT; t /= tiles_x;
        y0 = (t % tiles_y) * kUT;
        b = t / tiles_y;
    };
    auto issue = [&](int t, int buf) {
        int b, y0, x0, cc;
        decode(t, b, y0, x0, cc);
        const int ix0 = (x0 - p.px0) >> 1, iy0 = (y0 - p.py0) >> 1;      // floor: first input column / row of the tile
        const float* xb = x + static_cast<long long>(b) * p.Hi * p.Wi * p.C + cc * 32;
        for (int idx = threadIdx.x; idx < TILE_F4; idx += 256) {
            const int cl = idx & 7, pix = idx >> 3;
            const int px = pix % TI, py = pix / TI;
            const int gx = ix0 + px, gy = iy0 + py;
            const bool ok = static_cast<unsigned>(gx) < static_cast<unsigned>(p.Wi) &&
                            static_cast<unsigned>(gy) < static_cast<unsigned>(p.Hi);
            const float* src = ok ? xb + (static_cast<long long>(gy) * p.Wi + gx) * p.C + cl * 4 : x;
            cp_async16(&tiles[buf][idx], src, ok ? 16 : 0);
        }
        cp_async_commit();
    };

    int t = blockIdx.x, buf = 0;
    if (t < total_tiles) issue(t, 0);
    for (; t < total_tiles; t += gridDim.x, buf ^= 1) {
        const int tn = t + gridDim.x;
        if (tn < total_tiles) { issue(tn, buf ^ 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
        __syncthreads();
        const float4* tile = tiles[buf];
        int b, y0, x0, cc;
        decode(t, b, y0, x0, cc);
        const int xo = x0 + lx;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int m = i >> 1, r = i & 1;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int sl = 0; sl < 2; ++sl)
#pragma unroll
                for (int tt = 0; tt < 2; ++tt) {
                    const float4 v = tile[((m + 4 * half + offy[r][sl]) * TI + mx + offx[tt]) * 8 + c4];
                    const float kv = kk[r][sl][tt];
                    acc.x += kv * v.x; acc.y += kv * v.y; acc.z += kv * v.z; acc.w += kv * v.w;
                }
            const int yo = y0 + half * 8 + i;
            if (xo < p.Wo && yo < p.Ho) {
                if (p.rtf32) { acc.x = round_tf32(acc.x); acc.y = round_tf32(acc.y); acc.z = round_tf32(acc.z); acc.w = round_tf32(acc.w); }
                reinterpret_cast<float4*>(y + ((static_cast<long long>(b) * p.Ho + yo) * p.Wo + xo) * p.C + cc * 32)[c4] = acc;
            }
        }
        __syncthreads();
    }
}

}  // namespace gifb200

using namespace gifb200;

extern "C" int gifb200_upfirdn2d(const float* x, const float* kernel, float* y, int B, int Hi, int Wi, int C, int Ho,
                                 int Wo, int kh, int kw, int up, int down, int pad_y0, int pad_x0, int flip,
                                 int round_tf32, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && Hi > 0 && Wi > 0 && C > 0 && Ho >= 0 && Wo >= 0, GIFB200_E_SHAPE, "upfirdn2d: bad shape");
    GIFB200_REQUIRE(kh >= 1 && kw >= 1 && kh <= 8 && kw <= 8, GIFB200_E_SHAPE, "upfirdn2d: kernel must be <= 8x8");
    GIFB200_REQUIRE(up >= 1 && down >= 1, GIFB200_E_SHAPE, "upfirdn2d: up/down must be >= 1");
    const long long total = static_cast<long long>(B) * Ho * Wo * C;
    if (total == 0) return GIFB200_OK;
    UpfirdnParams p{B, Hi, Wi, C, Ho, Wo, kh, kw, up, down, pad_y0, pad_x0, flip, round_tf32};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool vec = (C % 4 == 0) && aligned16(x) && aligned16(y);
    if (vec && C % 32 == 0 && kh == 4 && kw == 4 && up == 2 && down == 1 && Ho >= 8 && Wo >= 8 && pad_y0 >= 0 &&
        pad_x0 >= 0 && pad_y0 <= 3 && pad_x0 <= 3) {
        const int tiles_x = (Wo + kUT - 1) / kUT, tiles_y = (Ho + kUT - 1) / kUT;
        const long long tiles = static_cast<long long>(B) * tiles_x * tiles_y * (C / 32);
        GIFB200_REQUIRE(tiles <= 2147483647LL, GIFB200_E_SHAPE, "upfirdn2d: grid too large");
        const int ctas = static_cast<int>(tiles < 4LL * kNumSMs ? tiles : 4LL * kNumSMs);
        upfirdn2d_up2_pipe_kernel<<<ctas, 256, 0, st>>>(x, kernel, y, p, tiles_x, tiles_y, static_cast<int>(tiles));
        GIFB200_LAUNCH_CHECK("upfirdn2d_up2_pipe_kernel");
        return GIFB200_OK;
    }
    if (vec && C % 32 == 0 && kh == 4 && kw == 4 && up == 1 && (down == 1 || down == 2) && Ho >= 4 && Wo >= 4) {
        const int to = down == 1 ? kBT : kDT, ti = down == 1 ? kBTI : kDTI;
        const int tiles_x = (Wo + to - 1) / to, tiles_y = (Ho + to - 1) / to;
        const long long tiles = static_cast<long long>(B) * tiles_x * tiles_y * (C / 32);
        GIFB200_REQUIRE(tiles <= 2147483647LL, GIFB200_E_SHAPE, "upfirdn2d: grid too large");
        const int smem = 2 * ti * ti * 8 * static_cast<int>(sizeof(float4));
        const int ctas = static_cast<int>(tiles < 2LL * kNumSMs ? tiles : 2LL * kNumSMs);
        static const cudaError_t attr = [] {
            cudaError_t e1 = cudaFuncSetAttribute(upfirdn2d_fir4_pipe_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                  2 * kBTI * kBTI * 8 * static_cast<int>(sizeof(float4)));
            cudaError_t e2 = cudaFuncSetAttribute(upfirdn2d_fir4_pipe_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                  2 * kDTI * kDTI * 8 * static_cast<int>(sizeof(float4)));
            return e1 != cudaSuccess ? e1 : e2;
        }();
        if (attr != cudaSuccess) return fail(GIFB200_E_CUDA, "upfirdn2d smem attribute", cudaGetErrorString(attr));
        if (down == 1)
            upfirdn2d_fir4_pipe_kernel<1><<<ctas, 256, smem, st>>>(x, kernel, y, p, tiles_x, tiles_y, static_cast<int>(tiles));
        else
            upfirdn2d_fir4_pipe_kernel<2><<<ctas, 256, smem, st>>>(x, kernel, y, p, tiles_x, tiles_y, static_cast<int>(tiles));
        GIFB200_LAUNCH_CHECK("upfirdn2d_fir4_pipe_kernel");
        return GIFB200_OK;
    }
    if (vec && kh == 4 && kw == 4 && up == 1 && down == 1 && Ho >= 4) {
        constexpr int R = 4;
        const long long items4 = static_cast<long long>(B) * ((Ho + R - 1) / R) * Wo * (C / 4);
        long long blocks4 = (items4 + 255) / 256;
        const long long cap4 = static_cast<long long>(kNumSMs) * 32;
        if (blocks4 > cap4) blocks4 = cap4;
        upfirdn2d_blur4_kernel<R><<<static_cast<int>(blocks4), 256, 0, st>>>(x, kernel, y, p);
        GIFB200_LAUNCH_CHECK("upfirdn2d_blur4_kernel");
        return GIFB200_OK;
    }
    const long long items = vec ? total / 4 : total;
    long long blocks = (items + 255) / 256;
    const long long cap = static_cast<long long>(kNumSMs) * 32;
    if (blocks > cap) blocks = cap;
    if (vec) upfirdn2d_kernel<true><<<static_cast<int>(blocks), 256, 0, st>>>(x, kernel, y, p);
    else upfirdn2d_kernel<false><<<static_cast<int>(blocks), 256, 0, st>>>(x, kernel, y, p);
    GIFB200_LAUNCH_CHECK("upfirdn2d_kernel");
    return GIFB200_OK;
}
