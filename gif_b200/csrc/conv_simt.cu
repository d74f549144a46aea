// SIMT fp32 implicit-GEMM convolution (forward / input-gradient for all three modes, and weight gradient).
//
// Role: (1) the exact-fp32 path for shapes the tensor-core kernel does not take (Ci or Co not a multiple of 32/16:
// the 9-channel D stem, the 6->12->24 NoiseInjection convs, ragged test shapes), (2) the on-GPU cross-check of the
// tensor-core kernel.  Tiling: 64 output pixels x 64 output channels per CTA, K chunks of 16 input channels per
// tap, 256 threads with 4x4 register micro-tiles.
#include "common.cuh"

namespace gifb200 {

struct ConvParams {
    int B, Hi, Wi, Ci, Ho, Wo, Co, k, flip;
    long long M;  // number of output pixels (B*Ho*Wo)
    ConvEpilogue epi;
};

// m-th output pixel of the launch -> (b, yo, xo)
__device__ __forceinline__ void decode_pixel(const ConvParams& p, long long m, int& b, int& yo, int& xo) {
    xo = static_cast<int>(m % p.Wo);
    const long long r = m / p.Wo;
    yo = static_cast<int>(r % p.Ho);
    b = static_cast<int>(r / p.Ho);
}

constexpr int BM = 64, BN = 64, BK = 16;

// input pixel for output pixel (yo,xo) and tap (kh,kw); returns false if the tap reads a structural zero
template <int MODE>
__device__ __forceinline__ bool tap_source(const ConvParams& p, int yo, int xo, int kh, int kw, int& yi, int& xi) {
    if (MODE == 0) {
        yi = yo + kh - p.k / 2;
        xi = xo + kw - p.k / 2;
    } else if (MODE == 1) {
        yi = 2 * yo + kh;
        xi = 2 * xo + kw;
    } else {
        const int ty = yo - kh, tx = xo - kw;
        if (ty < 0 || tx < 0 || (ty & 1) || (tx & 1)) return false;
        yi = ty >> 1;
        xi = tx >> 1;
    }
    return yi >= 0 && yi < p.Hi && xi >= 0 && xi < p.Wi;
}

template <int MODE, bool WT>
__global__ void __launch_bounds__(256) conv_simt_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                        float* __restrict__ y, ConvParams p) {
    __shared__ float As[BK][BM + 4];
    __shared__ float Bs[BK][BN + 4];
    const int tid = threadIdx.x;
    const long long m0 = static_cast<long long>(blockIdx.x) * BM;
    const int n0 = blockIdx.y * BN;
    const int T = p.k * p.k;

    // A-load role: pixel (tid/4), channel sub-chunk (tid%4)*4 .. +3
    const int a_row = tid >> 2, a_c = (tid & 3) << 2;
    const long long a_m = m0 + a_row;
    int a_b = 0, a_yo = 0, a_xo = 0;
    const bool a_ok = a_m < p.M;
    if (a_ok) decode_pixel(p, a_m, a_b, a_yo, a_xo);
    const int tm = (tid >> 4) << 2, tn = (tid & 15) << 2;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int t = 0; t < T; ++t) {
        const int kh = t / p.k, kw = t % p.k;
        const int tt = p.flip ? T - 1 - t : t;
        int yi = 0, xi = 0;
        const bool src_ok = a_ok && tap_source<MODE>(p, a_yo, a_xo, kh, kw, yi, xi);
        if (MODE == 2 && !__syncthreads_or(src_ok)) continue;   // no pixel of this tile reads this tap (T2 parity / border)
        const float* xrow = x + ((static_cast<long long>(a_b) * p.Hi + yi) * p.Wi + xi) * p.Ci;
        const float* wt = w + static_cast<long long>(tt) * p.Co * p.Ci;
        for (int c0 = 0; c0 < p.Ci; c0 += BK) {
            // ---- A tile: As[k][m] = x[pixel m][c0+k]
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int c = c0 + a_c + j;
                As[a_c + j][a_row] = (src_ok && c < p.Ci) ? __ldg(xrow + c) : 0.f;
            }
            // ---- B tile: Bs[k][n] = W[t][n0+n][c0+k]
            if (!WT) {  // physical w[tt][o][i]: read 4 consecutive i for one o
                const int o = n0 + (tid >> 2), ib = (tid & 3) << 2;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int c = c0 + ib + j;
                    Bs[ib + j][tid >> 2] = (o < p.Co && c < p.Ci) ? __ldg(wt + static_cast<long long>(o) * p.Ci + c) : 0.f;
                }
            } else {  // physical w[tt][i][o]: read 4 consecutive o for one i
                const int i = c0 + (tid >> 4), ob = (tid & 15) << 2;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int o = n0 + ob + j;
                    Bs[tid >> 4][ob + j] = (i < p.Ci && o < p.Co) ? __ldg(wt + static_cast<long long>(i) * p.Co + o) : 0.f;
                }
            }
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < BK; ++kk) {
                const float4 a = *reinterpret_cast<const float4*>(&As[kk][tm]);
                const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tn]);
                const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] += av[i] * bv[j];
            }
            __syncthreads();
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long m = m0 + tm + i;
        if (m >= p.M) continue;
        int ob, oy, ox;
        decode_pixel(p, m, ob, oy, ox);
        float* yrow = y + ((static_cast<long long>(ob) * p.Ho + oy) * p.Wo + ox) * p.Co;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int o = n0 + tn + j;
            if (o < p.Co) yrow[o] = apply_epilogue(p.epi, acc[i][j], o);
        }
    }
}

// -------------------------------------------------------------------------------------------------- wgrad
// R[t][cs][cb] = sum_{pixels p of the SMALL grid} S[p][cs] * Bg[map(p,t)][cb],   map(p,t) = (st*y + kh - pad, st*x + kw - pad)
//   S1: S = gy (Cs=Co), Bg = x (Cb=Ci), st=1, pad=k/2;   S2: S = gy, Bg = x, st=2, pad=0;
//   T2: S = x (Cs=Ci), Bg = gy (Cb=Co), st=2, pad=0  (the roles of the two tensors swap).
// The result is scattered into the physical weight layout through (stride_cs, stride_cb).  Split over pixels
// (gridDim.z = T * splits): every split writes its own slot of a Slots buffer (common.cuh), added in split order.
struct WgradParams {
    int B, Hs, Ws, Cs, Hb, Wb, Cb, k, st, pad, flip, splits;
    long long Ms;  // B*Hs*Ws
    long long stride_t, stride_cs, stride_cb;
};

__global__ void __launch_bounds__(256) wgrad_simt_kernel(const float* __restrict__ S, const float* __restrict__ Bg,
                                                         float* __restrict__ out, WgradParams p) {
    __shared__ float As[BK][BM + 4];  // [pixel][cs]
    __shared__ float Bs[BK][BN + 4];  // [pixel][cb]
    const int tid = threadIdx.x;
    const int cs0 = blockIdx.x * BM, cb0 = blockIdx.y * BN;
    const int t = blockIdx.z / p.splits, split = blockIdx.z % p.splits;
    const int kh = t / p.k, kw = t % p.k;
    const long long chunk = ((p.Ms + p.splits - 1) / p.splits + BK - 1) / BK * BK;
    const long long p_begin = split * chunk;
    const long long p_end = min(p.Ms, p_begin + chunk);
    const int tm = (tid >> 4) << 2, tn = (tid & 15) << 2;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    // load role: pixel row (tid/16), 4 consecutive channels (tid%16)*4
    const int lrow = tid >> 4, lc = (tid & 15) << 2;
    for (long long p0 = p_begin; p0 < p_end; p0 += BK) {
        const long long pix = p0 + lrow;
        const bool ok = pix < p_end;
        int xs = 0, ys = 0, b = 0;
        if (ok) {
            xs = static_cast<int>(pix % p.Ws);
            const long long r = pix / p.Ws;
            ys = static_cast<int>(r % p.Hs);
            b = static_cast<int>(r / p.Hs);
        }
        const int yb = p.st * ys + kh - p.pad, xb = p.st * xs + kw - p.pad;
        const bool okb = ok && yb >= 0 && yb < p.Hb && xb >= 0 && xb < p.Wb;
        const float* srow = S + pix * p.Cs;
        const float* brow = Bg + ((static_cast<long long>(b) * p.Hb + yb) * p.Wb + xb) * p.Cb;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int cs = cs0 + lc + j, cb = cb0 + lc + j;
            As[lrow][lc + j] = (okb && cs < p.Cs) ? __ldg(srow + cs) : 0.f;   // okb: a zero on either side kills the term
            Bs[lrow][lc + j] = (okb && cb < p.Cb) ? __ldg(brow + cb) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            const float4 a = *reinterpret_cast<const float4*>(&As[kk][tm]);
            const float4 bq = *reinterpret_cast<const float4*>(&Bs[kk][tn]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {bq.x, bq.y, bq.z, bq.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] += av[i] * bv[j];
        }
        __syncthreads();
    }
    const int tt = p.flip ? p.k * p.k - 1 - t : t;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int cs = cs0 + tm + i;
        if (cs >= p.Cs) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int cb = cb0 + tn + j;
            if (cb < p.Cb) out[split * p.k * p.k * p.stride_t + tt * p.stride_t + cs * p.stride_cs + cb * p.stride_cb] = acc[i][j];
        }
    }
}

static int check_conv_shape(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode) {
    GIFB200_REQUIRE(B >= 0 && Hi > 0 && Wi > 0 && Ci > 0 && Ho > 0 && Wo > 0 && Co > 0, GIFB200_E_SHAPE, "conv2d: bad shape");
    GIFB200_REQUIRE(k == 1 || k == 3, GIFB200_E_SHAPE, "conv2d: k must be 1 or 3");
    if (mode == 0) GIFB200_REQUIRE(Ho == Hi && Wo == Wi, GIFB200_E_SHAPE, "conv2d S1: output size must equal input size");
    else if (mode == 1)
        GIFB200_REQUIRE(Hi >= 2 * (Ho - 1) + k && Wi >= 2 * (Wo - 1) + k, GIFB200_E_SHAPE, "conv2d S2: input too small");
    else if (mode == 2)
        GIFB200_REQUIRE(Ho == 2 * (Hi - 1) + k && Wo == 2 * (Wi - 1) + k, GIFB200_E_SHAPE,
                        "conv2d T2: output size must be 2*(in-1)+k");
    else return fail(GIFB200_E_SHAPE, "conv2d: mode must be 0, 1 or 2");
    return GIFB200_OK;
}

int conv2d_simt(const float* x, const float* w, float* y, int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k,
                int mode, int flip, int transposed, const ConvEpilogue& epi, cudaStream_t st) {
    int rc = check_conv_shape(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode);
    if (rc != GIFB200_OK) return rc;
    if (B == 0) return GIFB200_OK;
    ConvParams p{B, Hi, Wi, Ci, Ho, Wo, Co, k, flip, static_cast<long long>(B) * Ho * Wo, epi};
    const long long mb = (p.M + BM - 1) / BM;
    GIFB200_REQUIRE(mb <= 2147483647LL && cdiv(Co, BN) <= 65535, GIFB200_E_SHAPE, "conv2d: grid too large");
    dim3 grid(static_cast<unsigned>(mb), cdiv(Co, BN));
#define LAUNCH(MODE, WT) conv_simt_kernel<MODE, WT><<<grid, 256, 0, st>>>(x, w, y, p)
    if (mode == 0) { if (transposed) LAUNCH(0, true); else LAUNCH(0, false); }
    else if (mode == 1) { if (transposed) LAUNCH(1, true); else LAUNCH(1, false); }
    else { if (transposed) LAUNCH(2, true); else LAUNCH(2, false); }
#undef LAUNCH
    GIFB200_LAUNCH_CHECK("conv_simt_kernel");
    return GIFB200_OK;
}

int conv2d_wgrad_simt(const float* x, const float* gy, float* gw, int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co,
                      int k, int mode, int flip, int transposed, cudaStream_t st) {
    int rc = check_conv_shape(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode);
    if (rc != GIFB200_OK) return rc;
    const int T = k * k;
    cudaError_t e = cudaMemsetAsync(gw, 0, sizeof(float) * static_cast<size_t>(T) * Co * Ci, st);
    if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "wgrad memset", cudaGetErrorString(e));
    if (B == 0) return GIFB200_OK;
    WgradParams p;
    p.B = B; p.k = k; p.flip = flip;
    const float *S, *Bg;
    // physical layout of gw: transposed ? [t][i][o] : [t][o][i]
    const long long stride_o = transposed ? 1 : Ci, stride_i = transposed ? Co : 1;
    if (mode == 2) {  // small grid = conv input x (channels i), big = gy (channels o)
        S = x; Bg = gy;
        p.Hs = Hi; p.Ws = Wi; p.Cs = Ci; p.Hb = Ho; p.Wb = Wo; p.Cb = Co; p.st = 2; p.pad = 0;
        p.stride_cs = stride_i; p.stride_cb = stride_o;
    } else {          // small grid = gy (channels o), big = x (channels i)
        S = gy; Bg = x;
        p.Hs = Ho; p.Ws = Wo; p.Cs = Co; p.Hb = Hi; p.Wb = Wi; p.Cb = Ci;
        p.st = mode == 1 ? 2 : 1; p.pad = mode == 1 ? 0 : k / 2;
        p.stride_cs = stride_o; p.stride_cb = stride_i;
    }
    p.stride_t = static_cast<long long>(Co) * Ci;
    p.Ms = static_cast<long long>(B) * p.Hs * p.Ws;
    const int gx = cdiv(p.Cs, BM), gy_ = cdiv(p.Cb, BN);
    long long splits = (static_cast<long long>(kNumSMs) * 4 + static_cast<long long>(gx) * gy_ * T - 1) /
                       (static_cast<long long>(gx) * gy_ * T);
    const long long max_splits = (p.Ms + 255) / 256;  // at least 256 pixels per split
    if (splits > max_splits) splits = max_splits;
    if (splits < 1) splits = 1;
    if (splits * T > 65535) splits = 65535 / T;
    p.splits = static_cast<int>(splits);
    Slots sl;
    if (int rc2 = slots_take(sl, gw, p.splits, static_cast<long long>(T) * Co * Ci, st)) return rc2;
    wgrad_simt_kernel<<<dim3(gx, gy_, T * p.splits), 256, 0, st>>>(S, Bg, gw, p);
    GIFB200_LAUNCH_CHECK("wgrad_simt_kernel");
    return slots_reduce(sl, st);
}

}  // namespace gifb200
