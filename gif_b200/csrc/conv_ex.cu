// gifb200_conv2d_ex: forward convolution of general geometry (any kh, kw <= 7, stride 1 or 2, any pads, any map size),
// written into a channel slice [c0, c0+Co) of an output with Cy channels per pixel.  The FID InceptionV3 runs on it.
//
// GEMM view: D[m, o] = sum_{t, i} A[m, t, i] * W[t][o][i], m = flattened output pixel (b, yo, xo).  Flattening M (instead
// of the 2-D site boxes of conv_tc.cu) wastes no tile rows on 17x17 / 8x8 maps and needs no power-of-two grid.
//   * impl 1: exact fp32 SIMT kernel (64 pixels x 64 channels per CTA, 4x4 register micro-tiles).
//   * impl 2 / 3: wgmma, 128 pixels x BN channels per CTA (BN = 128 / 64 / 32), K = taps x 32-channel chunks.  All 256
//     threads gather the A tile with cp.async (zero fill for padding, out-of-map taps and rows past M) straight into the
//     K-major swizzled layout wgmma reads, and the B tile (staged weights) the same way; a 4-stage ring.  Each of the two
//     warpgroups issues m64nBN wgmmas on its 64 rows.  impl 3 ("bf16x3") reads the two bf16 planes of gifb200_split_bf16
//     and accumulates lo*hi + hi*lo + hi*hi per 16-channel slice, in that order, as conv_tc.cu does.
//   * Few output tiles (8x8 / 17x17 maps at small batch): split-K into per-split partial buffers, added in split order by a
//     reduction pass that applies the epilogue.  Every schedule is a fixed function of the shape: results are bitwise
//     repeatable.
#include <cuda_bf16.h>

#include "tc_common.cuh"

namespace gifb200 {

namespace {

constexpr int kMaxK = 7;
constexpr int kChunk = 32;          // input channels per pipeline stage (one 128-byte swizzle row of fp32)
constexpr int kBM = 128;            // output pixels per tensor-core tile
constexpr int kStages = 4;
constexpr int kThreads = 256;       // two warpgroups

struct ExParams {
    int B, Hi, Wi, Ci, Ho, Wo, Co, kh, kw, stride, pad_h, pad_w, Cy, c0;
    int M;                          // B * Ho * Wo
    ConvEpilogue epi;
};

// ----------------------------------------------------------------------------------------------- SIMT (exact fp32)
constexpr int SBM = 64, SBN = 64, SBK = 16;

__global__ void __launch_bounds__(256) conv_ex_simt_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                           float* __restrict__ y, ExParams p) {
    __shared__ float As[SBK][SBM + 4];
    __shared__ float Bs[SBK][SBN + 4];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.x * SBM, n0 = blockIdx.y * SBN;
    // load roles: A pixel tid/4 with channels (tid%4)*4..+3 of the chunk; B output channel tid/4, same channels
    const int a_row = tid >> 2, a_c = (tid & 3) << 2;
    const int a_m = m0 + a_row;
    int a_b = 0, a_yo = 0, a_xo = 0;
    const bool a_ok = a_m < p.M;
    if (a_ok) { a_xo = a_m % p.Wo; a_yo = (a_m / p.Wo) % p.Ho; a_b = a_m / (p.Wo * p.Ho); }
    const int b_o = n0 + a_row;
    // compute role: pixels ty*4..+3, channels tx*4..+3
    const int tx = tid & 15, ty = tid >> 4;
    float acc[4][4] = {};
    const int T = p.kh * p.kw;
    for (int t = 0; t < T; ++t) {
        const int yi = a_yo * p.stride - p.pad_h + t / p.kw, xi = a_xo * p.stride - p.pad_w + t % p.kw;
        const bool in = a_ok && yi >= 0 && yi < p.Hi && xi >= 0 && xi < p.Wi;
        const float* xp = x + ((static_cast<long long>(a_b) * p.Hi + yi) * p.Wi + xi) * p.Ci;
        const float* wp = w + (static_cast<long long>(t) * p.Co + b_o) * p.Ci;
        for (int c = 0; c < p.Ci; c += SBK) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int ci = c + a_c + j;
                As[a_c + j][a_row] = (in && ci < p.Ci) ? xp[ci] : 0.f;
                Bs[a_c + j][a_row] = (b_o < p.Co && ci < p.Ci) ? wp[ci] : 0.f;
            }
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < SBK; ++kk) {
                float a[4], b[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
            }
            __syncthreads();
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= p.M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int o = n0 + tx * 4 + j;
            if (o < p.Co) y[static_cast<long long>(m) * p.Cy + p.c0 + o] = apply_epilogue(p.epi, acc[i][j], o);
        }
    }
}

// ----------------------------------------------------------------------------------------------- tensor cores
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int BN>
struct ExCfg {
    static constexpr int kATileBytes = kBM * kChunk * 4;           // 16 KB (X3: hi tile, then lo tile, 8 KB each)
    static constexpr int kBTileBytes = BN * kChunk * 4;
    static constexpr int kStageBytes = kATileBytes + kBTileBytes;
    static constexpr int kDynamic = kStages * kStageBytes + 1024;  // slack for manual 1024 B alignment
    static constexpr int kMinBlocks = BN <= 64 ? 2 : 1;
};

// grid: (M tiles, Co / BN, ksplit).  part != nullptr: write the raw accumulators of split blockIdx.z to
// part[z][m][o] (dense, Co channels); the reduction pass applies the epilogue.
template <int BN, bool X3>
__global__ void __launch_bounds__(kThreads, ExCfg<BN>::kMinBlocks)
    conv_ex_tc_kernel(const void* __restrict__ xv, const void* __restrict__ wv, float* __restrict__ y, float* __restrict__ part,
                      const ExParams p, const long long x_plane, const long long w_plane) {
    using L = ExCfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    const uint32_t sbase = smem_u32(smem);
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * BN;
    const int kchunks = p.Ci / kChunk;
    const int iters = p.kh * p.kw * kchunks;
    const int it0 = static_cast<int>(static_cast<long long>(iters) * blockIdx.z / gridDim.z);
    const int it1 = static_cast<int>(static_cast<long long>(iters) * (blockIdx.z + 1) / gridDim.z);

    // A gather role: tile row tid/2.  fp32: 16-byte chunks (tid&1)*4..+3 of the 128-byte row.  X3: plane tid&1, the four
    // chunks of its 64-byte row.
    const int a_row = tid >> 1;
    const int a_m = m0 + a_row;
    const bool a_ok = a_m < p.M;
    int a_b = 0, a_yo = 0, a_xo = 0;
    if (a_ok) { a_xo = a_m % p.Wo; a_yo = (a_m / p.Wo) % p.Ho; a_b = a_m / (p.Wo * p.Ho); }
    const int a_iy0 = a_yo * p.stride - p.pad_h, a_ix0 = a_xo * p.stride - p.pad_w;
    constexpr int es = X3 ? 2 : 4;
    const char* xb = static_cast<const char*>(xv) + (X3 ? (tid & 1) * x_plane * es : 0) +
                     static_cast<long long>(a_b) * p.Hi * p.Wi * p.Ci * es;
    const char* wb = static_cast<const char*>(wv);

    auto load_stage = [&](int it, int slot) {
        const int tap = it / kchunks, cc = (it - tap * kchunks) * kChunk;
        const int iy = a_iy0 + tap / p.kw, ix = a_ix0 + tap % p.kw;
        const bool in = a_ok && iy >= 0 && iy < p.Hi && ix >= 0 && ix < p.Wi;
        const char* src = xb + ((static_cast<long long>(in ? iy : 0) * p.Wi + (in ? ix : 0)) * p.Ci + cc) * es;
        const uint32_t a_dst = sbase + slot * L::kStageBytes;
        if (X3) {
            const uint32_t row = a_dst + (tid & 1) * (L::kATileBytes / 2) + a_row * 64;
#pragma unroll
            for (int c = 0; c < 4; ++c) cp_async16(row + ((c ^ ((a_row >> 1) & 3)) << 4), src + c * 16, in);
        } else {
            const uint32_t row = a_dst + a_row * 128;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int c = (tid & 1) * 4 + j;
                cp_async16(row + ((c ^ (a_row & 7)) << 4), src + c * 16, in);
            }
        }
        const uint32_t b_dst = a_dst + L::kATileBytes;
#pragma unroll
        for (int j = 0; j < BN / 32; ++j) {
            const int idx = tid + kThreads * j;
            if (X3) {
                const int plane = idx / (BN * 4), rem = idx % (BN * 4), r = rem >> 2, c = rem & 3;
                const char* s = wb + (plane * w_plane + (static_cast<long long>(tap) * p.Co + n0 + r) * p.Ci + cc) * es + c * 16;
                cp_async16(b_dst + plane * (L::kBTileBytes / 2) + r * 64 + ((c ^ ((r >> 1) & 3)) << 4), s, true);
            } else {
                const int r = idx >> 3, c = idx & 7;
                const char* s = wb + ((static_cast<long long>(tap) * p.Co + n0 + r) * p.Ci + cc) * es + c * 16;
                cp_async16(b_dst + r * 128 + ((c ^ (r & 7)) << 4), s, true);
            }
        }
    };

#pragma unroll
    for (int s = 0; s < kStages - 1; ++s) {
        if (it0 + s < it1) load_stage(it0 + s, s);
        cp_async_commit();
    }
    const int wg = warp >> 2;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int it = it0; it < it1; ++it) {
        const int slot = (it - it0) % kStages;
        cp_async_wait<kStages - 2>();
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // cp.async (generic proxy) -> wgmma (async proxy)
        __syncthreads();
        const uint32_t a_addr = sbase + slot * L::kStageBytes;
        wgmma_fence();
        fence_regs<BN / 2>(acc);
        if (X3) {
            const uint32_t a_wg = a_addr + wg * 64 * 64;
            const uint64_t ah = make_kmajor_sw64_desc(a_wg), al = make_kmajor_sw64_desc(a_wg + L::kATileBytes / 2);
            const uint64_t bh = make_kmajor_sw64_desc(a_addr + L::kATileBytes);
            const uint64_t bl = make_kmajor_sw64_desc(a_addr + L::kATileBytes + L::kBTileBytes / 2);
#pragma unroll
            for (int k = 0; k < kChunk / 16; ++k) {
                wgmma_bf16<BN>(acc, al + 2 * k, bh + 2 * k, 1, Trans<0>());
                wgmma_bf16<BN>(acc, ah + 2 * k, bl + 2 * k, 1, Trans<0>());
                wgmma_bf16<BN>(acc, ah + 2 * k, bh + 2 * k, 1, Trans<0>());
            }
        } else {
            const uint64_t adesc = make_kmajor_sw128_desc(a_addr + wg * 64 * 128);
            const uint64_t bdesc = make_kmajor_sw128_desc(a_addr + L::kATileBytes);
#pragma unroll
            for (int k = 0; k < kChunk / 8; ++k) wgmma_tf32<BN>(acc, adesc + 2 * k, bdesc + 2 * k, 1);
        }
        wgmma_commit();
        // refill the slot of iteration it-1: every warpgroup retired its MMAs on it before the barrier above
        const int next = it + kStages - 1;
        if (next < it1) load_stage(next, (next - it0) % kStages);
        cp_async_commit();
        wgmma_wait<0>();
        fence_regs<BN / 2>(acc);
    }
    cp_async_wait<0>();
    // epilogue: accumulator fragment -> channels-last rows (8-byte stores)
    const int wq = warp & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = m0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
        if (m >= p.M) continue;
        const int o0 = n0 + 2 * (lane & 3);
        float* dst = part ? part + (static_cast<long long>(blockIdx.z) * p.M + m) * p.Co + o0
                          : y + static_cast<long long>(m) * p.Cy + p.c0 + o0;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            float2 v = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            if (!part) {
                v.x = apply_epilogue(p.epi, v.x, o0 + 8 * j);
                v.y = apply_epilogue(p.epi, v.y, o0 + 8 * j + 1);
            }
            *reinterpret_cast<float2*>(dst + 8 * j) = v;
        }
    }
}

// y[m, c0+o] = epilogue(sum_s part[s][m][o]) in split order; one thread per output pair
__global__ void __launch_bounds__(256) conv_ex_reduce_kernel(const float* __restrict__ part, float* __restrict__ y, ExParams p,
                                                             int ksplit) {
    const long long n2 = static_cast<long long>(p.M) * p.Co / 2;
    const long long stride = static_cast<long long>(p.M) * p.Co;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n2;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        float2 a = reinterpret_cast<const float2*>(part)[i];
        for (int s = 1; s < ksplit; ++s) {
            const float2 b = reinterpret_cast<const float2*>(part + s * stride)[i];
            a.x += b.x; a.y += b.y;
        }
        const long long m = (2 * i) / p.Co;
        const int o = static_cast<int>(2 * i - m * p.Co);
        a.x = apply_epilogue(p.epi, a.x, o);
        a.y = apply_epilogue(p.epi, a.y, o + 1);
        *reinterpret_cast<float2*>(y + m * p.Cy + p.c0 + o) = a;
    }
}

// [T][Co][Ci] fp32 weights -> tf32-rounded copy, or (X3) two bf16 planes [2][T][Co][Ci] in the same number of bytes
template <bool X3>
__global__ void __launch_bounds__(256) conv_ex_stage_kernel(const float* __restrict__ w, void* __restrict__ out, long long n) {
    for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const float v = w[e];
        if (X3) {
            __nv_bfloat16* planes = static_cast<__nv_bfloat16*>(out);
            const __nv_bfloat16 h = __float2bfloat16_rn(v);
            planes[e] = h;
            planes[n + e] = __float2bfloat16_rn(v - __bfloat162float(h));
        } else {
            static_cast<float*>(out)[e] = round_tf32(v);
        }
    }
}

int pick_bn(int Co) { return Co % 128 == 0 ? 128 : (Co % 64 == 0 ? 64 : 32); }

// K splits when the output tiles fill less than half of the SMs: enough splits for about one wave, at least 4 stages each
int pick_ksplit_ex(long long tiles, int iters) {
    if (tiles * 2 > kNumSMs || iters < 8) return 1;
    long long ks = kNumSMs / tiles;
    if (ks > iters / 4) ks = iters / 4;
    if (ks > 16) ks = 16;
    return ks < 2 ? 1 : static_cast<int>(ks);
}

bool geometry_ok(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int kh, int kw, int stride, int pad_h, int pad_w,
                 int Cy, int c0) {
    if (B <= 0 || Hi <= 0 || Wi <= 0 || Ci <= 0 || Ho <= 0 || Wo <= 0 || Co <= 0) return false;
    if (kh < 1 || kw < 1 || kh > kMaxK || kw > kMaxK || (stride != 1 && stride != 2) || pad_h < 0 || pad_w < 0) return false;
    if (c0 < 0 || c0 + Co > Cy) return false;
    // every output pixel sees at least its top-left tap's row / column range inside the padded input
    if ((Ho - 1) * stride + kh > Hi + 2 * pad_h || (Wo - 1) * stride + kw > Wi + 2 * pad_w) return false;
    return static_cast<long long>(B) * Ho * Wo < 2147483647LL / 2;
}

bool tc_ok(int Ci, int Co, int Cy, int c0) { return Ci % kChunk == 0 && Co % 32 == 0 && Cy % 2 == 0 && c0 % 2 == 0; }

size_t staged_bytes(int Ci, int Co, int kh, int kw) {
    return (static_cast<size_t>(kh) * kw * Co * Ci * sizeof(float) + 255) / 256 * 256;
}

int ksplit_of(int B, int Ho, int Wo, int Ci, int Co, int kh, int kw) {
    const long long mtiles = (static_cast<long long>(B) * Ho * Wo + kBM - 1) / kBM;
    return pick_ksplit_ex(mtiles * (Co / pick_bn(Co)), kh * kw * (Ci / kChunk));
}

template <int BN, bool X3>
int launch_ex(const void* x, const void* w, float* y, float* part, const ExParams& p, int ksplit, long long x_plane,
              long long w_plane, cudaStream_t st) {
    using L = ExCfg<BN>;
    static bool attr_set = false;   // per-process, idempotent
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(conv_ex_tc_kernel<BN, X3>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kDynamic);
        if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "cudaFuncSetAttribute(conv_ex_tc_kernel)", cudaGetErrorString(e));
        attr_set = true;
    }
    const dim3 grid(static_cast<unsigned>((p.M + kBM - 1) / kBM), static_cast<unsigned>(p.Co / BN), static_cast<unsigned>(ksplit));
    conv_ex_tc_kernel<BN, X3><<<grid, kThreads, L::kDynamic, st>>>(x, w, y, part, p, x_plane, w_plane);
    GIFB200_LAUNCH_CHECK("conv_ex_tc_kernel");
    return GIFB200_OK;
}

template <bool X3>
int launch_ex_bn(const void* x, const void* w, float* y, float* part, const ExParams& p, int ksplit, long long x_plane,
                 long long w_plane, cudaStream_t st) {
    switch (pick_bn(p.Co)) {
        case 128: return launch_ex<128, X3>(x, w, y, part, p, ksplit, x_plane, w_plane, st);
        case 64: return launch_ex<64, X3>(x, w, y, part, p, ksplit, x_plane, w_plane, st);
        default: return launch_ex<32, X3>(x, w, y, part, p, ksplit, x_plane, w_plane, st);
    }
}

}  // namespace

}  // namespace gifb200

using namespace gifb200;

extern "C" size_t gifb200_conv2d_ex_workspace_bytes(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int kh, int kw,
                                                    int stride, int pad_h, int pad_w, int impl) {
    impl &= 0xF;
    if (impl == 1 || !geometry_ok(B, Hi, Wi, Ci, Ho, Wo, Co, kh, kw, stride, pad_h, pad_w, Co, 0) || !tc_ok(Ci, Co, Co, 0))
        return 0;
    size_t bytes = staged_bytes(Ci, Co, kh, kw);
    const int ks = ksplit_of(B, Ho, Wo, Ci, Co, kh, kw);
    if (ks > 1) bytes += static_cast<size_t>(ks) * B * Ho * Wo * Co * sizeof(float);
    return bytes + 256;
}

extern "C" int gifb200_conv2d_ex(const void* x, const float* w, float* y, int B, int Hi, int Wi, int Ci, int Ho, int Wo,
                                 int Co, int kh, int kw, int stride, int pad_h, int pad_w, int Cy, int c0, int impl, int act,
                                 const float* bias, int round_tf32, void* workspace, size_t workspace_bytes,
                                 gifb200_stream_t stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool prestaged = (impl & GIFB200_CONV_PRESTAGED) != 0;
    impl &= 0xF;
    GIFB200_REQUIRE(impl >= 0 && impl <= 3, GIFB200_E_SHAPE,
                    "conv2d_ex: impl must be 0 (auto), 1 (simt), 2 (wgmma tf32) or 3 (wgmma bf16x3 on split planes)");
    GIFB200_REQUIRE(geometry_ok(B, Hi, Wi, Ci, Ho, Wo, Co, kh, kw, stride, pad_h, pad_w, Cy, c0), GIFB200_E_SHAPE,
                    "conv2d_ex: unsupported geometry (kh, kw <= 7, stride 1 or 2, pads >= 0, c0 + Co <= Cy, Ho / Wo within "
                    "the padded input)");
    ExParams p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.Hi = Hi; p.Wi = Wi; p.Ci = Ci; p.Ho = Ho; p.Wo = Wo; p.Co = Co; p.kh = kh; p.kw = kw; p.stride = stride;
    p.pad_h = pad_h; p.pad_w = pad_w; p.Cy = Cy; p.c0 = c0; p.M = B * Ho * Wo;
    p.epi = ConvEpilogue{act, bias, 0.f, 1.f, round_tf32};
    const bool tc = tc_ok(Ci, Co, Cy, c0);
    if (impl >= 2 && !tc)
        return fail(GIFB200_E_SHAPE, "conv2d_ex: the tensor-core path needs Ci % 32 == 0, Co % 32 == 0 and an even Cy / c0");
    if (impl == 1 || !tc) {
        const dim3 grid(static_cast<unsigned>((p.M + SBM - 1) / SBM), static_cast<unsigned>((Co + SBN - 1) / SBN));
        conv_ex_simt_kernel<<<grid, 256, 0, st>>>(static_cast<const float*>(x), w, y, p);
        GIFB200_LAUNCH_CHECK("conv_ex_simt_kernel");
        return GIFB200_OK;
    }
    const bool x3 = impl == 3;
    GIFB200_REQUIRE(workspace && workspace_bytes >= gifb200_conv2d_ex_workspace_bytes(B, Hi, Wi, Ci, Ho, Wo, Co, kh, kw, stride,
                                                                                       pad_h, pad_w, impl),
                    GIFB200_E_WORKSPACE, "conv2d_ex: workspace too small (see gifb200_conv2d_ex_workspace_bytes)");
    GIFB200_REQUIRE(aligned16(x) && (reinterpret_cast<uintptr_t>(y) & 7u) == 0, GIFB200_E_ALIGN,
                    "conv2d_ex: x must be 16-byte and y 8-byte aligned");
    char* wst = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~static_cast<uintptr_t>(255));
    const long long nw = static_cast<long long>(kh) * kw * Co * Ci;
    if (!prestaged) {
        int blocks = cdiv(nw, 256 * 4);
        if (blocks > kNumSMs * 4) blocks = kNumSMs * 4;
        if (x3) conv_ex_stage_kernel<true><<<blocks, 256, 0, st>>>(w, wst, nw);
        else conv_ex_stage_kernel<false><<<blocks, 256, 0, st>>>(w, wst, nw);
        GIFB200_LAUNCH_CHECK("conv_ex_stage_kernel");
    }
    const int ks = ksplit_of(B, Ho, Wo, Ci, Co, kh, kw);
    float* part = ks > 1 ? reinterpret_cast<float*>(wst + staged_bytes(Ci, Co, kh, kw)) : nullptr;
    const long long x_plane = static_cast<long long>(B) * Hi * Wi * Ci;
    const int rc = x3 ? launch_ex_bn<true>(x, wst, y, part, p, ks, x_plane, nw, st)
                      : launch_ex_bn<false>(x, wst, y, part, p, ks, x_plane, nw, st);
    if (rc != GIFB200_OK || ks == 1) return rc;
    const long long n2 = static_cast<long long>(p.M) * Co / 2;
    int blocks = cdiv(n2, 256);
    if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
    conv_ex_reduce_kernel<<<blocks, 256, 0, st>>>(part, y, p, ks);
    GIFB200_LAUNCH_CHECK("conv_ex_reduce_kernel");
    return GIFB200_OK;
}
