// wgmma implicit-GEMM convolution for sm_90a (tf32 operands, fp32 accumulation in registers).
//
// GEMM view (per output "phase"):  D[site, o] = sum_{tap} sum_{i} A_tap[site, i] * W[tap][o][i]
//   M = 128 sites per CTA (a wt x ht x nt box of the site grid (B, Hs, Ws)), N = BLOCK_N output channels,
//   K = 32 input channels per pipeline stage (one 128-byte swizzle row of fp32), taps x Ci/32 stages per tile.
//   * A operand: the activation tensor itself (channels-last fp32) -- no im2col buffer.  Each tap is the same TMA box
//     shifted by the tap offset; TMA's out-of-bounds zero fill implements the padding.  Stride-2 convolutions (S2)
//     read through a 5-D view that splits W into (parity, W/2) and load one site row per TMA issue; transposed
//     stride-2 convolutions (T2) run as 4 output phases (Y%2, X%2), each an ordinary stride-1 gather with its own
//     subset of the 9 taps, and write with output stride 2.
//   * B operand: the tap-major weights [T][Co][Ci] staged once per call into the workspace (honouring flip /
//     transposed, rounded to tf32), K-major, 128B swizzle.
//   * Both operands are K-major SWIZZLE_128B; each of two consumer warpgroups issues one wgmma.m64nNk8.tf32 (its 64 rows
//     of the tile, N = BLOCK_N) per 32-byte K slice; accumulators live in registers (BLOCK_N / 2 per thread).
//   * Warp roles (288 threads): warps 0-7 two consumer warpgroups (MMA + fused epilogue from registers, 8-byte global
//     stores, channels-last), warp 8 TMA producer.
//   * 3-stage smem ring (96 KB) so that two CTAs share an SM: one CTA's epilogue overlaps the other's main loop.
//
// Operand precision: the tf32 MMA reads the upper 19 bits of each fp32 (truncation).  Callers hand in activations that
// are already rounded to tf32 (gif_b200.ops rounds in the producing kernel), weights are rounded here, so the
// truncation is exact and the contraction is an unbiased tf32 x tf32 -> fp32 product sum.
//
// X3 = true is the error-compensated mode ("bf16x3", gifb200_conv2d impl 3): operands arrive as two bf16 planes (hi, lo)
// per tensor (gifb200_split_bf16; the weights are split while staging), a stage holds the hi and the lo tile of A and of B
// as K-major SWIZZLE_64B tiles of 32 channels (128 rows x 64 B: the SAME number of bytes per stage as the fp32 tiles), and
// each 16-channel slice issues three bf16 wgmmas -- lo*hi, hi*lo, hi*hi -- into the one fp32 register accumulator.
// Everything else (tile walk, ring, epilogue) is shared with the tf32 kernel.
#include <cuda_bf16.h>

#include "tc_common.cuh"

namespace gifb200 {

namespace {

constexpr int kStages = 3;
constexpr int kBlockM = 128;
constexpr int kBlockK = 32;                         // fp32 elements = 128 bytes = one swizzle row
constexpr int kATileBytes = kBlockM * kBlockK * 4;  // 16 KB
constexpr int kMaxTaps = 9;
constexpr int kConsumerWarps = 8;                   // two warpgroups: rows 0-63 and 64-127 of the tile
constexpr int kTcThreads = 32 * kConsumerWarps + 32;   // + one TMA producer warp

struct TcParams {
    int B, Hs, Ws;          // site grid per image
    int wt, ht, nt;         // tile box (wt*ht*nt == 128)
    int tiles_x, tiles_y;   // tiles per image group
    int Ci, Co;
    int s2;                 // 1: A loads go through the 5-D parity view, one site row per TMA issue
    int Ho, Wo;             // output tensor spatial size
    int oys, oxs;           // output pixel = site * o?s + o?0
    int nphase;
    int phase_oy0[4], phase_ox0[4], phase_ntaps[4];
    int tap_w[4][kMaxTaps];     // weight tap index (into the staged [T][Co][Ci] buffer)
    int tap_dy[4][kMaxTaps];    // input row    = site_y * in_sy + tap_dy
    int tap_dx[4][kMaxTaps];    // input column = site_x + tap_dx        (S2: column in the W/2 space)
    int tap_par[4][kMaxTaps];   // S2: W parity plane
    int in_sy;
    int ksplit;             // > 1: the K loop (taps x channel chunks) of every tile is cut into ksplit ranges, one tile each,
    float* part;            //      whose accumulators go to part[ks][...] (same indexing as y); splitk_reduce_kernel sums them
    long long part_stride;  //      in a fixed order and applies the epilogue (small layers: 16 output tiles cannot fill 132 SMs)
    ConvEpilogue epi;
};

template <int BLOCK_N>
struct SmemLayout {
    static constexpr int kBTileBytes = BLOCK_N * kBlockK * 4;
    static constexpr int kStageBytes = kATileBytes + kBTileBytes;
    static constexpr int kBarrierOffset = kStages * kStageBytes;
    static constexpr int kTotal = kBarrierOffset + 64;    // full[3], empty[3]
    static constexpr int kDynamic = kTotal + 1024;        // slack for manual 1024 B alignment
};

// Tile order: (output-channel block, phase) vary FASTEST, the site tile slowest, so that the CTAs running at the same
// time read the same activation boxes and the re-reads (once per channel block, per phase, per tap) hit L2 instead of
// DRAM.  Phases have 4/2/2/1 taps; the phase a CTA gets is rotated from round to round (rot = (mtile / rot_div) % nphase,
// a function of the site tile only, hence still a bijection) so every CTA sees all phases equally often.
__device__ __forceinline__ void decode_tile(int tile, int nblocks, int nphase, int rot_div, int& mt, int& nblk, int& phase) {
    const int inner = nblocks * nphase;
    mt = tile / inner;
    const int rem = tile - mt * inner;
    nblk = rem % nblocks;
    phase = nphase == 1 ? 0 : (rem / nblocks + mt / rot_div) % nphase;
}

// Persistent: gridDim.x CTAs (<= 2 per SM) walk the tile list (see decode_tile).  Warps 0-7 are two consumer warpgroups
// (wgmma into register accumulators, then the fused epilogue straight from registers), warp 8 is the TMA producer.  The
// smem ring and its phase bits run continuously across tiles; the second resident CTA overlaps its main loop with this
// CTA's epilogue.
template <int BLOCK_N, bool X3>
__global__ void __launch_bounds__(kTcThreads, 2) conv_tc_kernel(const __grid_constant__ CUtensorMap map_a,
                                                         const __grid_constant__ CUtensorMap map_a2,
                                                         const __grid_constant__ CUtensorMap map_b,
                                                         const __grid_constant__ CUtensorMap map_b2,
                                                         float* __restrict__ y, const TcParams p, const int mtiles,
                                                         const int total_tiles) {
    using L = SmemLayout<BLOCK_N>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarrierOffset);
    uint64_t* empty_bar = full_bar + kStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nblocks = p.Co / BLOCK_N;
    const int kchunks = p.Ci / kBlockK;
    const int rot_div = max(1, static_cast<int>(gridDim.x) / (nblocks * p.nphase));
    (void)mtiles;

    if (warp == kConsumerWarps && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
        if (X3) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a2) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b2) : "memory");
        }
        for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();

    if (warp == kConsumerWarps) {
        // ===================== TMA producer =====================
        // Lane 0 owns the barriers.  In stride-2 row mode the A tile is nt*ht separate row boxes (the parity view cannot be
        // one box): the 32 lanes issue them in parallel.
        int stage = 0;
        uint32_t ph = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            int mt, nblk, phase;
            const int ks = tile % p.ksplit;
            decode_tile(tile / p.ksplit, nblocks, p.nphase, rot_div, mt, nblk, phase);
            int m = mt;
            const int tx = m % p.tiles_x; m /= p.tiles_x;
            const int ty = m % p.tiles_y; m /= p.tiles_y;
            const int n0 = m * p.nt, y0 = ty * p.ht, x0 = tx * p.wt;
            const int iters = p.phase_ntaps[phase] * kchunks;
            const int it0 = iters * ks / p.ksplit, it1 = iters * (ks + 1) / p.ksplit;      // the whole loop when ksplit == 1
            for (int it = it0; it < it1; ++it) {
                const int tap = it / kchunks, c0 = (it % kchunks) * kBlockK;
                uint8_t* a_dst = smem + stage * L::kStageBytes;
                uint8_t* b_dst = a_dst + kATileBytes;
                if (lane == 0) {
                    mbar_wait(&empty_bar[stage], ph ^ 1);
                    mbar_expect_tx(&full_bar[stage], L::kStageBytes);
                }
                __syncwarp();
                const int dy = p.tap_dy[phase][tap], dx = p.tap_dx[phase][tap];
                // X3: the hi plane's tile fills the first half of the A (B) slot, the lo plane's tile the second half
                if (!p.s2) {
                    if (lane == 0) {
                        tma_load_4d(a_dst, &map_a, &full_bar[stage], c0, x0 + dx, y0 + dy, n0);
                        if (X3) tma_load_4d(a_dst + kATileBytes / 2, &map_a2, &full_bar[stage], c0, x0 + dx, y0 + dy, n0);
                    }
                } else if (p.s2 == 2) {
                    // the nt x ht rows of the tile through ONE 5-D box per plane: traversal stride 2 along the input rows
                    if (lane == 0) {
                        const int par = p.tap_par[phase][tap];
                        tma_load_5d(a_dst, &map_a, &full_bar[stage], c0, par, x0 + dx, y0 * p.in_sy + dy, n0);
                        if (X3) tma_load_5d(a_dst + kATileBytes / 2, &map_a2, &full_bar[stage], c0, par, x0 + dx, y0 * p.in_sy + dy, n0);
                    }
                } else {
                    const int par = p.tap_par[phase][tap];
                    const int row_bytes = p.wt * kBlockK * (X3 ? 2 : 4);
                    const int rows = p.nt * p.ht;
                    for (int r = lane; r < rows; r += 32) {
                        const int n = r / p.ht, h = r - n * p.ht;
                        tma_load_5d(a_dst + r * row_bytes, &map_a, &full_bar[stage], c0, par, x0 + dx,
                                    (y0 + h) * p.in_sy + dy, n0 + n);
                        if (X3)
                            tma_load_5d(a_dst + kATileBytes / 2 + r * row_bytes, &map_a2, &full_bar[stage], c0, par, x0 + dx,
                                        (y0 + h) * p.in_sy + dy, n0 + n);
                    }
                }
                if (lane == 0) {
                    tma_load_3d(b_dst, &map_b, &full_bar[stage], c0, nblk * BLOCK_N, p.tap_w[phase][tap]);
                    if (X3) tma_load_3d(b_dst + L::kBTileBytes / 2, &map_b2, &full_bar[stage], c0, nblk * BLOCK_N, p.tap_w[phase][tap]);
                }
                if (++stage == kStages) { stage = 0; ph ^= 1; }
            }
        }
    } else {
        // ===================== consumers: wgmma main loop + epilogue =====================
        const int wg = warp >> 2;                    // rows 64*wg .. 64*wg+63 of the tile
        const int wq = warp & 3;
        constexpr int kAcc = BLOCK_N / 2;
        float acc[kAcc];
        // the two rows (h = 0, 1) this thread holds in the accumulator fragment, and their place in the site box
        int w_in[2], h_in[2], n_in[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
            w_in[h] = r % p.wt; h_in[h] = (r / p.wt) % p.ht; n_in[h] = r / (p.wt * p.ht);
        }
        int stage = 0;
        uint32_t ph = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            int mt, nblk, phase;
            const int ks = tile % p.ksplit;
            decode_tile(tile / p.ksplit, nblocks, p.nphase, rot_div, mt, nblk, phase);
            const int iters = p.phase_ntaps[phase] * kchunks;
            const int it0 = iters * ks / p.ksplit, it1 = iters * (ks + 1) / p.ksplit;
            int prev = -1;
            for (int it = it0; it < it1; ++it) {
                mbar_wait(&full_bar[stage], ph);
                const uint32_t a_addr = smem_u32(smem + stage * L::kStageBytes);
                wgmma_fence();
                fence_regs<kAcc>(acc);
                if (X3) {
                    // v = hi + lo per operand: acc += a_lo*b_hi + a_hi*b_lo + a_hi*b_hi (the 2^-18 lo*lo term is dropped);
                    // small terms first.  K = 16 bf16 = 32 bytes: two slices per 32-channel stage.  A rows of 64 B.
                    const uint32_t a_wg = a_addr + wg * 64 * 64;
                    const uint64_t ah = make_kmajor_sw64_desc(a_wg), al = make_kmajor_sw64_desc(a_wg + kATileBytes / 2);
                    const uint64_t bh = make_kmajor_sw64_desc(a_addr + kATileBytes);
                    const uint64_t bl = make_kmajor_sw64_desc(a_addr + kATileBytes + L::kBTileBytes / 2);
#pragma unroll
                    for (int k = 0; k < kBlockK / 16; ++k) {
                        wgmma_bf16<BLOCK_N>(acc, al + 2 * k, bh + 2 * k, (it != it0) || k != 0, Trans<0>());
                        wgmma_bf16<BLOCK_N>(acc, ah + 2 * k, bl + 2 * k, 1, Trans<0>());
                        wgmma_bf16<BLOCK_N>(acc, ah + 2 * k, bh + 2 * k, 1, Trans<0>());
                    }
                } else {
                    const uint64_t adesc = make_kmajor_sw128_desc(a_addr + wg * 64 * 128);
                    const uint64_t bdesc = make_kmajor_sw128_desc(a_addr + kATileBytes);
#pragma unroll
                    for (int k = 0; k < kBlockK / 8; ++k)   // K = 8 tf32 = 32 bytes: advance the start address by 32 B (>>4 = 2)
                        wgmma_tf32<BLOCK_N>(acc, adesc + 2 * k, bdesc + 2 * k, (it != it0) || k != 0);
                }
                wgmma_commit();
                fence_regs<kAcc>(acc);
                // keep this stage's MMAs in flight; the previous stage's have retired -> its smem slot is free
                wgmma_wait<1>();
                if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
                prev = stage;
                if (++stage == kStages) { stage = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            fence_regs<kAcc>(acc);
            if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
            // ---- epilogue: registers -> channels-last global (split-K: this split's partial buffer, epilogue deferred)
            int m = mt;
            const int tx = m % p.tiles_x; m /= p.tiles_x;
            const int ty = m % p.tiles_y; m /= p.tiles_y;
            float* base = p.ksplit > 1 ? p.part + ks * p.part_stride : y;
            const int c0 = nblk * BLOCK_N + 2 * (lane & 3);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int n = m * p.nt + n_in[h];
                const int Y = (ty * p.ht + h_in[h]) * p.oys + p.phase_oy0[phase], X = (tx * p.wt + w_in[h]) * p.oxs + p.phase_ox0[phase];
                if (n < p.B && Y < p.Ho && X < p.Wo) {
                    float* dst = base + ((static_cast<long long>(n) * p.Ho + Y) * p.Wo + X) * p.Co + c0;
#pragma unroll
                    for (int j = 0; j < BLOCK_N / 8; ++j) {
                        float2 v = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                        if (p.epi.act && p.ksplit == 1) {      // split-K: the reduction pass applies the epilogue to the sum
                            v.x = apply_epilogue(p.epi, v.x, c0 + 8 * j);
                            v.y = apply_epilogue(p.epi, v.y, c0 + 8 * j + 1);
                        }
                        *reinterpret_cast<float2*>(dst + 8 * j) = v;
                    }
                }
            }
        }
    }
}

// stage logical weights W[t][o][i] (from the physical buffer + flip/transposed) as [T][Co][Ci], rounded to tf32;
// X3: as two bf16 planes [2][T][Co][Ci] (hi, lo) in the same number of bytes
template <bool X3>
__global__ void __launch_bounds__(256) stage_weights_kernel(const float* __restrict__ w, float* __restrict__ out, int T,
                                                            int Co, int Ci, int flip, int transposed) {
    const long long total = static_cast<long long>(T) * Co * Ci;
    for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int i = static_cast<int>(e % Ci);
        const int o = static_cast<int>((e / Ci) % Co);
        const int t = static_cast<int>(e / (static_cast<long long>(Ci) * Co));
        const int tt = flip ? T - 1 - t : t;
        const float v = transposed ? w[(static_cast<long long>(tt) * Ci + i) * Co + o]
                                   : w[(static_cast<long long>(tt) * Co + o) * Ci + i];
        if (X3) {
            __nv_bfloat16* planes = reinterpret_cast<__nv_bfloat16*>(out);
            const __nv_bfloat16 h = __float2bfloat16_rn(v);
            planes[e] = h;
            planes[total + e] = __float2bfloat16_rn(v - __bfloat162float(h));
        } else {
            out[e] = round_tf32(v);
        }
    }
}

// y[e] = epilogue(sum_s part[s][e]) in split order (deterministic); n4 = elements / 4, Co % 4 == 0
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ part, float* __restrict__ y, long long n4,
                                                            int ksplit, long long stride, ConvEpilogue epi, int Co) {
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        float4 a = __ldcs(reinterpret_cast<const float4*>(part) + i);
        for (int s = 1; s < ksplit; ++s) {
            const float4 b = __ldcs(reinterpret_cast<const float4*>(part + s * stride) + i);
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        const int o = static_cast<int>((i * 4) % Co);
        a.x = apply_epilogue(epi, a.x, o); a.y = apply_epilogue(epi, a.y, o + 1);
        a.z = apply_epilogue(epi, a.z, o + 2); a.w = apply_epilogue(epi, a.w, o + 3);
        reinterpret_cast<float4*>(y)[i] = a;
    }
}

// K splits for a layer whose output tiles cannot fill the machine (4x4 / 8x8 layers at batch 32: 16-64 tiles, 144 pipeline
// iterations each: otherwise one CTA's TMA issue rate bounds the layer).  Stride-1 / stride-2 modes.
int pick_ksplit(long long tiles, int iters, int mode) {
    if (mode == 2 || tiles > kNumSMs / 2 || iters < 8) return 1;
    long long ks = (2LL * kNumSMs) / tiles;
    if (ks > iters / 4) ks = iters / 4;
    if (ks > 16) ks = 16;
    return ks < 2 ? 1 : static_cast<int>(ks);
}

void tile_geometry(int B, int Hs, int Ws, int& wt, int& ht, int& nt, long long& mtiles) {
    wt = Ws < 128 ? Ws : 128;
    ht = (128 / wt) < Hs ? (128 / wt) : Hs;
    nt = 128 / (wt * ht);
    mtiles = static_cast<long long>(Ws / wt) * (Hs / ht) * ((B + nt - 1) / nt);
}

// ----------------------------------------------------------------------------------------------- host side
inline bool pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

int pick_block_n(int Co) {
    if (Co % 128 == 0) return 128;
    if (Co % 64 == 0) return 64;
    if (Co % 32 == 0) return 32;
    return 0;
}

// T2 corner pixel (2*Hi, 2*Wi): only tap (2,2) on input pixel (Hi-1, Wi-1) reaches it.  One warp per (b, o), staged
// (tf32-rounded) weights like the tensor-core path.
// X3: xpix / w22 point into the hi planes; the lo planes lie x_plane / w_plane elements further.
template <bool X3>
__global__ void __launch_bounds__(256) t2_corner_kernel(const void* __restrict__ xpix_v, const void* __restrict__ w22_v,
                                                        float* __restrict__ y, int B, long long x_batch_stride, int Ci, int Co,
                                                        int Ho, int Wo, ConvEpilogue epi, long long x_plane, long long w_plane) {
    const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= static_cast<long long>(B) * Co) return;
    const int b = static_cast<int>(warp / Co), o = static_cast<int>(warp % Co);
    float a = 0.f;
    if (X3) {
        const __nv_bfloat16* xv = static_cast<const __nv_bfloat16*>(xpix_v) + b * x_batch_stride;
        const __nv_bfloat16* wv = static_cast<const __nv_bfloat16*>(w22_v) + static_cast<long long>(o) * Ci;
        for (int i = lane; i < Ci; i += 32)
            a = fmaf(__bfloat162float(xv[i]) + __bfloat162float(xv[x_plane + i]),
                     __bfloat162float(wv[i]) + __bfloat162float(wv[w_plane + i]), a);
    } else {
        const float* xv = static_cast<const float*>(xpix_v) + b * x_batch_stride;
        const float* wv = static_cast<const float*>(w22_v) + static_cast<long long>(o) * Ci;
        for (int i = lane; i < Ci; i += 32) a = fmaf(xv[i], wv[i], a);
    }
    a = warp_sum(a);
    if (lane == 0) y[((static_cast<long long>(b) * Ho + (Ho - 1)) * Wo + (Wo - 1)) * Co + o] = apply_epilogue(epi, a, o);
}

void site_grid(int Hi, int Wi, int Ho, int Wo, int mode, int& Hs, int& Ws) {
    if (mode == 2) { Hs = Hi; Ws = Wi; } else { Hs = Ho; Ws = Wo; }
}

template <int BLOCK_N, bool X3>
int launch(const CUtensorMap& ma, const CUtensorMap& ma2, const CUtensorMap& mb, const CUtensorMap& mb2, float* y,
           const TcParams& p, int mtiles, cudaStream_t st) {
    using L = SmemLayout<BLOCK_N>;
    static bool attr_set = false;   // per-process, idempotent
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<BLOCK_N, X3>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kDynamic);
        if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "cudaFuncSetAttribute(conv_tc_kernel)", cudaGetErrorString(e));
        attr_set = true;
    }
    const long long total = static_cast<long long>(mtiles) * (p.Co / BLOCK_N) * p.nphase * p.ksplit;
    if (total > 2147483647LL) return fail(GIFB200_E_SHAPE, "conv2d_tc: too many tiles");
    const int grid = total < 2 * kNumSMs ? static_cast<int>(total) : 2 * kNumSMs;   // persistent: <= 2 CTAs per SM
    conv_tc_kernel<BLOCK_N, X3><<<grid, kTcThreads, L::kDynamic, st>>>(ma, ma2, mb, mb2, y, p, mtiles, static_cast<int>(total));
    GIFB200_LAUNCH_CHECK("conv_tc_kernel");
    return GIFB200_OK;
}

int launch_any(int bn, bool x3, const CUtensorMap& ma, const CUtensorMap& ma2, const CUtensorMap& mb, const CUtensorMap& mb2,
               float* y, const TcParams& p, int mtiles, cudaStream_t st) {
    if (x3) {
        if (bn == 128) return launch<128, true>(ma, ma2, mb, mb2, y, p, mtiles, st);
        if (bn == 64) return launch<64, true>(ma, ma2, mb, mb2, y, p, mtiles, st);
        return launch<32, true>(ma, ma2, mb, mb2, y, p, mtiles, st);
    }
    if (bn == 128) return launch<128, false>(ma, ma2, mb, mb2, y, p, mtiles, st);
    if (bn == 64) return launch<64, false>(ma, ma2, mb, mb2, y, p, mtiles, st);
    return launch<32, false>(ma, ma2, mb, mb2, y, p, mtiles, st);
}

}  // namespace

bool conv2d_tc_supported(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode) {
    if (B <= 0 || Ci % 32 != 0 || pick_block_n(Co) == 0) return false;
    if (!(k == 3 || (k == 1 && mode == 0))) return false;
    if (mode == 0 && !(Ho == Hi && Wo == Wi)) return false;
    if (mode == 1 && !(Hi == 2 * Ho + 1 && Wi == 2 * Wo + 1)) return false;
    if (mode == 2 && !(Ho == 2 * Hi + 1 && Wo == 2 * Wi + 1)) return false;
    int Hs, Ws;
    site_grid(Hi, Wi, Ho, Wo, mode, Hs, Ws);
    if (!pow2(Hs) || !pow2(Ws) || Ws < 4 || Hs < 4 || Ws > 4096 || Hs > 4096) return false;
    return true;
}

static size_t staged_weight_bytes(int Ci, int Co, int k) {
    return (static_cast<size_t>(k) * k * Co * Ci * sizeof(float) + 256 + 255) / 256 * 256;
}

// split-K geometry of a supported shape: the number of splits (1 = none)
static int ksplit_of(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode) {
    int Hs, Ws, wt, ht, nt;
    long long mtiles;
    site_grid(Hi, Wi, Ho, Wo, mode, Hs, Ws);
    tile_geometry(B, Hs, Ws, wt, ht, nt, mtiles);
    const int bn = pick_block_n(Co);
    if (bn == 0) return 1;
    return pick_ksplit(mtiles * (Co / bn), k * k * (Ci / kBlockK), mode);
}

size_t conv2d_tc_workspace_bytes(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode, int) {
    size_t bytes = staged_weight_bytes(Ci, Co, k);
    if (conv2d_tc_supported(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode)) {
        const int ks = ksplit_of(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode);
        if (ks > 1) bytes += static_cast<size_t>(ks) * B * Ho * Wo * Co * sizeof(float) + 256;     // the partial accumulators
    }
    return bytes;
}

int conv2d_tc(const float* x, const float* w, float* y, int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k,
              int mode, int flip, int transposed, const ConvEpilogue& epi, void* ws, size_t ws_bytes, cudaStream_t st,
              bool x3, bool prestaged) {
    GIFB200_REQUIRE(conv2d_tc_supported(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode), GIFB200_E_SHAPE, "conv2d_tc: unsupported shape");
    GIFB200_REQUIRE(ws && ws_bytes >= conv2d_tc_workspace_bytes(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, transposed),
                    GIFB200_E_WORKSPACE, "conv2d_tc: workspace too small (see gifb200_conv2d_workspace_bytes)");
    GIFB200_REQUIRE(aligned16(x) && aligned16(y), GIFB200_E_ALIGN, "conv2d_tc: x / y must be 16-byte aligned");
    const int T = k * k;
    float* wst = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~static_cast<uintptr_t>(255));
    if (!prestaged) {     // prestaged: the caller kept the workspace of an earlier call with the same (w, flip, transposed, impl)
        const long long total = static_cast<long long>(T) * Co * Ci;
        int blocks = cdiv(total, 256 * 4);
        if (blocks > kNumSMs * 4) blocks = kNumSMs * 4;
        if (x3) stage_weights_kernel<true><<<blocks, 256, 0, st>>>(w, wst, T, Co, Ci, flip, transposed);
        else stage_weights_kernel<false><<<blocks, 256, 0, st>>>(w, wst, T, Co, Ci, flip, transposed);
        GIFB200_LAUNCH_CHECK("stage_weights_kernel");
    }
    // element size / tile geometry of the operand tensors: fp32 + 128-byte swizzle rows, or bf16 planes + 64-byte rows
    const cuuint64_t es = x3 ? 2 : 4;
    const CUtensorMapSwizzle swz = x3 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
    const CUtensorMapDataType dt = x3 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    const long long x_plane = static_cast<long long>(B) * Hi * Wi * Ci;       // elements between the hi and the lo plane
    const long long w_plane = static_cast<long long>(T) * Co * Ci;
    const char* xb = reinterpret_cast<const char*>(x);
    const char* wb = reinterpret_cast<const char*>(wst);
    TcParams p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.Ci = Ci; p.Co = Co; p.Ho = Ho; p.Wo = Wo; p.epi = epi;
    site_grid(Hi, Wi, Ho, Wo, mode, p.Hs, p.Ws);
    long long mtiles;
    tile_geometry(B, p.Hs, p.Ws, p.wt, p.ht, p.nt, mtiles);
    p.tiles_x = p.Ws / p.wt; p.tiles_y = p.Hs / p.ht;
    GIFB200_REQUIRE(mtiles <= 2147483647LL, GIFB200_E_SHAPE, "conv2d_tc: too many tiles");
    p.ksplit = ksplit_of(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode);
    if (p.ksplit > 1) {
        p.part_stride = static_cast<long long>(B) * Ho * Wo * Co;
        p.part = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(reinterpret_cast<char*>(wst) + staged_weight_bytes(Ci, Co, k) - 256) + 255) &
                                          ~static_cast<uintptr_t>(255));
    }
    p.s2 = mode == 1;
    p.in_sy = mode == 1 ? 2 : 1;
    const int pad = k / 2;
    if (mode == 0) {
        p.nphase = 1; p.oys = p.oxs = 1; p.phase_ntaps[0] = T;
        for (int t = 0; t < T; ++t) { p.tap_w[0][t] = t; p.tap_dy[0][t] = t / k - pad; p.tap_dx[0][t] = t % k - pad; }
    } else if (mode == 1) {
        p.nphase = 1; p.oys = p.oxs = 1; p.phase_ntaps[0] = T;
        for (int t = 0; t < T; ++t) {
            const int kh = t / k, kw = t % k;
            p.tap_w[0][t] = t; p.tap_dy[0][t] = kh; p.tap_dx[0][t] = kw >> 1; p.tap_par[0][t] = kw & 1;
        }
    } else {
        // output (Y,X) = (2y+py, 2x+px), y<Hi, x<Wi; taps with kh%2==py, kw%2==px read input (y+(py-kh)/2, x+(px-kw)/2).
        // Row Y=2Hi and column X=2Wi are produced by the two edge launches below.
        p.nphase = 4; p.oys = p.oxs = 2;
        for (int ph = 0; ph < 4; ++ph) {
            const int py = ph >> 1, px = ph & 1;
            p.phase_oy0[ph] = py; p.phase_ox0[ph] = px;
            int n = 0;
            for (int kh = py; kh < 3; kh += 2)
                for (int kw = px; kw < 3; kw += 2) {
                    p.tap_w[ph][n] = kh * 3 + kw; p.tap_dy[ph][n] = (py - kh) / 2; p.tap_dx[ph][n] = (px - kw) / 2;
                    ++n;
                }
            p.phase_ntaps[ph] = n;
        }
    }
    // ---- tensor maps
    CUtensorMap ma, ma2, mb, mb2;
    int rc;
    if (mode != 1) {
        const cuuint64_t dims[4] = {static_cast<cuuint64_t>(Ci), static_cast<cuuint64_t>(Wi), static_cast<cuuint64_t>(Hi), static_cast<cuuint64_t>(B)};
        const cuuint64_t strides[3] = {static_cast<cuuint64_t>(Ci) * es, static_cast<cuuint64_t>(Wi) * Ci * es,
                                       static_cast<cuuint64_t>(Hi) * Wi * Ci * es};
        const cuuint32_t box[4] = {kBlockK, static_cast<cuuint32_t>(p.wt), static_cast<cuuint32_t>(p.ht), static_cast<cuuint32_t>(p.nt)};
        rc = encode_map(&ma, xb, 4, dims, strides, box, swz, dt);
        if (rc == GIFB200_OK && x3) rc = encode_map(&ma2, xb + x_plane * es, 4, dims, strides, box, swz, dt);
    } else {
        // (C, parity, ceil(W/2), H, N): column 2*j + par of row h.  The (par=1, j=W/2) element of an odd-width row lies in
        // the next row; it is never addressed (max column read is 2*(Wo-1)+2 = Wi-1).
        const cuuint64_t dims[5] = {static_cast<cuuint64_t>(Ci), 2, static_cast<cuuint64_t>((Wi + 1) / 2), static_cast<cuuint64_t>(Hi), static_cast<cuuint64_t>(B)};
        const cuuint64_t strides[4] = {static_cast<cuuint64_t>(Ci) * es, static_cast<cuuint64_t>(Ci) * 2 * es,
                                       static_cast<cuuint64_t>(Wi) * Ci * es, static_cast<cuuint64_t>(Hi) * Wi * Ci * es};
        // the whole tile (ht rows 2y + kh of nt images) as one box with traversal stride 2 along H (boxDim counts traversed
        // elements: 2*ht -> ht rows); the per-row form remains for GIFB200_CONV_S2_ROWS=1 (A/B switch)
        static const bool per_row = [] { const char* e = getenv("GIFB200_CONV_S2_ROWS"); return e && atoi(e) != 0; }();
        const bool onebox = !per_row && p.ht * p.nt > 1;
        if (onebox) p.s2 = 2;
        const cuuint32_t box[5] = {kBlockK, 1, static_cast<cuuint32_t>(p.wt), static_cast<cuuint32_t>(onebox ? 2 * p.ht : 1),
                                   static_cast<cuuint32_t>(onebox ? p.nt : 1)};
        const cuuint32_t estr[5] = {1, 1, 1, static_cast<cuuint32_t>(onebox ? 2 : 1), 1};
        rc = encode_map(&ma, xb, 5, dims, strides, box, swz, dt, estr);
        if (rc == GIFB200_OK && x3) rc = encode_map(&ma2, xb + x_plane * es, 5, dims, strides, box, swz, dt, estr);
    }
    if (rc != GIFB200_OK) return rc;
    const int bn = pick_block_n(Co);
    {
        const cuuint64_t dims[3] = {static_cast<cuuint64_t>(Ci), static_cast<cuuint64_t>(Co), static_cast<cuuint64_t>(T)};
        const cuuint64_t strides[2] = {static_cast<cuuint64_t>(Ci) * es, static_cast<cuuint64_t>(Co) * Ci * es};
        const cuuint32_t box[3] = {kBlockK, static_cast<cuuint32_t>(bn), 1};
        rc = encode_map(&mb, wb, 3, dims, strides, box, swz, dt);
        if (rc == GIFB200_OK && x3) rc = encode_map(&mb2, wb + w_plane * es, 3, dims, strides, box, swz, dt);
        if (rc != GIFB200_OK) return rc;
    }
    if (!x3) { ma2 = ma; mb2 = mb; }
    rc = launch_any(bn, x3, ma, ma2, mb, mb2, y, p, static_cast<int>(mtiles), st);
    if (rc == GIFB200_OK && p.ksplit > 1) {
        const long long n4 = p.part_stride / 4;
        int blocks = cdiv(n4, 256);
        if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
        splitk_reduce_kernel<<<blocks, 256, 0, st>>>(p.part, y, n4, p.ksplit, p.part_stride, epi, Co);
        GIFB200_LAUNCH_CHECK("splitk_reduce_kernel");
    }
    if (mode != 2 || rc != GIFB200_OK) return rc;
    // ---- T2 border: output row Y = 2*Hi and column X = 2*Wi (the sites y = Hi / x = Wi that the power-of-two site grid does
    // not cover).  Row Y = 2*Hi only sees kernel row kh = 2 applied to input row Hi-1: a 1-D transposed convolution along x;
    // likewise the column along y with kw = 2.  Both run through the SAME tensor-core kernel on 1-row / 1-column views of
    // the input (two more launches of ~1/64 of the main work each); the single corner pixel is a dot product per (b, o).
    for (int edge = 0; edge < 2 && rc == GIFB200_OK; ++edge) {
        const bool row = edge == 0;
        TcParams q;
        memset(&q, 0, sizeof(q));
        q.B = B; q.Ci = Ci; q.Co = Co; q.Ho = Ho; q.Wo = Wo; q.epi = epi;
        q.Hs = row ? 1 : Hi; q.Ws = row ? Wi : 1;
        q.wt = q.Ws < 128 ? q.Ws : 128;
        q.ht = (128 / q.wt) < q.Hs ? (128 / q.wt) : q.Hs;
        q.nt = 128 / (q.wt * q.ht);
        q.tiles_x = q.Ws / q.wt; q.tiles_y = q.Hs / q.ht;
        const long long mt_e = static_cast<long long>(q.tiles_x) * q.tiles_y * ((B + q.nt - 1) / q.nt);
        q.s2 = 0; q.in_sy = 1; q.nphase = 2; q.oys = q.oxs = 2; q.ksplit = 1;
        for (int ph = 0; ph < 2; ++ph) {          // parity along the strip
            q.phase_oy0[ph] = row ? 2 * Hi : ph;
            q.phase_ox0[ph] = row ? ph : 2 * Wi;
            int n = 0;
            for (int kk = ph; kk < 3; kk += 2) {   // the kernel index along the strip with the right parity
                q.tap_w[ph][n] = row ? (2 * 3 + kk) : (kk * 3 + 2);
                q.tap_dy[ph][n] = row ? 0 : (ph - kk) / 2;
                q.tap_dx[ph][n] = row ? (ph - kk) / 2 : 0;
                ++n;
            }
            q.phase_ntaps[ph] = n;
        }
        CUtensorMap me, me2;
        const char* base = xb + (row ? static_cast<long long>(Hi - 1) * Wi * Ci : static_cast<long long>(Wi - 1) * Ci) * es;
        const cuuint64_t dims[4] = {static_cast<cuuint64_t>(Ci), static_cast<cuuint64_t>(row ? Wi : 1),
                                    static_cast<cuuint64_t>(row ? 1 : Hi), static_cast<cuuint64_t>(B)};
        const cuuint64_t strides[3] = {static_cast<cuuint64_t>(Ci) * es, static_cast<cuuint64_t>(Wi) * Ci * es,
                                       static_cast<cuuint64_t>(Hi) * Wi * Ci * es};
        const cuuint32_t box[4] = {kBlockK, static_cast<cuuint32_t>(q.wt), static_cast<cuuint32_t>(q.ht), static_cast<cuuint32_t>(q.nt)};
        rc = encode_map(&me, base, 4, dims, strides, box, swz, dt);
        if (rc == GIFB200_OK && x3) rc = encode_map(&me2, base + x_plane * es, 4, dims, strides, box, swz, dt);
        if (rc != GIFB200_OK) return rc;
        if (!x3) me2 = me;
        rc = launch_any(bn, x3, me, me2, mb, mb2, y, q, static_cast<int>(mt_e), st);
    }
    if (rc != GIFB200_OK) return rc;
    {
        const char* xpix = xb + (static_cast<long long>(Hi - 1) * Wi + (Wi - 1)) * Ci * es;
        const char* w22 = wb + static_cast<long long>(8) * Co * Ci * es;
        const int blocks = cdiv(static_cast<long long>(B) * Co * 32, 256);
        if (x3)
            t2_corner_kernel<true><<<blocks, 256, 0, st>>>(xpix, w22, y, B, static_cast<long long>(Hi) * Wi * Ci, Ci, Co, Ho, Wo,
                                                           epi, x_plane, w_plane);
        else
            t2_corner_kernel<false><<<blocks, 256, 0, st>>>(xpix, w22, y, B, static_cast<long long>(Hi) * Wi * Ci, Ci, Co, Ho, Wo,
                                                            epi, 0, 0);
    }
    GIFB200_LAUNCH_CHECK("t2_corner_kernel");
    return rc;
}

}  // namespace gifb200
