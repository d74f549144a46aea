// Tensor-core weight-gradient kernel for sm_90a: R[t][cs][cb] = sum_{pixels p} S[p][cs] * Bg[map(p,t)][cb]
//
//   S  = "small-grid" tensor (B,Hs,Ws,Cs): the conv OUTPUT gradient for S1/S2, the conv INPUT for T2
//   Bg = "big" tensor (B,Hb,Wb,Cb) read at map(p,t) = (y+kh-pad, x+kw-pad)  (S1)  or (2y+kh, 2x+kw)  (S2 / T2)
//
// GEMM view per CTA: M = 128 small channels, N = BLOCK_N (<= 64) big channels, K = pixels.  Both operands are
// channels-last, i.e. MN-contiguous ("MN-major"): a TMA box (32 channels x P pixels) lands as P rows of 32 channels.
// A CTA owns one kernel row kh and all KW taps of it: the S tile is loaded once per stage and multiplied with the KW
// shifted Bg tiles into KW separate register accumulators.  The pixel range is split across CTAs (split-K); every split
// writes its own slice of a partial buffer and wgrad_reduce_kernel sums the slices in a fixed order (deterministic).
// Warps 0-7 consume, warp 8 is the TMA producer.
//
// tf32: wgmma takes 32-bit operands K-major only, so the MN-major fp32 tiles are read as mma.sync.m16n8k8 fragments.
//
// STACK variant (Cs == 32, stride-1 3x3: the zero-padded NoiseInjection convs): M = 128 cannot be filled with channels,
// so the four 32-row chunks of the A tile hold the SAME 32 channels of S at three different row shifts (dy = +1, 0, -1;
// the 4th chunk is a duplicate) -- chunk kh then accumulates kernel row kh, the KW shifted Bg tiles give the kernel
// columns, and ONE CTA produces all 9 taps (no kh split).
//
// NARROW variant (AC = 2: Cs == 64, or Cs == 32 with Cb <= 64 for the 1x1 stride-1 layers -- the 512^2 / 1024^2 layers): M = 64, two A
// chunks.  tf32: the 8 mma.sync warps are 2 (rows) x 4 (columns).  X3: both warpgroups issue m64 wgmma on all 64 rows,
// warpgroup wg on the 16-pixel slice wg of every stage; at the end warpgroup 1 hands its sums to warpgroup 0 through the
// drained stage ring (fixed order: slice 0 + slice 1).  With Cs == 32 the second chunk repeats the first and its rows are
// not written.
//
// X3 = true ("bf16x3", gifb200_conv2d_wgrad impl 3): both operands arrive as two bf16 planes (hi, lo; gifb200_split_bf16).
// 16-bit MN-major tiles of 32 channels use the canonical SWIZZLE_64B layout (rows of 64 bytes, 8-pixel K atoms of 512 B; TMA
// side CU_TENSOR_MAP_SWIZZLE_64B), which wgmma reads transposed; a stage holds the hi and the lo chunk set of each operand --
// the SAME bytes as the fp32 tiles -- and every 16-pixel slice issues three bf16 wgmmas (lo*hi, hi*lo, hi*hi) per
// warpgroup into the tap's fp32 accumulator.
#include "tc_common.cuh"

namespace gifb200 {
namespace {

constexpr int kWgStages = 4;
constexpr int kPix = 32;                       // pixels (GEMM K) per stage
constexpr int kWgConsumerWarps = 8;            // two warpgroups (X3: wgmma on rows 0-63 / 64-127) or 4 x 2 mma.sync warps
constexpr int kWgThreads = 32 * kWgConsumerWarps + 32;   // + one TMA producer warp

struct WgParams {
    int B, Hs, Ws, Cs, Hb, Wb, Cb;
    int k, pad, s2, flip;
    int pw;                 // pixels per TMA row load (min(Ws, 32)); rows per stage = 32 / pw
    int mr_s, mr_b;         // narrow images (pw < 32): the S / Bg tensor map's box spans ALL rows of a stage (by rows x bn images),
                            // one TMA issue per chunk and tap instead of one per row
    long long units;        // number of 32-pixel units in the small grid
    int splits;
    long long stride_t, stride_cs, stride_cb;
    long long part_stride;   // floats per split in the partial buffer: T * Cs_total * Cb (layout [split][t][cs][cb])
};

constexpr int kHaloRows = kPix + 2;                 // 34 pixel rows: the 32 of the stage + one on each side

// HALO (stride-1 3x3 layers with Ws >= 32): the KW shifted big-tensor tiles of a stage overlap in all but 2 pixel rows, so
// the stage holds ONE (32 + 2)-row tile per 32-channel chunk and tap kw reads it from pixel row kw on.
template <int KW, int BLOCK_N, bool HALO = false, bool X3 = false, int AC = 4>
struct WgSmem {
    static constexpr int kRowBytes = X3 ? 64 : 128;                   // 32 channels of one pixel
    static constexpr int kChunkBytes = kPix * kRowBytes;              // one 32-channel x 32-pixel chunk: 4 KB fp32, 2 KB bf16
    static constexpr int kHaloChunkBytes = X3 ? 2560 : 5120;          // 34 rows padded to the swizzle atom (512 B bf16, 1024 B fp32)
    static constexpr int kPlanes = X3 ? 2 : 1;                        // hi and lo chunk sets, hi first
    static constexpr int kBChunks = BLOCK_N / 32;
    static constexpr int kAPlaneBytes = AC * kChunkBytes;         // AC 32-channel A chunks: M = 32 * AC small channels
    static constexpr int kABytes = kPlanes * kAPlaneBytes;
    static constexpr int kBPlaneBytes = kBChunks * (HALO ? kHaloChunkBytes : kChunkBytes);   // one tap (or the halo tile), one plane
    static constexpr int kBBytesPerTap = kPlanes * kBPlaneBytes;
    static constexpr int kStages = HALO ? 5 : kWgStages;
    static constexpr int kStageBytes = HALO ? kABytes + kBBytesPerTap : kABytes + KW * kBBytesPerTap;
    static constexpr int kTxBytes = HALO ? kABytes + kPlanes * kBChunks * kHaloRows * kRowBytes : kStageBytes;
    static constexpr int kBarrierOffset = (kStages * kStageBytes + 1023) / 1024 * 1024;
    static constexpr int kDynamic = kBarrierOffset + 128 + 1024;
};

// byte offset of (pixel row, channel) in a 32-channel fp32 chunk written by TMA with SWIZZLE_128B (1024 B aligned chunk):
// the 16-byte column index is XOR-ed with the row index mod 8
__device__ __forceinline__ uint32_t sw128_off(int row, int ch) {
    return static_cast<uint32_t>(row * 128 + ((((ch >> 2) ^ row) & 7) << 4) + (ch & 3) * 4);
}

template <int KW, int BLOCK_N, bool STACK, bool HALO, bool X3, int AC>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_tc_kernel(const __grid_constant__ CUtensorMap map_s,
                                                                 const __grid_constant__ CUtensorMap map_s2,
                                                                 const __grid_constant__ CUtensorMap map_b,
                                                                 const __grid_constant__ CUtensorMap map_b2,
                                                                 float* __restrict__ part, const WgParams p) {
    using L = WgSmem<KW, BLOCK_N, HALO, X3, AC>;
    constexpr int kM = 32 * AC;
    constexpr int kChunkBytes = L::kChunkBytes;
    constexpr int kHaloChunkBytes = L::kHaloChunkBytes;
    constexpr int kNStages = L::kStages;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarrierOffset);
    uint64_t* empty_bar = full_bar + kNStages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    const int ms = blockIdx.x;                       // kM-channel tile of the small tensor
    const int nb = blockIdx.y;                       // BLOCK_N-channel tile of the big tensor
    const int kh = STACK ? 0 : blockIdx.z / p.splits, split = STACK ? blockIdx.z : blockIdx.z % p.splits;
    const long long per = (p.units + p.splits - 1) / p.splits;
    const long long u0 = split * per;
    const long long u1 = u0 + per < p.units ? u0 + per : p.units;
    const int iters = u1 > u0 ? static_cast<int>(u1 - u0) : 0;

    if (warp == kWgConsumerWarps && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_s) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
        if (X3) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_s2) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b2) : "memory");
        }
        for (int s = 0; s < kNStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kWgConsumerWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();

    if (warp == kWgConsumerWarps) {
        if (lane == 0) {
            // ===================== TMA producer (one thread) =====================
            const int rows = kPix / p.pw;                    // rows of the small grid per stage
            const int segs = p.Ws / p.pw;                    // 32-pixel segments per row (>= 1 when pw == 32)
            const int row_bytes = p.pw * L::kRowBytes;
            int stage = 0;
            uint32_t ph = 0;
            for (int it = 0; it < iters; ++it) {
                const long long u = u0 + it;
                mbar_wait(&empty_bar[stage], ph ^ 1);
                uint8_t* a_dst = smem + stage * L::kStageBytes;
                uint8_t* b_dst = a_dst + L::kABytes;
                mbar_expect_tx(&full_bar[stage], L::kTxBytes);
                for (int r = 0; r < rows; ++r) {
                    long long grow;                          // global row index n*Hs + y
                    int x0;
                    if (rows == 1) { grow = u / segs; x0 = static_cast<int>(u % segs) * kPix; }
                    else { grow = u * rows + r; x0 = 0; }
                    const int n = static_cast<int>(grow / p.Hs), y = static_cast<int>(grow % p.Hs);
#pragma unroll
                    for (int pl = 0; pl < L::kPlanes; ++pl) {    // X3: plane 0 = hi, plane 1 = lo (same coordinates, own map)
                        const CUtensorMap* ms_ = pl ? &map_s2 : &map_s;
                        const CUtensorMap* mb_ = pl ? &map_b2 : &map_b;
                        uint8_t* a_pl = a_dst + pl * L::kAPlaneBytes;
                        if (r == 0 || !p.mr_s) {
                            for (int c = 0; c < AC; ++c) {
                                if (STACK)   // chunk kh = S shifted by dy = 1 - kh rows (rows outside the image are zero-filled)
                                    tma_load_4d(a_pl + c * kChunkBytes + r * row_bytes, ms_, &full_bar[stage], 0, x0,
                                                y + 1 - (c < 3 ? c : 2), n);
                                else if (AC == 2)   // Cs == 32: the second chunk repeats the first
                                    tma_load_4d(a_pl + c * kChunkBytes + r * row_bytes, ms_, &full_bar[stage],
                                                c * 32 < p.Cs ? c * 32 : 0, x0, y, n);
                                else
                                    tma_load_4d(a_pl + c * kChunkBytes + r * row_bytes, ms_, &full_bar[stage], ms * 128 + c * 32, x0, y, n);
                            }
                        }
                        if (HALO) {      // one (32+2)-pixel tile per 32-channel chunk, starting one pixel to the left
                            for (int c = 0; c < L::kBChunks; ++c)
                                tma_load_4d(b_dst + pl * L::kBPlaneBytes + c * kHaloChunkBytes, mb_, &full_bar[stage],
                                            nb * BLOCK_N + c * 32, x0 - 1, y + (STACK ? 0 : kh - p.pad), n);
                            continue;
                        }
                        if (r != 0 && p.mr_b) continue;
                        for (int kw = 0; kw < KW; ++kw)
                            for (int c = 0; c < L::kBChunks; ++c) {
                                uint8_t* dst = b_dst + kw * L::kBBytesPerTap + pl * L::kBPlaneBytes + c * kChunkBytes + r * row_bytes;
                                const int ch = nb * BLOCK_N + c * 32;
                                if (STACK)
                                    tma_load_4d(dst, mb_, &full_bar[stage], ch, x0 + kw - 1, y, n);
                                else if (!p.s2)
                                    tma_load_4d(dst, mb_, &full_bar[stage], ch, x0 + kw - p.pad, y + kh - p.pad, n);
                                else
                                    tma_load_5d(dst, mb_, &full_bar[stage], ch, kw & 1, x0 + (kw >> 1), 2 * y + kh, n);
                            }
                    }
                }
                if (++stage == kNStages) { stage = 0; ph ^= 1; }
            }
        }
        return;
    }

    // ===================== consumers =====================
    // The epilogue writes this split's slice of the partial buffer; a split without work (units not divisible) writes zeros,
    // so the slice is always defined for the reduction.
    float* pbase = part + split * p.part_stride;
    const int g = lane >> 2, tq = lane & 3;
    if (X3) {
        // wgmma, both operands MN-major SWIZZLE_64B (rows of 64 B = 32 bf16, 8-pixel K atoms of 512 B): LBO = distance between
        // 32-channel chunks, SBO = 512 B.  AC = 4: warpgroup wg owns A chunks 2wg, 2wg+1 (its 64 rows) and both 16-pixel
        // slices; AC = 2: all 64 rows and slice wg.  One accumulator per tap.
        const int wg = warp >> 2, wq = warp & 3;
        constexpr int kSlices = AC == 4 ? kPix / 16 : 1;
        constexpr int kAcc = BLOCK_N / 2;
        float acc[KW][kAcc];
#pragma unroll
        for (int kw = 0; kw < KW; ++kw)
#pragma unroll
            for (int i = 0; i < kAcc; ++i) acc[kw][i] = 0.f;
        int stage = 0, prev = -1;
        uint32_t ph = 0;
        // The A operand of a slice (this warpgroup's 64 rows x 16 pixels of S, hi and lo plane) is the same for all KW taps
        // and for two of the three MMAs of each tap, so it is loaded into registers once per slice (ldmatrix .trans of the
        // MN-major tile) and only B is read from shared memory by the wgmmas.  wgmma reads the fragments asynchronously and
        // the previous stage's group is still in flight when the next stage loads its own, so the fragments alternate
        // between two sets.
        uint32_t afr[2][kSlices][2][4];      // [set][slice][plane: 0 = hi, 1 = lo][register]
        // this lane's ldmatrix row: matrix mi = lane / 8 covers rows +8 (mi & 1) and pixels +8 (mi >> 1) of the warp's 16 x 16
        // block, row r = lane % 8 is pixel r of it; a pixel row is 64 B and SWIZZLE_64B XORs its 16 B unit with (pixel / 2) % 4
        const int mi = lane >> 3, r8 = lane & 7;
        const uint32_t a_lane = (AC == 4 ? wg * 2 * kChunkBytes : 0) + (wq >> 1) * kChunkBytes + (8 * (mi >> 1) + r8) * 64 +
                                ((((2 * wq + (mi & 1)) & 3) ^ (r8 >> 1)) << 4);
        auto run_stage = [&](uint32_t (&fr)[kSlices][2][4]) {
            mbar_wait(&full_bar[stage], ph);
            const uint32_t a_addr = smem_u32(smem + stage * L::kStageBytes);
#pragma unroll
            for (int jj = 0; jj < kSlices; ++jj) {
                const int j = AC == 4 ? jj : wg;
#pragma unroll
                for (int pl = 0; pl < 2; ++pl) ldmatrix_x4_trans(fr[jj][pl], a_addr + pl * L::kAPlaneBytes + a_lane + 1024 * j);
            }
            wgmma_fence();
#pragma unroll
            for (int kw = 0; kw < KW; ++kw) {
                fence_regs<kAcc>(acc[kw]);
                // HALO: tap kw starts kw pixel rows (64 B each) into the halo tile, inside a 512 B swizzle atom.  wgmma applies
                // the SWIZZLE_64B XOR to the absolute shared-memory address, as TMA wrote it, so the descriptor simply starts
                // there (base offset 0; the tests compare every tap bitwise with the one-tile-per-tap layout).
                const uint32_t b_addr = a_addr + L::kABytes + (HALO ? kw * L::kRowBytes : kw * L::kBBytesPerTap);
                const uint32_t b_lbo = HALO ? kHaloChunkBytes : kChunkBytes;
                const uint64_t bdesc = make_smem_desc(b_addr, b_lbo, 512, 2);
                const uint64_t bdesc_lo = make_smem_desc(b_addr + L::kBPlaneBytes, b_lbo, 512, 2);
#pragma unroll
                for (int jj = 0; jj < kSlices; ++jj) {   // 16 pixels per MMA = two 8-pixel atoms: next slice = +1024 B (>>4 = 64)
                    const int j = AC == 4 ? jj : wg;
                    wgmma_bf16_rs<BLOCK_N>(acc[kw], fr[jj][1], bdesc + 64 * j, 1, Trans<1>());
                    wgmma_bf16_rs<BLOCK_N>(acc[kw], fr[jj][0], bdesc_lo + 64 * j, 1, Trans<1>());
                    wgmma_bf16_rs<BLOCK_N>(acc[kw], fr[jj][0], bdesc + 64 * j, 1, Trans<1>());
                }
            }
            wgmma_commit();
#pragma unroll
            for (int kw = 0; kw < KW; ++kw) fence_regs<kAcc>(acc[kw]);
            wgmma_wait<1>();
            if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
            prev = stage;
            if (++stage == kNStages) { stage = 0; ph ^= 1; }
        };
        for (int it = 0; it < iters; it += 2) {
            run_stage(afr[0]);
            if (it + 1 < iters) run_stage(afr[1]);
        }
        wgmma_wait<0>();
#pragma unroll
        for (int kw = 0; kw < KW; ++kw) fence_regs<kAcc>(acc[kw]);
        if constexpr (AC == 2) {
            // every MMA of both warpgroups has completed past the barrier, so the stage ring is free to carry the exchange
            static_assert(KW * kAcc * 128 * 4 <= kNStages * L::kStageBytes, "exchange buffer exceeds the stage ring");
            float* xch = reinterpret_cast<float*>(smem) + (threadIdx.x & 127);
            asm volatile("bar.sync 1, %0;" ::"n"(32 * kWgConsumerWarps) : "memory");
            if (wg == 1) {
#pragma unroll
                for (int kw = 0; kw < KW; ++kw)
#pragma unroll
                    for (int i = 0; i < kAcc; ++i) xch[(kw * kAcc + i) * 128] = acc[kw][i];
            }
            asm volatile("bar.sync 1, %0;" ::"n"(32 * kWgConsumerWarps) : "memory");
            if (wg == 1) return;
#pragma unroll
            for (int kw = 0; kw < KW; ++kw)
#pragma unroll
                for (int i = 0; i < kAcc; ++i) acc[kw][i] += xch[(kw * kAcc + i) * 128];
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = (AC == 4 ? wg * 64 : 0) + wq * 16 + g + 8 * h;      // row of the kM-row A tile
            const int q = r >> 5;
            if (STACK && q == 3) continue;                    // duplicate chunk
            if (AC == 2 && r >= p.Cs) continue;               // Cs == 32: repeated chunk
            const int cs = STACK ? (r & 31) : ms * kM + r;
#pragma unroll
            for (int kw = 0; kw < KW; ++kw) {
                const int t = (STACK ? q : kh) * p.k + kw;
                float* obase = pbase + (static_cast<long long>(t) * p.Cs + cs) * p.Cb + nb * BLOCK_N + 2 * tq;
#pragma unroll
                for (int j = 0; j < BLOCK_N / 8; ++j)
                    *reinterpret_cast<float2*>(obase + 8 * j) = make_float2(acc[kw][4 * j + 2 * h], acc[kw][4 * j + 2 * h + 1]);
            }
        }
    } else {
        // mma.sync m16n8k8 tf32: warp (wm, wn) computes rows 32wm..32wm+31 (= A chunk wm) x columns wn*BLOCK_N/kWN .. of
        // every tap.  Fragments are gathered from the SWIZZLE_128B tiles with 32-bit shared loads.
        constexpr int kWN = kWgConsumerWarps / AC;       // warps along N: 2 (AC = 4) or 4 (AC = 2)
        const int wm = warp % AC, wn = warp / AC;
        constexpr int NT = BLOCK_N / (8 * kWN);          // n8 tiles per warp
        float acc[KW][2][NT][4];
#pragma unroll
        for (int kw = 0; kw < KW; ++kw)
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) acc[kw][mt][nt][e] = 0.f;
        int stage = 0;
        uint32_t ph = 0;
        for (int it = 0; it < iters; ++it) {
            mbar_wait(&full_bar[stage], ph);
            const uint8_t* sa = smem + stage * L::kStageBytes + wm * kChunkBytes;
            const uint8_t* sb = smem + stage * L::kStageBytes + L::kABytes;
#pragma unroll
            for (int k8 = 0; k8 < kPix / 8; ++k8) {
                const int k0 = k8 * 8 + tq;
                uint32_t a[2][4];
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    const int ch = mt * 16 + g;
                    a[mt][0] = *reinterpret_cast<const uint32_t*>(sa + sw128_off(k0, ch));
                    a[mt][1] = *reinterpret_cast<const uint32_t*>(sa + sw128_off(k0, ch + 8));
                    a[mt][2] = *reinterpret_cast<const uint32_t*>(sa + sw128_off(k0 + 4, ch));
                    a[mt][3] = *reinterpret_cast<const uint32_t*>(sa + sw128_off(k0 + 4, ch + 8));
                }
#pragma unroll
                for (int kw = 0; kw < KW; ++kw) {
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt) {
                        const int n = wn * (BLOCK_N / kWN) + nt * 8 + g;
                        const uint8_t* chunk = HALO ? sb + (n >> 5) * kHaloChunkBytes : sb + kw * L::kBBytesPerTap + (n >> 5) * kChunkBytes;
                        const int row = HALO ? k0 + kw : k0;     // HALO: tap kw starts kw pixel rows into the halo tile
                        uint32_t b[2];
                        b[0] = *reinterpret_cast<const uint32_t*>(chunk + sw128_off(row, n & 31));
                        b[1] = *reinterpret_cast<const uint32_t*>(chunk + sw128_off(row + 4, n & 31));
#pragma unroll
                        for (int mt = 0; mt < 2; ++mt) mma_tf32_m16n8k8(acc[kw][mt][nt], a[mt], b);
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
            if (++stage == kNStages) { stage = 0; ph ^= 1; }
        }
        if (STACK && wm == 3) return;                           // duplicate chunk
        if (AC == 2 && wm * 32 >= p.Cs) return;                 // Cs == 32: repeated chunk
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = wm * 32 + mt * 16 + g + 8 * h;
                const int cs = STACK ? (r & 31) : ms * kM + r;
#pragma unroll
                for (int kw = 0; kw < KW; ++kw) {
                    const int t = (STACK ? wm : kh) * p.k + kw;
                    float* obase = pbase + (static_cast<long long>(t) * p.Cs + cs) * p.Cb + nb * BLOCK_N + wn * (BLOCK_N / kWN) + 2 * tq;
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt)
                        *reinterpret_cast<float2*>(obase + nt * 8) = make_float2(acc[kw][mt][nt][2 * h], acc[kw][mt][nt][2 * h + 1]);
                }
            }
    }
}

// gw (physical weight-gradient layout, via strides) = sum over splits of part[split][t][cs][cb]
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ out,
                                                           WgParams p, int T) {
    const long long total = static_cast<long long>(T) * p.Cs * p.Cb;
    for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        float acc = 0.f;
        for (int s = 0; s < p.splits; ++s) acc += part[s * p.part_stride + e];
        const int cb = static_cast<int>(e % p.Cb);
        const int cs = static_cast<int>((e / p.Cb) % p.Cs);
        const int t = static_cast<int>(e / (static_cast<long long>(p.Cb) * p.Cs));
        const int tt = p.flip ? T - 1 - t : t;
        out[tt * p.stride_t + cs * p.stride_cs + cb * p.stride_cb] = acc;
    }
}

inline bool pow2i(int v) { return v > 0 && (v & (v - 1)) == 0; }

// at most 64 big channels per CTA: KW accumulators of 128 x BLOCK_N live in the registers of the consumer warps
int pick_bn(int Cb) {
    if (Cb % 64 == 0) return 64;
    if (Cb % 32 == 0) return 32;
    return 0;
}

struct WgMaps { CUtensorMap s, s2, b, b2; };

template <int KW, int BLOCK_N, bool STACK, bool HALO, bool X3, int AC>
int launch_wg(const WgMaps& m, float* out, float* part, const WgParams& p, cudaStream_t st) {
    using L = WgSmem<KW, BLOCK_N, HALO, X3, AC>;
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(wgrad_tc_kernel<KW, BLOCK_N, STACK, HALO, X3, AC>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kDynamic);
        if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "cudaFuncSetAttribute(wgrad_tc_kernel)", cudaGetErrorString(e));
        attr_set = true;
    }
    dim3 grid(STACK || AC == 2 ? 1 : p.Cs / 128, p.Cb / BLOCK_N, STACK ? p.splits : p.k * p.splits);
    wgrad_tc_kernel<KW, BLOCK_N, STACK, HALO, X3, AC><<<grid, kWgThreads, L::kDynamic, st>>>(m.s, m.s2, m.b, m.b2, part, p);
    GIFB200_LAUNCH_CHECK("wgrad_tc_kernel");
    const int T = p.k * p.k;
    const long long total = static_cast<long long>(T) * p.Cs * p.Cb;
    int blocks = cdiv(total, 256);
    if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
    wgrad_reduce_kernel<<<blocks, 256, 0, st>>>(part, out, p, T);
    GIFB200_LAUNCH_CHECK("wgrad_reduce_kernel");
    return GIFB200_OK;
}

inline bool is_stack(int Cs, int k, int mode) { return Cs == 32 && mode == 0 && k == 3; }
// 32 small channels only up to 64 big ones: with 128 (the 1x1 256^2 discriminator stem's R1 term, Cs = 9 padded to 32) the
// exact SIMT kernel keeps the 256^2 step's results bitwise as they were
inline bool is_narrow(int Cs, int Cb, int k, int mode) { return Cs == 64 || (Cs == 32 && mode == 0 && k == 1 && Cb <= 64); }

void roles(int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int mode, int& Hs, int& Ws, int& Cs, int& Hb, int& Wb, int& Cb) {
    if (mode == 2) { Hs = Hi; Ws = Wi; Cs = Ci; Hb = Ho; Wb = Wo; Cb = Co; }
    else { Hs = Ho; Ws = Wo; Cs = Co; Hb = Hi; Wb = Wi; Cb = Ci; }
}

}  // namespace

bool conv2d_wgrad_tc_supported(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode) {
    if (B <= 0 || !(k == 3 || (k == 1 && mode == 0))) return false;
    if (mode == 0 && !(Ho == Hi && Wo == Wi)) return false;
    if (mode == 1 && !(Hi == 2 * Ho + 1 && Wi == 2 * Wo + 1)) return false;
    if (mode == 2 && !(Ho == 2 * Hi + 1 && Wo == 2 * Wi + 1)) return false;
    int Hs, Ws, Cs, Hb, Wb, Cb;
    roles(Hi, Wi, Ci, Ho, Wo, Co, mode, Hs, Ws, Cs, Hb, Wb, Cb);
    if ((Cs % 128 != 0 && !is_stack(Cs, k, mode) && !is_narrow(Cs, Cb, k, mode)) || pick_bn(Cb) == 0) return false;
    if (!pow2i(Hs) || !pow2i(Ws) || Ws < 4 || Hs < 4) return false;
    if ((static_cast<long long>(B) * Hs * Ws) % kPix != 0) return false;
    const int pw = Ws < kPix ? Ws : kPix;
    if ((static_cast<long long>(B) * Hs) % (kPix / pw) != 0) return false;
    return true;
}

static long long wgrad_splits(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode, long long* units_out) {
    int Hs, Ws, Cs, Hb, Wb, Cb;
    roles(Hi, Wi, Ci, Ho, Wo, Co, mode, Hs, Ws, Cs, Hb, Wb, Cb);
    const long long units = static_cast<long long>(B) * Hs * Ws / kPix;
    const int bn = pick_bn(Cb);
    const long long m_tiles = is_narrow(Cs, Cb, k, mode) ? 1 : Cs / 128;
    const long long base_ctas = is_stack(Cs, k, mode) ? (Cb / bn) : m_tiles * (Cb / bn) * k;
    // ONE wave: the kernel runs one CTA per SM (90-160 KB of shared memory), so the grid must not exceed the SM count
    // (rounding the split count up would leave a second wave of a few stragglers that doubles the kernel time).
    long long splits = kNumSMs / base_ctas;
    if (splits > units) splits = units;
    if (splits < 1) splits = 1;
    if (units_out) *units_out = units;
    return splits;
}

size_t conv2d_wgrad_tc_workspace_bytes(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode) {
    if (!conv2d_wgrad_tc_supported(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode)) return 0;
    return static_cast<size_t>(wgrad_splits(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, nullptr)) * k * k * Co * Ci * sizeof(float) + 256;
}

template <bool X3>
static int dispatch_wg(int k, int bn, bool stack, bool narrow, bool halo, const WgMaps& m, float* gw, float* part, const WgParams& p,
                       cudaStream_t st) {
#define GIFB200_WG(KW, BN, ST, HA) launch_wg<KW, BN, ST, HA, X3, 4>(m, gw, part, p, st)
#define GIFB200_WGN(KW, BN, HA) launch_wg<KW, BN, false, HA, X3, 2>(m, gw, part, p, st)
    if (narrow) {
        if (halo) return bn == 64 ? GIFB200_WGN(3, 64, true) : GIFB200_WGN(3, 32, true);
        if (k == 3) return bn == 64 ? GIFB200_WGN(3, 64, false) : GIFB200_WGN(3, 32, false);
        return bn == 64 ? GIFB200_WGN(1, 64, false) : GIFB200_WGN(1, 32, false);
    }
    if (stack && halo) return bn == 64 ? GIFB200_WG(3, 64, true, true) : GIFB200_WG(3, 32, true, true);
    if (halo) return bn == 64 ? GIFB200_WG(3, 64, false, true) : GIFB200_WG(3, 32, false, true);
    if (stack) return bn == 64 ? GIFB200_WG(3, 64, true, false) : GIFB200_WG(3, 32, true, false);
    if (k == 3) return bn == 64 ? GIFB200_WG(3, 64, false, false) : GIFB200_WG(3, 32, false, false);
    return bn == 64 ? GIFB200_WG(1, 64, false, false) : GIFB200_WG(1, 32, false, false);
#undef GIFB200_WGN
#undef GIFB200_WG
}

int conv2d_wgrad_tc(const float* x, const float* gy, float* gw, int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co,
                    int k, int mode, int flip, int transposed, void* ws, size_t ws_bytes, cudaStream_t st, bool x3) {
    GIFB200_REQUIRE(ws && ws_bytes >= conv2d_wgrad_tc_workspace_bytes(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode), GIFB200_E_WORKSPACE,
                    "conv2d_wgrad_tc: workspace too small (see gifb200_conv2d_wgrad_workspace_bytes)");
    float* part = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~static_cast<uintptr_t>(255));
    GIFB200_REQUIRE(conv2d_wgrad_tc_supported(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode), GIFB200_E_SHAPE,
                    "conv2d_wgrad_tc: unsupported shape");
    GIFB200_REQUIRE(aligned16(x) && aligned16(gy), GIFB200_E_ALIGN, "conv2d_wgrad_tc: x / gy must be 16-byte aligned");
    WgParams p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.k = k; p.flip = flip;
    roles(Hi, Wi, Ci, Ho, Wo, Co, mode, p.Hs, p.Ws, p.Cs, p.Hb, p.Wb, p.Cb);
    const float* S = mode == 2 ? x : gy;
    const float* Bg = mode == 2 ? gy : x;
    p.s2 = mode != 0;
    p.pad = mode == 0 ? k / 2 : 0;
    p.pw = p.Ws < kPix ? p.Ws : kPix;
    p.units = static_cast<long long>(B) * p.Hs * p.Ws / kPix;
    // physical layout of gw: transposed ? [t][i][o] : [t][o][i];  small channels are o for S1/S2, i for T2
    const long long stride_o = transposed ? 1 : Ci, stride_i = transposed ? Co : 1;
    p.stride_cs = mode == 2 ? stride_i : stride_o;
    p.stride_cb = mode == 2 ? stride_o : stride_i;
    p.stride_t = static_cast<long long>(Co) * Ci;
    const int bn = pick_bn(p.Cb);
    const bool stack = is_stack(p.Cs, k, mode), narrow = is_narrow(p.Cs, p.Cb, k, mode);
    p.splits = static_cast<int>(wgrad_splits(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, nullptr));
    p.part_stride = static_cast<long long>(k) * k * Co * Ci;
    // operand element size / tile layout: fp32 (SWIZZLE_128B, read by mma.sync fragments) or bf16 planes (MN-major SWIZZLE_64B)
    const cuuint64_t es = x3 ? 2 : 4;
    const CUtensorMapSwizzle swz = x3 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
    const CUtensorMapDataType dt = x3 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    const char* Sb = reinterpret_cast<const char*>(S);
    const char* Bb = reinterpret_cast<const char*>(Bg);
    const long long s_plane = static_cast<long long>(B) * p.Hs * p.Ws * p.Cs * es;   // bytes between the hi and the lo plane
    const long long b_plane = static_cast<long long>(B) * p.Hb * p.Wb * p.Cb * es;
    WgMaps m;
    {
        const cuuint64_t dims[4] = {static_cast<cuuint64_t>(p.Cs), static_cast<cuuint64_t>(p.Ws), static_cast<cuuint64_t>(p.Hs), static_cast<cuuint64_t>(B)};
        const cuuint64_t strides[3] = {static_cast<cuuint64_t>(p.Cs) * es, static_cast<cuuint64_t>(p.Ws) * p.Cs * es,
                                       static_cast<cuuint64_t>(p.Hs) * p.Ws * p.Cs * es};
        // narrow images: one box = all rows of a stage (rows consecutive in (n, y): by rows of bn images)
        const int rows_per_stage = kPix / p.pw;
        const int by = rows_per_stage < p.Hs ? rows_per_stage : p.Hs, bnimg = rows_per_stage / by;
        p.mr_s = rows_per_stage > 1;
        p.mr_b = rows_per_stage > 1;      // stride-2 modes: the big tensor's rows 2y + kh through a traversal stride of 2
        const cuuint32_t box[4] = {32, static_cast<cuuint32_t>(p.pw), static_cast<cuuint32_t>(by), static_cast<cuuint32_t>(bnimg)};
        int rc = encode_map(&m.s, Sb, 4, dims, strides, box, swz, dt);
        if (rc == GIFB200_OK && x3) rc = encode_map(&m.s2, Sb + s_plane, 4, dims, strides, box, swz, dt);
        if (rc != GIFB200_OK) return rc;
    }
    const bool halo = mode == 0 && k == 3 && p.pw == kPix;
    if (!p.s2) {
        const cuuint64_t dims[4] = {static_cast<cuuint64_t>(p.Cb), static_cast<cuuint64_t>(p.Wb), static_cast<cuuint64_t>(p.Hb), static_cast<cuuint64_t>(B)};
        const cuuint64_t strides[3] = {static_cast<cuuint64_t>(p.Cb) * es, static_cast<cuuint64_t>(p.Wb) * p.Cb * es,
                                       static_cast<cuuint64_t>(p.Hb) * p.Wb * p.Cb * es};
        const int rows_per_stage = kPix / p.pw;       // mode 0: the big grid is the small grid (Hb == Hs)
        const int by = rows_per_stage < p.Hs ? rows_per_stage : p.Hs, bnimg = rows_per_stage / by;
        const cuuint32_t box[4] = {32, static_cast<cuuint32_t>(halo ? kHaloRows : p.pw), static_cast<cuuint32_t>(p.mr_b ? by : 1),
                                   static_cast<cuuint32_t>(p.mr_b ? bnimg : 1)};
        int rc = encode_map(&m.b, Bb, 4, dims, strides, box, swz, dt);
        if (rc == GIFB200_OK && x3) rc = encode_map(&m.b2, Bb + b_plane, 4, dims, strides, box, swz, dt);
        if (rc != GIFB200_OK) return rc;
    } else {
        const cuuint64_t dims[5] = {static_cast<cuuint64_t>(p.Cb), 2, static_cast<cuuint64_t>((p.Wb + 1) / 2), static_cast<cuuint64_t>(p.Hb), static_cast<cuuint64_t>(B)};
        const cuuint64_t strides[4] = {static_cast<cuuint64_t>(p.Cb) * es, static_cast<cuuint64_t>(p.Cb) * 2 * es,
                                       static_cast<cuuint64_t>(p.Wb) * p.Cb * es, static_cast<cuuint64_t>(p.Hb) * p.Wb * p.Cb * es};
        // rows 2y + kh of a stage through ONE box: traversal stride 2 along H (boxDim counts traversed elements: 2*by -> by rows)
        const int rows_per_stage = kPix / p.pw;
        const int by = rows_per_stage < p.Hs ? rows_per_stage : p.Hs, bnimg = rows_per_stage / by;
        const cuuint32_t box[5] = {32, 1, static_cast<cuuint32_t>(p.pw), static_cast<cuuint32_t>(p.mr_b ? 2 * by : 1),
                                   static_cast<cuuint32_t>(p.mr_b ? bnimg : 1)};
        const cuuint32_t estr[5] = {1, 1, 1, static_cast<cuuint32_t>(p.mr_b ? 2 : 1), 1};
        int rc = encode_map(&m.b, Bb, 5, dims, strides, box, swz, dt, estr);
        if (rc == GIFB200_OK && x3) rc = encode_map(&m.b2, Bb + b_plane, 5, dims, strides, box, swz, dt, estr);
        if (rc != GIFB200_OK) return rc;
    }
    if (!x3) { m.s2 = m.s; m.b2 = m.b; }
    return x3 ? dispatch_wg<true>(k, bn, stack, narrow, halo, m, gw, part, p, st)
              : dispatch_wg<false>(k, bn, stack, narrow, halo, m, gw, part, p, st);
}

}  // namespace gifb200
