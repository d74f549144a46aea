// Baseline JPEG encoding on the device, byte for byte what Pillow's save(format="JPEG", quality=q) writes for an RGB image
// with default options (libjpeg-turbo: 4:2:0, islow FDCT, Annex K Huffman tables, no restart interval).  The host side is
// gif_b200/image_encode.py (headers and tables); oracle/jpeg_encode_oracle.py restates every stage in numpy.
//
//   jpeg_enc_blocks   8 threads per 8x8 block: RGB->YCbCr, h2v2 downsampling, islow FDCT, reciprocal quantisation, the
//                     block's AC code length
//   jpeg_enc_scan     one CTA per image: DC differences chained per component, exclusive scan of the block bit offsets,
//                     zeroes the image's word buffer
//   jpeg_enc_pack     one thread per block: codes OR-ed into the word buffer at the block's bit offset (atomicOr into zeroed
//                     words is order-independent, so the bytes are deterministic); the last block pads with 1-bits
//   jpeg_enc_count / jpeg_enc_stuff_scan / jpeg_enc_stuff
//                     0xFF -> 0xFF 0x00 byte stuffing: 0xFF bytes per 32-byte chunk, their exclusive scan per image, then
//                     the scatter into one output buffer, images back to back
#include "common.cuh"

namespace gifb200 {
namespace {

constexpr int kBlocksPerCta = 32;       // jpeg_enc_blocks: 8 threads each
constexpr int kScanThreads = 1024;
constexpr int kChunkBytes = 32;         // byte-stuffing granularity
constexpr int kMaxBlockBits = 22 + 63 * 26;
// table offsets (image_encode.encoder_tables)
constexpr int kQuantInts = 3 * 64;      // reciprocal, correction, shift per coefficient (zigzag)
constexpr int kHuffBase = 2 * kQuantInts;

__constant__ uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct EncGeom {
    int B, H, W, mx, my, nb, wb, hb;    // MCU grid, blocks per image, luma blocks inside the image
    long long words;                    // 32-bit words per image in the bit buffer
    int chunks;                         // stuffing chunks per image
};

EncGeom enc_geom(int B, int H, int W) {
    EncGeom g;
    g.B = B;
    g.H = H;
    g.W = W;
    g.mx = (W + 15) / 16;
    g.my = (H + 15) / 16;
    g.nb = g.mx * g.my * 6;
    g.wb = (W + 7) / 8;
    g.hb = (H + 7) / 8;
    g.words = (static_cast<long long>(g.nb) * kMaxBlockBits + 31) / 32 + 2;
    g.chunks = static_cast<int>((g.words * 4 + kChunkBytes - 1) / kChunkBytes);
    return g;
}

struct EncWs {
    int16_t* coef;        // (B * nb, 64) quantised, zigzag
    uint32_t* ac_bits;    // (B * nb) AC code length of each block
    uint32_t* bit_off;    // (B * nb) first bit of each block in its image
    uint32_t* nbytes;     // (B) entropy-coded bytes before stuffing, padding included
    uint32_t* words;      // (B, words) big-endian bit stream, byte order as in the file
    uint32_t* ff;         // (B, chunks) 0xFF bytes per chunk, then their exclusive scan
};

size_t align256(size_t n) { return (n + 255) & ~static_cast<size_t>(255); }

size_t enc_ws_layout(const EncGeom& g, char* base, EncWs* w) {
    const long long n = static_cast<long long>(g.B) * g.nb;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char* p = base ? base + off : nullptr;
        off += align256(bytes);
        return p;
    };
    char* coef = take(128ull * n);
    char* ac = take(4ull * n);
    char* bo = take(4ull * n);
    char* nbytes = take(4ull * g.B);
    char* words = take(4ull * g.B * g.words);
    char* ff = take(4ull * g.B * g.chunks);
    if (w) {
        w->coef = reinterpret_cast<int16_t*>(coef);
        w->ac_bits = reinterpret_cast<uint32_t*>(ac);
        w->bit_off = reinterpret_cast<uint32_t*>(bo);
        w->nbytes = reinterpret_cast<uint32_t*>(nbytes);
        w->words = reinterpret_cast<uint32_t*>(words);
        w->ff = reinterpret_cast<uint32_t*>(ff);
    }
    return off;
}

// ------------------------------------------------------------------------------------------------------- pixels -> blocks
// libjpeg's rgb_ycc_convert: 16-bit fixed point; Cb / Cr round with 0.5 - epsilon so they stay below 256
__device__ __forceinline__ int to_y(const uint8_t* p) { return (19595 * p[0] + 38470 * p[1] + 7471 * p[2] + 32768) >> 16; }
__device__ __forceinline__ int to_c(const uint8_t* p, int cr) {
    return cr ? (32768 * p[0] - 27439 * p[1] - 5329 * p[2] + (128 << 16) + 32767) >> 16
              : (-11059 * p[0] - 21709 * p[1] + 32768 * p[2] + (128 << 16) + 32767) >> 16;
}

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// one pass of libjpeg's islow FDCT (jfdctint.c): 13-bit constants, PASS1_BITS = 2 extra bits kept after the rows
template <bool kRows>
__device__ __forceinline__ void fdct_1d(int* d) {
    constexpr int sh = kRows ? 13 - 2 : 13 + 2;
    const int t0 = d[0] + d[7], t7 = d[0] - d[7], t1 = d[1] + d[6], t6 = d[1] - d[6];
    const int t2 = d[2] + d[5], t5 = d[2] - d[5], t3 = d[3] + d[4], t4 = d[3] - d[4];
    const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    d[0] = kRows ? (t10 + t11) * 4 : descale(t10 + t11, 2);
    d[4] = kRows ? (t10 - t11) * 4 : descale(t10 - t11, 2);
    int z1 = (t12 + t13) * 4433;
    d[2] = descale(z1 + t13 * 6270, sh);
    d[6] = descale(z1 - t12 * 15137, sh);
    z1 = t4 + t7;
    int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
    const int z5 = (z3 + z4) * 9633;
    const int u4 = t4 * 2446, u5 = t5 * 16819, u6 = t6 * 25172, u7 = t7 * 12299;
    z1 *= -7373;
    z2 *= -20995;
    z3 = z3 * -16069 + z5;
    z4 = z4 * -3196 + z5;
    d[7] = descale(u4 + z1 + z3, sh);
    d[5] = descale(u5 + z2 + z4, sh);
    d[3] = descale(u6 + z2 + z3, sh);
    d[1] = descale(u7 + z1 + z4, sh);
}

__device__ __forceinline__ int nbits(int v) { return v ? 32 - __clz(v < 0 ? -v : v) : 0; }

__global__ void __launch_bounds__(kBlocksPerCta * 8) jpeg_enc_blocks(const uint8_t* __restrict__ x, const int32_t* __restrict__ tab,
                                                                      EncGeom g, EncWs w) {
    __shared__ int s[kBlocksPerCta][8][9];
    __shared__ __align__(16) int16_t q[kBlocksPerCta][64];
    const int lb = threadIdx.x >> 3, r = threadIdx.x & 7;
    const long long gb = static_cast<long long>(blockIdx.x) * kBlocksPerCta + lb;
    const bool live = gb < static_cast<long long>(g.B) * g.nb;
    const int img = live ? static_cast<int>(gb / g.nb) : 0, b = live ? static_cast<int>(gb % g.nb) : 0;
    const int mcu = b / 6, j = b - mcu * 6, mxi = mcu % g.mx, myi = mcu / g.mx;
    const int comp = j < 4 ? 0 : j - 3;
    const int bx = 2 * mxi + (j & 1), by = 2 * myi + (j >> 1);
    const bool dummy = !live || (j < 4 && (bx >= g.wb || by >= g.hb));
    const uint8_t* im = x + static_cast<long long>(img) * g.H * g.W * 3;
    int d[8];
    if (dummy) {
        for (int c = 0; c < 8; ++c) d[c] = 0;
    } else if (comp == 0) {                    // luma, edge-replicated to the block grid
        const uint8_t* row = im + static_cast<long long>(min(by * 8 + r, g.H - 1)) * g.W * 3;
#pragma unroll
        for (int c = 0; c < 8; ++c) d[c] = to_y(row + min(bx * 8 + c, g.W - 1) * 3) - 128;
    } else {                                   // h2v2: right edge replicated at full size, odd last row doubled, bias 1, 2, ...
        const int cy = min(myi * 8 + r, (g.H + 1) / 2 - 1);
        const uint8_t* r0 = im + static_cast<long long>(min(2 * cy, g.H - 1)) * g.W * 3;
        const uint8_t* r1 = im + static_cast<long long>(min(2 * cy + 1, g.H - 1)) * g.W * 3;
        const int cr = comp == 2;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int cx = mxi * 8 + c;
            const int c0 = min(2 * cx, g.W - 1) * 3, c1 = min(2 * cx + 1, g.W - 1) * 3;
            d[c] = ((to_c(r0 + c0, cr) + to_c(r0 + c1, cr) + to_c(r1 + c0, cr) + to_c(r1 + c1, cr) + 1 + (c & 1)) >> 2) - 128;
        }
    }
    fdct_1d<true>(d);
#pragma unroll
    for (int c = 0; c < 8; ++c) s[lb][r][c] = d[c];
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = s[lb][k][r];
    fdct_1d<false>(d);
#pragma unroll
    for (int k = 0; k < 8; ++k) s[lb][k][r] = d[k];
    __syncthreads();
    const int32_t* qt = tab + (comp ? kQuantInts : 0);
#pragma unroll
    for (int i = 0; i < 8; ++i) {              // libjpeg-turbo's reciprocal quantisation: (|v| + corr) * recip >> (16 + shift)
        const int k = r * 8 + i, nat = kNatural[k];
        const int v = s[lb][nat >> 3][nat & 7];
        const int a = static_cast<int>((static_cast<unsigned>(abs(v) + qt[64 + k]) * static_cast<unsigned>(qt[k])) >> (16 + qt[128 + k]));
        q[lb][k] = static_cast<int16_t>(dummy ? 0 : (v < 0 ? -a : a));
    }
    __syncthreads();
    if (!live) return;
    int16_t* out = w.coef + gb * 64;
    reinterpret_cast<int4*>(out)[r] = reinterpret_cast<const int4*>(q[lb])[r];
    if (r == 0) {                              // AC code length: run/size symbols, ZRL per 16 zeros, EOB unless k = 63 is nonzero
        const int32_t* ac = tab + kHuffBase + (comp ? 3 : 1) * 256;
        unsigned bits = 0;
        int run = 0;
        for (int k = 1; k < 64; ++k) {
            const int v = q[lb][k];
            if (v == 0) {
                ++run;
                continue;
            }
            bits += (run >> 4) * (ac[0xF0] >> 16);
            const int n = nbits(v);
            bits += (ac[(run & 15) << 4 | n] >> 16) + n;
            run = 0;
        }
        if (run) bits += ac[0] >> 16;
        w.ac_bits[gb] = bits;
    }
}

// ----------------------------------------------------------------------------------------------------- DC and the scan
// The quantised DC of block b of an image.  A luma block wholly outside the image is a dummy block (libjpeg's
// compress_data): zero AC and the DC of the block before it in the MCU -- the left neighbour at the right edge, the MCU's
// top-right block (itself resolved) at the bottom.
__device__ __forceinline__ int block_dc(const int16_t* coef, const EncGeom& g, int b) {
    const int mcu = b / 6;
    int j = b - mcu * 6;
    if (j < 4) {
        const int mxi = mcu % g.mx, myi = mcu / g.mx;
        const bool right = 2 * mxi + 1 >= g.wb, bottom = 2 * myi + 1 >= g.hb;
        if ((j >= 2 && bottom) || (j == 1 && right)) j = (j >= 2 && bottom) ? (right ? 0 : 1) : 0;
        else if (j == 3 && right) j = 2;
        return coef[static_cast<long long>(mcu * 6 + j) * 64];
    }
    return coef[static_cast<long long>(b) * 64];
}

// block b's DC difference: the previous block of its component in scan order (0 before the first)
__device__ __forceinline__ int dc_diff(const int16_t* coef, const EncGeom& g, int b) {
    const int j = b % 6;
    const int prev = j < 4 ? (j > 0 ? b - 1 : b - 3) : b - 6;
    return block_dc(coef, g, b) - (prev >= 0 ? block_dc(coef, g, prev) : 0);
}

// exclusive scan of v over the CTA (kScanThreads threads); *total gets the sum
__device__ __forceinline__ unsigned cta_exclusive_scan(unsigned v, unsigned* total) {
    __shared__ unsigned warp_sum[kScanThreads / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) warp_sum[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        unsigned s = warp_sum[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned t = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += t;
        }
        warp_sum[lane] = s;
    }
    __syncthreads();
    const unsigned base = wid ? warp_sum[wid - 1] : 0u;
    *total = warp_sum[kScanThreads / 32 - 1];
    __syncthreads();
    return base + inc - v;
}

__global__ void __launch_bounds__(kScanThreads) jpeg_enc_scan(const int32_t* __restrict__ tab, EncGeom g, EncWs w) {
    const int img = blockIdx.x;
    const int16_t* coef = w.coef + static_cast<long long>(img) * g.nb * 64;
    const uint32_t* ac = w.ac_bits + static_cast<long long>(img) * g.nb;
    uint32_t* off = w.bit_off + static_cast<long long>(img) * g.nb;
    const int per = (g.nb + kScanThreads - 1) / kScanThreads, lo = threadIdx.x * per, hi = min(lo + per, g.nb);
    unsigned sum = 0;
    for (int b = lo; b < hi; ++b) {
        const int n = nbits(dc_diff(coef, g, b));
        const int32_t* dc = tab + kHuffBase + (b % 6 < 4 ? 0 : 2) * 256;
        off[b] = ac[b] + (dc[n] >> 16) + n;    // the block's length, turned into its offset below
        sum += off[b];
    }
    unsigned total;
    unsigned pos = cta_exclusive_scan(sum, &total);
    for (int b = lo; b < hi; ++b) {
        const unsigned len = off[b];
        off[b] = pos;
        pos += len;
    }
    const unsigned nbytes = (total + 7) >> 3;
    if (threadIdx.x == 0) w.nbytes[img] = nbytes;
    uint32_t* words = w.words + img * g.words;
    for (long long i = threadIdx.x; i < (nbytes + 3) / 4 + 1; i += kScanThreads) words[i] = 0u;
}

// ------------------------------------------------------------------------------------------------------------- packing
struct BitWriter {
    uint32_t* words;
    unsigned long long acc = 0;
    int n = 0;
    unsigned pos;
    // 32 bits at bit position pos, as big-endian words stored in file byte order
    __device__ void emit32(uint32_t v, unsigned p) {
        const unsigned k = p >> 5, sh = p & 31;
        atomicOr(words + k, __byte_perm(v >> sh, 0, 0x0123));
        if (sh) atomicOr(words + k + 1, __byte_perm(v << (32 - sh), 0, 0x0123));
    }
    __device__ void put(uint32_t code, int len) {
        acc = (acc << len) | code;
        n += len;
        if (n >= 32) {
            n -= 32;
            emit32(static_cast<uint32_t>(acc >> n), pos);
            pos += 32;
        }
    }
    __device__ void flush() {
        if (n) emit32(static_cast<uint32_t>(acc << (32 - n)), pos);
    }
};

__global__ void __launch_bounds__(256) jpeg_enc_pack(const int32_t* __restrict__ tab, EncGeom g, EncWs w) {
    const long long gb = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (gb >= static_cast<long long>(g.B) * g.nb) return;
    const int img = static_cast<int>(gb / g.nb), b = static_cast<int>(gb % g.nb);
    const int16_t* coef = w.coef + static_cast<long long>(img) * g.nb * 64;
    const int chroma = b % 6 >= 4;
    const int32_t* dct = tab + kHuffBase + (chroma ? 2 : 0) * 256;
    const int32_t* act = dct + 256;
    BitWriter bw{w.words + img * g.words};
    bw.pos = w.bit_off[gb];
    const int diff = dc_diff(coef, g, b);
    int n = nbits(diff);
    bw.put(dct[n] & 0xFFFF, dct[n] >> 16);
    if (n) bw.put((diff < 0 ? diff - 1 : diff) & ((1u << n) - 1), n);
    const int16_t* blk = coef + static_cast<long long>(b) * 64;
    int run = 0;
    for (int k = 1; k < 64; ++k) {
        const int v = blk[k];
        if (v == 0) {
            ++run;
            continue;
        }
        for (; run > 15; run -= 16) bw.put(act[0xF0] & 0xFFFF, act[0xF0] >> 16);
        n = nbits(v);
        const int32_t c = act[run << 4 | n];
        bw.put(c & 0xFFFF, c >> 16);
        bw.put((v < 0 ? v - 1 : v) & ((1u << n) - 1), n);
        run = 0;
    }
    if (run) bw.put(act[0] & 0xFFFF, act[0] >> 16);
    if (b == g.nb - 1) {                       // pad the last byte with 1-bits
        const int pad = (8 - ((bw.pos + bw.n) & 7)) & 7;
        if (pad) bw.put((1u << pad) - 1, pad);
    }
    bw.flush();
}

// ------------------------------------------------------------------------------------------------------------ stuffing
__global__ void __launch_bounds__(256) jpeg_enc_count(EncGeom g, EncWs w) {
    const int img = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= g.chunks) return;
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(w.words + img * g.words);
    const unsigned nbytes = w.nbytes[img];
    unsigned cnt = 0;
    for (unsigned i = c * kChunkBytes, e = min(i + kChunkBytes, nbytes); i < e; ++i) cnt += bytes[i] == 0xFF;
    w.ff[static_cast<long long>(img) * g.chunks + c] = cnt;
}

__global__ void __launch_bounds__(kScanThreads) jpeg_enc_stuff_scan(EncGeom g, EncWs w, long long* sizes) {
    const int img = blockIdx.x;
    uint32_t* ff = w.ff + static_cast<long long>(img) * g.chunks;
    const int used = (w.nbytes[img] + kChunkBytes - 1) / kChunkBytes;
    const int per = (used + kScanThreads - 1) / kScanThreads, lo = threadIdx.x * per, hi = min(lo + per, used);
    unsigned sum = 0;
    for (int c = lo; c < hi; ++c) sum += ff[c];
    unsigned total;
    unsigned pos = cta_exclusive_scan(sum, &total);
    for (int c = lo; c < hi; ++c) {
        const unsigned v = ff[c];
        ff[c] = pos;
        pos += v;
    }
    if (threadIdx.x == 0) sizes[img] = static_cast<long long>(w.nbytes[img]) + total;
}

__global__ void __launch_bounds__(256) jpeg_enc_stuff(EncGeom g, EncWs w, const long long* sizes, uint8_t* out) {
    const int img = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
    __shared__ long long base;
    if (threadIdx.x == 0) {
        long long s = 0;
        for (int i = 0; i < img; ++i) s += sizes[i];
        base = s;
    }
    __syncthreads();
    const unsigned nbytes = w.nbytes[img];
    if (c >= g.chunks || static_cast<unsigned>(c) * kChunkBytes >= nbytes) return;
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(w.words + img * g.words);
    uint8_t* o = out + base + w.ff[static_cast<long long>(img) * g.chunks + c] + static_cast<long long>(c) * kChunkBytes;
    for (unsigned i = c * kChunkBytes, e = min(i + kChunkBytes, nbytes); i < e; ++i) {
        const uint8_t v = bytes[i];
        *o++ = v;
        if (v == 0xFF) *o++ = 0;
    }
}

bool enc_shape_ok(int B, int H, int W) {
    // bit offsets within an image are 32-bit
    return B > 0 && H > 0 && W > 0 && H < 65536 && W < 65536 &&
           static_cast<long long>((H + 15) / 16) * ((W + 15) / 16) * 6 * kMaxBlockBits < (1ll << 32) - 64;
}

}  // namespace
}  // namespace gifb200

using namespace gifb200;

extern "C" size_t gifb200_jpeg_encode_workspace_bytes(int B, int H, int W) {
    if (!enc_shape_ok(B, H, W)) return 0;
    return enc_ws_layout(enc_geom(B, H, W), nullptr, nullptr);
}

extern "C" size_t gifb200_jpeg_encode_out_bytes(int B, int H, int W) {
    if (!enc_shape_ok(B, H, W)) return 0;
    const EncGeom g = enc_geom(B, H, W);
    return 2ull * B * ((static_cast<unsigned long long>(g.nb) * kMaxBlockBits + 7) / 8 + 1);
}

extern "C" int gifb200_jpeg_encode(const uint8_t* x, const int32_t* tables, int B, int H, int W, uint8_t* out, long long* sizes,
                                   void* ws, size_t ws_bytes, gifb200_stream_t stream) {
    GIFB200_REQUIRE(enc_shape_ok(B, H, W), GIFB200_E_SHAPE, "jpeg_encode: B > 0, 0 < H, W < 65536, and an image's code bits below 2^32");
    const EncGeom g = enc_geom(B, H, W);
    GIFB200_REQUIRE(ws && ws_bytes >= enc_ws_layout(g, nullptr, nullptr), GIFB200_E_WORKSPACE,
                    "jpeg_encode: workspace smaller than gifb200_jpeg_encode_workspace_bytes");
    GIFB200_REQUIRE(x && tables && out && sizes, GIFB200_E_SHAPE, "jpeg_encode: NULL pointer");
    EncWs w;
    enc_ws_layout(g, static_cast<char*>(ws), &w);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long n = static_cast<long long>(B) * g.nb;
    jpeg_enc_blocks<<<cdiv(n, kBlocksPerCta), kBlocksPerCta * 8, 0, st>>>(x, tables, g, w);
    GIFB200_LAUNCH_CHECK("jpeg_enc_blocks");
    jpeg_enc_scan<<<B, kScanThreads, 0, st>>>(tables, g, w);
    GIFB200_LAUNCH_CHECK("jpeg_enc_scan");
    jpeg_enc_pack<<<cdiv(n, 256), 256, 0, st>>>(tables, g, w);
    GIFB200_LAUNCH_CHECK("jpeg_enc_pack");
    jpeg_enc_count<<<dim3(cdiv(g.chunks, 256), B), 256, 0, st>>>(g, w);
    GIFB200_LAUNCH_CHECK("jpeg_enc_count");
    jpeg_enc_stuff_scan<<<B, kScanThreads, 0, st>>>(g, w, sizes);
    GIFB200_LAUNCH_CHECK("jpeg_enc_stuff_scan");
    jpeg_enc_stuff<<<dim3(cdiv(g.chunks, 256), B), 256, 0, st>>>(g, w, sizes, out);
    GIFB200_LAUNCH_CHECK("jpeg_enc_stuff");
    return GIFB200_OK;
}
