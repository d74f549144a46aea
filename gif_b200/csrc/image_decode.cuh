// Per-thread pieces of the image decoders (image_decode.cu): baseline-JPEG entropy decoding, libjpeg's integer "islow" IDCT,
// its fancy chroma upsampling and YCbCr->RGB, PNG scanline unfiltering and Pillow's fixed-point bicubic resampling.  They are
// __host__ __device__ so a host program can run them on the same inputs as the kernels.
#pragma once
#include <stdint.h>

#include "gifb200.h"

#ifndef __CUDACC__
#define __host__
#define __device__
#define __forceinline__ inline
#endif

namespace gifb200 {
namespace img {

// ---------------------------------------------------------------------------------------------------------------- JPEG
// Descriptor fields (int32 per image, GIFB200_JPEG_DESC_INTS of them), written by gif_b200/image_decode.py.
enum JpegDesc {
    JD_W = 0, JD_H, JD_NCOMP, JD_HMAX, JD_VMAX, JD_MCUX, JD_MCUY, JD_BPM, JD_BLOCK_BASE, JD_NBLOCKS, JD_OUT_OFF,
    JD_H0, JD_V0 = JD_H0 + 3, JD_BW0 = JD_V0 + 3, JD_CBASE0 = JD_BW0 + 3, JD_DCT0 = JD_CBASE0 + 3, JD_ACT0 = JD_DCT0 + 3,
    JD_BLK0 = JD_ACT0 + 3,      // 10 entries: comp | dx << 4 | dy << 8 of each block of an MCU, in decode order
    JD_END = JD_BLK0 + 10
};
// Segment descriptor (int32 x GIFB200_JPEG_SEG_INTS): one entropy-coded segment (a restart interval, or the whole scan).
enum JpegSeg { JS_IMG = 0, JS_OFF, JS_NBYTES, JS_FIRST_MCU, JS_NMCU, JS_FIRST_CHUNK, JS_NCHUNK };
// Huffman table (int32 x GIFB200_JPEG_HUFF_INTS): 9-bit lookahead (len << 8 | symbol, 0 = longer code), then maxcode[18],
// valoff[18] (symbol index - code for each length), vals[256].  Four per image: DC0, DC1, AC0, AC1.
constexpr int kLook = 9, kHuffLook = 0, kHuffMax = 512, kHuffOff = 530, kHuffVals = 548;

constexpr unsigned long long kInvalid = ~0ull;   // decoding state after an invalid code
__host__ __device__ __forceinline__ unsigned long long pack_state(uint32_t pos, int blk, int k) {
    return (static_cast<unsigned long long>(pos) << 16) | (static_cast<unsigned long long>(blk) << 8) | static_cast<unsigned>(k);
}

// 32 bits of the segment starting at bit p (big-endian bit order); bytes past the end read as zero
__host__ __device__ __forceinline__ uint32_t peek32(const uint8_t* seg, int nbytes, uint32_t p) {
    const int b = static_cast<int>(p >> 3);
    unsigned long long w = 0;
    for (int i = 0; i < 5; ++i) w = (w << 8) | (b + i < nbytes ? seg[b + i] : 0u);
    return static_cast<uint32_t>(w >> (8 - (p & 7)));
}

// one Huffman symbol at the top of win: returns the symbol (its length in len), or -1 for a code no table entry matches
__host__ __device__ __forceinline__ int huff_decode(const int32_t* t, uint32_t win, int& len) {
    const int e = t[kHuffLook + (win >> (32 - kLook))];
    if (e) {
        len = e >> 8;
        return e & 255;
    }
    for (int l = kLook + 1; l <= 16; ++l) {
        const int code = static_cast<int>(win >> (32 - l));
        if (code <= t[kHuffMax + l]) {
            len = l;
            return t[kHuffVals + ((code + t[kHuffOff + l]) & 255)];
        }
    }
    return -1;
}

__host__ __device__ __forceinline__ int huff_extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

// libjpeg's jpeg_natural_order, with its 16 extra entries: a run that overshoots coefficient 63 lands on 63
__host__ __device__ __forceinline__ int natural_order(int k) {
    constexpr unsigned char z[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
    return k > 63 ? 63 : z[k];
}

// decode-order block b of an image -> its component and its index in the image's block grid (component grids one after another)
__host__ __device__ __forceinline__ int block_locate(const int32_t* d, long long b, int& comp) {
    const int bpm = d[JD_BPM];
    const int m = static_cast<int>(b / bpm), j = static_cast<int>(b % bpm);
    if (d[JD_NCOMP] == 1) {
        comp = 0;
        return m;
    }
    const int info = d[JD_BLK0 + j];
    comp = info & 15;
    const int bx = (m % d[JD_MCUX]) * d[JD_H0 + comp] + ((info >> 4) & 15);
    const int by = (m / d[JD_MCUX]) * d[JD_V0 + comp] + (info >> 8);
    return d[JD_CBASE0 + comp] + by * d[JD_BW0 + comp] + bx;
}

// Outputs of one run of the entropy decoder when it writes coefficients.
struct JpegEmit {
    int16_t* coef;           // the image's block grid, 64 coefficients per block
    int32_t* dc_local;       // per block: DC differences summed from the start of the run (per component)
    int32_t* dc_chunk;       // per block: the chunk whose run decoded its DC
    int chunk;
    long long first_block;   // decode-order index of the block in progress at the run's start
    long long end_block;     // blocks at and after this index are not written (the segment's end)
    int32_t dc_sum[3];       // out: DC differences of the run per component
};

// Entropy-decode from state s until the bit position reaches `end` (or the segment's bits run out mid-symbol).  Returns the
// state at the first symbol boundary at or after `end`, kInvalid after an invalid code; nblk counts the blocks completed.
// This is the step function of the self-synchronising decode: a run from a guessed state usually reaches the same state as
// a run from the true one within a few symbols.
template <bool EMIT>
__host__ __device__ unsigned long long jpeg_run(const int32_t* d, const int32_t* htab, const uint8_t* seg, int nbytes,
                                                unsigned long long s, uint32_t end, int& nblk, JpegEmit* em) {
    nblk = 0;
    if (s == kInvalid) return kInvalid;
    uint32_t pos = static_cast<uint32_t>(s >> 16);
    int blk = static_cast<int>((s >> 8) & 255), k = static_cast<int>(s & 255);
    const uint32_t nbits = static_cast<uint32_t>(nbytes) * 8u;
    const int bpm = d[JD_BPM], ncomp = d[JD_NCOMP];
    long long b = EMIT ? em->first_block : 0;
    int comp = ncomp == 1 ? 0 : (d[JD_BLK0 + blk] & 15);
    int gidx = 0;
    bool bad = false;
    int dc0 = 0, dc1 = 0, dc2 = 0;      // scalars, not an array: a dynamic index would put them in local memory
    if (EMIT && b < em->end_block) gidx = block_locate(d, b, comp);
    while (pos < end) {
        const uint32_t win = peek32(seg, nbytes, pos);
        const int32_t* t = htab + (k == 0 ? d[JD_DCT0 + comp] : 2 + d[JD_ACT0 + comp]) * GIFB200_JPEG_HUFF_INTS;
        int len = 0;
        const int sym = huff_decode(t, win, len);
        if (sym < 0) {                  // near the end the window holds zeros past the data: the padding ends the segment
            bad = nbits - pos >= 16;
            break;
        }
        const int sbits = sym & 15;
        if (pos + len + (k == 0 ? sym : sbits) > nbits) break;          // the segment ends inside this symbol
        const int v = (k == 0 ? sym : sbits) ? static_cast<int>((win << len) >> (32 - (k == 0 ? sym : sbits))) : 0;
        if (k == 0) {
            const int diff = sym ? huff_extend(v, sym) : 0;
            pos += len + sym;
            if (EMIT && b < em->end_block) {
                int& acc = comp == 0 ? dc0 : (comp == 1 ? dc1 : dc2);
                acc += diff;
                em->dc_local[gidx] = acc;
                em->dc_chunk[gidx] = em->chunk;
            }
            k = 1;
        } else {
            const int r = sym >> 4;
            pos += len + sbits;
            if (sbits) {
                k += r;
                if (EMIT && b < em->end_block) em->coef[gidx * 64ll + natural_order(k)] = static_cast<int16_t>(huff_extend(v, sbits));
                ++k;
            } else {
                k = r == 15 ? k + 16 : 64;
            }
        }
        if (k >= 64) {
            k = 0;
            ++nblk;
            if (++blk == bpm) blk = 0;
            if (ncomp > 1) comp = d[JD_BLK0 + blk] & 15;
            if (EMIT && ++b < em->end_block) gidx = block_locate(d, b, comp);
        }
    }
    if (EMIT) {
        em->dc_sum[0] = dc0;
        em->dc_sum[1] = dc1;
        em->dc_sum[2] = dc2;
    }
    return bad ? kInvalid : pack_state(pos, blk, k);
}

// jidctint.c jpeg_idct_islow (64-bit JLONG arithmetic), dequantisation included; out = 8x8 samples after range_limit.
__host__ __device__ inline void idct_islow(const int16_t* in, const int32_t* q, uint8_t* out) {
    constexpr long long F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
                        F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
    int ws[64];
    for (int c = 0; c < 8; ++c) {
        long long z1, z2, z3, z4, z5, t0, t1, t2, t3, t10, t11, t12, t13;
        z2 = static_cast<long long>(in[16 + c]) * q[16 + c];
        z3 = static_cast<long long>(in[48 + c]) * q[48 + c];
        z1 = (z2 + z3) * F0541;
        t2 = z1 + z3 * -F1847;
        t3 = z1 + z2 * F0765;
        z2 = static_cast<long long>(in[c]) * q[c];
        z3 = static_cast<long long>(in[32 + c]) * q[32 + c];
        t0 = (z2 + z3) * 8192;
        t1 = (z2 - z3) * 8192;
        t10 = t0 + t3; t13 = t0 - t3; t11 = t1 + t2; t12 = t1 - t2;
        t0 = static_cast<long long>(in[56 + c]) * q[56 + c];
        t1 = static_cast<long long>(in[40 + c]) * q[40 + c];
        t2 = static_cast<long long>(in[24 + c]) * q[24 + c];
        t3 = static_cast<long long>(in[8 + c]) * q[8 + c];
        z1 = t0 + t3; z2 = t1 + t2; z3 = t0 + t2; z4 = t1 + t3;
        z5 = (z3 + z4) * F1175;
        t0 *= F0298; t1 *= F2053; t2 *= F3072; t3 *= F1501;
        z1 *= -F0899; z2 *= -F2562; z3 *= -F1961; z4 *= -F0390;
        z3 += z5; z4 += z5;
        t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
        ws[c] = static_cast<int>((t10 + t3 + 1024) >> 11);
        ws[56 + c] = static_cast<int>((t10 - t3 + 1024) >> 11);
        ws[8 + c] = static_cast<int>((t11 + t2 + 1024) >> 11);
        ws[48 + c] = static_cast<int>((t11 - t2 + 1024) >> 11);
        ws[16 + c] = static_cast<int>((t12 + t1 + 1024) >> 11);
        ws[40 + c] = static_cast<int>((t12 - t1 + 1024) >> 11);
        ws[24 + c] = static_cast<int>((t13 + t0 + 1024) >> 11);
        ws[32 + c] = static_cast<int>((t13 - t0 + 1024) >> 11);
    }
    for (int r = 0; r < 8; ++r) {
        const int* w = ws + r * 8;
        long long z1, z2, z3, z4, z5, t0, t1, t2, t3, t10, t11, t12, t13;
        z2 = w[2]; z3 = w[6];
        z1 = (z2 + z3) * F0541;
        t2 = z1 + z3 * -F1847;
        t3 = z1 + z2 * F0765;
        t0 = (static_cast<long long>(w[0]) + w[4]) * 8192;
        t1 = (static_cast<long long>(w[0]) - w[4]) * 8192;
        t10 = t0 + t3; t13 = t0 - t3; t11 = t1 + t2; t12 = t1 - t2;
        t0 = w[7]; t1 = w[5]; t2 = w[3]; t3 = w[1];
        z1 = t0 + t3; z2 = t1 + t2; z3 = t0 + t2; z4 = t1 + t3;
        z5 = (z3 + z4) * F1175;
        t0 *= F0298; t1 *= F2053; t2 *= F3072; t3 *= F1501;
        z1 *= -F0899; z2 *= -F2562; z3 *= -F1961; z4 *= -F0390;
        z3 += z5; z4 += z5;
        t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
        const long long o[8] = {t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3};
        for (int c = 0; c < 8; ++c) {
            // range_limit[x & RANGE_MASK]: the 10-bit wrap of the descaled value, read as signed, plus CENTERJSAMPLE, clamped
            int v = static_cast<int>((o[c] + (1ll << 17)) >> 18) & 1023;
            if (v >= 512) v -= 1024;
            v += 128;
            out[r * 8 + c] = static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
        }
    }
}

// sample (x, y) of a component stored as its block grid (8x8 samples per block, row-major blocks, bw blocks per row)
__host__ __device__ __forceinline__ int plane_at(const uint8_t* p, int bw, int x, int y) {
    return p[((static_cast<long long>(y >> 3) * bw + (x >> 3)) << 6) + ((y & 7) << 3) + (x & 7)];
}

// libjpeg-turbo's chroma upsampling (jdsample.c) at output pixel (x, y) of a chroma plane of cw x ch samples: fancy
// (triangle) h2v1 / h2v2 when cw > 2, plain replication otherwise, h1v2 always fancy; edges replicate.
// h1v2 (luma 1x2, 4:4:0) has no bit-exact test: Pillow cannot write such a file.
__host__ __device__ inline int chroma_at(const uint8_t* p, int bw, int cw, int ch, int hs, int vs, int x, int y) {
    if (hs == 1 && vs == 1) return plane_at(p, bw, x, y);
    const int cx = hs == 2 ? x >> 1 : x, cy = vs == 2 ? y >> 1 : y;
    if (hs == 1) {                         // h1v2
        const int oy = (y & 1) ? (cy + 1 < ch ? cy + 1 : cy) : (cy > 0 ? cy - 1 : 0);
        return (3 * plane_at(p, bw, cx, cy) + plane_at(p, bw, cx, oy) + ((y & 1) ? 2 : 1)) >> 2;
    }
    if (cw <= 2) return plane_at(p, bw, cx, cy);
    const int ox = (x & 1) ? (cx + 1 < cw ? cx + 1 : cx) : (cx > 0 ? cx - 1 : 0);
    if (vs == 1)                           // h2v1
        return (3 * plane_at(p, bw, cx, cy) + plane_at(p, bw, ox, cy) + ((x & 1) ? 2 : 1)) >> 2;
    const int oy = (y & 1) ? (cy + 1 < ch ? cy + 1 : cy) : (cy > 0 ? cy - 1 : 0);     // h2v2
    const int a = 3 * plane_at(p, bw, cx, cy) + plane_at(p, bw, cx, oy);
    const int o = 3 * plane_at(p, bw, ox, cy) + plane_at(p, bw, ox, oy);
    return (3 * a + o + ((x & 1) ? 7 : 8)) >> 4;
}

__host__ __device__ __forceinline__ uint8_t clamp255(int v) { return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// jdcolor.c ycc_rgb_convert with its tables (SCALEBITS = 16) evaluated inline
__host__ __device__ __forceinline__ void ycc_to_rgb(int y, int cb, int cr, uint8_t* rgb) {
    constexpr long long kCrR = 91881, kCbB = 116130, kCrG = 46802, kCbG = 22554, kHalf = 1 << 15;
    const long long xb = cb - 128, xr = cr - 128;
    rgb[0] = clamp255(y + static_cast<int>((kCrR * xr + kHalf) >> 16));
    rgb[1] = clamp255(y + static_cast<int>((-kCbG * xb + kHalf + -kCrG * xr) >> 16));
    rgb[2] = clamp255(y + static_cast<int>((kCbB * xb + kHalf) >> 16));
}

// ----------------------------------------------------------------------------------------------------------------- PNG
__host__ __device__ __forceinline__ int paeth(int a, int b, int c) {
    const int p = a + b - c;
    const int pa = p > a ? p - a : a - p, pb = p > b ? p - b : b - p, pc = p > c ? p - c : c - p;
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// undo the filter of bytes [i0, i1) of one scanline in place; up = the reconstructed row above (NULL for the first row)
__host__ __device__ inline void png_unfilter_span(uint8_t* cur, const uint8_t* up, int f, int bpp, int i0, int i1) {
    for (int i = i0; i < i1; ++i) {
        const int a = i >= bpp ? cur[i - bpp] : 0, b = up ? up[i] : 0, c = (up && i >= bpp) ? up[i - bpp] : 0;
        int p = 0;
        switch (f) {
            case 1: p = a; break;
            case 2: p = b; break;
            case 3: p = (a + b) >> 1; break;
            case 4: p = paeth(a, b, c); break;
            default: break;
        }
        cur[i] = static_cast<uint8_t>(cur[i] + p);
    }
}

// ------------------------------------------------------------------------------------------------------ bicubic resize
// Pillow's ImagingResample 8-bit pass: coefficients k (22-bit fixed point) over taps [xmin, xmin + n) of a line of samples
// `step` bytes apart; rounding bias 1 << 21, then clip8.
__host__ __device__ __forceinline__ uint8_t resample_tap(const uint8_t* src, long long step, const int32_t* k, int n) {
    int ss = 1 << 21;
    for (int i = 0; i < n; ++i) ss += static_cast<int>(src[i * step]) * k[i];
    return ss < 0 ? 0 : (ss >= (1 << 30) ? 255 : static_cast<uint8_t>(ss >> 22));
}

}  // namespace img
}  // namespace gifb200
