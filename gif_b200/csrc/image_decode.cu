// Image decoding on the device: baseline JPEG (parallel entropy decode, islow IDCT, fancy upsampling, YCbCr->RGB), PNG scanline
// reconstruction, Pillow's bicubic resize and the [-1, 1] normalisation into NCHW batches.  The host side is
// gif_b200/image_decode.py: it parses markers / chunks, builds the tables, inflates PNG data and packs the descriptors.
#include "common.cuh"
#include "image_decode.cuh"

namespace gifb200 {
namespace {

using namespace img;

constexpr int kScanThreads = 256;
constexpr int kSweeps = 3;

struct JpegWs {
    unsigned long long *in, *out_a, *out_b;
    int32_t *nblk, *first_block, *dc_sum, *dc_off, *seg_lo, *seg_hi, *dc_local, *dc_chunk;
    int16_t* coef;
    uint8_t* planes;
};

size_t align256(size_t n) { return (n + 255) & ~static_cast<size_t>(255); }

size_t jpeg_ws_layout(int n_chunk, int n_seg, long long n_blocks, char* base, JpegWs* w) {
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char* p = base ? base + off : nullptr;
        off += align256(bytes);
        return p;
    };
    char* in = take(8ull * n_chunk);
    char* oa = take(8ull * n_chunk);
    char* ob = take(8ull * n_chunk);
    char* nb = take(4ull * n_chunk);
    char* fb = take(4ull * n_chunk);
    char* ds = take(12ull * n_chunk);
    char* dof = take(12ull * n_chunk);
    char* lo = take(4ull * n_seg);
    char* hi = take(4ull * n_seg);
    char* dl = take(4ull * n_blocks);
    char* dch = take(4ull * n_blocks);
    char* cf = take(128ull * n_blocks);
    char* pl = take(64ull * n_blocks);
    if (w) {
        w->in = reinterpret_cast<unsigned long long*>(in);
        w->out_a = reinterpret_cast<unsigned long long*>(oa);
        w->out_b = reinterpret_cast<unsigned long long*>(ob);
        w->nblk = reinterpret_cast<int32_t*>(nb);
        w->first_block = reinterpret_cast<int32_t*>(fb);
        w->dc_sum = reinterpret_cast<int32_t*>(ds);
        w->dc_off = reinterpret_cast<int32_t*>(dof);
        w->seg_lo = reinterpret_cast<int32_t*>(lo);
        w->seg_hi = reinterpret_cast<int32_t*>(hi);
        w->dc_local = reinterpret_cast<int32_t*>(dl);
        w->dc_chunk = reinterpret_cast<int32_t*>(dch);
        w->coef = reinterpret_cast<int16_t*>(cf);
        w->planes = reinterpret_cast<uint8_t*>(pl);
    }
    return off;
}

struct JpegArgs {
    const uint8_t* data;
    const int32_t *img, *seg, *chunk_seg, *qtab, *htab;
    int n_img, n_seg, n_chunk;
    uint32_t chunk_bits;
    uint8_t* out;
    int32_t* status;
};

// run of chunk c (relative index cl in its segment) from state s; stops at the chunk's end bit
__device__ __forceinline__ unsigned long long chunk_run(const JpegArgs& a, int c, unsigned long long s, int& nblk) {
    const int32_t* sg = a.seg + a.chunk_seg[c] * GIFB200_JPEG_SEG_INTS;
    const int32_t* d = a.img + sg[JS_IMG] * GIFB200_JPEG_DESC_INTS;
    const uint32_t nbits = static_cast<uint32_t>(sg[JS_NBYTES]) * 8u;
    const uint32_t cl = static_cast<uint32_t>(c - sg[JS_FIRST_CHUNK]);
    const uint32_t end = cl + 1 == static_cast<uint32_t>(sg[JS_NCHUNK]) ? nbits : (cl + 1) * a.chunk_bits;
    // after an invalid code the run starts over from the chunk's guessed state: a wrong guess that hit an invalid code must
    // not pass "invalid" on to every later chunk (the final chain still reports it: jpeg_scan_blocks)
    if (s == kInvalid) s = pack_state(cl * a.chunk_bits, 0, 0);
    return jpeg_run<false>(d, a.htab + sg[JS_IMG] * 4 * GIFB200_JPEG_HUFF_INTS, a.data + sg[JS_OFF], sg[JS_NBYTES], s, end,
                           nblk, nullptr);
}

// 1. every chunk decodes from a guessed state (bit = chunk start, first block of an MCU, DC next); exact for a segment's
//    first chunk
__global__ void __launch_bounds__(256) jpeg_sync_init(JpegArgs a, JpegWs w) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= a.n_chunk) return;
    const int32_t* sg = a.seg + a.chunk_seg[c] * GIFB200_JPEG_SEG_INTS;
    const unsigned long long s = pack_state(static_cast<uint32_t>(c - sg[JS_FIRST_CHUNK]) * a.chunk_bits, 0, 0);
    int nb;
    w.in[c] = s;
    w.out_a[c] = chunk_run(a, c, s, nb);
    w.nblk[c] = nb;
    if (c == sg[JS_FIRST_CHUNK]) {
        w.seg_lo[a.chunk_seg[c]] = 0x7fffffff;
        w.seg_hi[a.chunk_seg[c]] = -1;
    }
}

// 2. one synchronisation sweep: a chunk whose start state differs from its predecessor's end state decodes again
__global__ void __launch_bounds__(256) jpeg_sync_step(JpegArgs a, JpegWs w, const unsigned long long* src, unsigned long long* dst) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= a.n_chunk) return;
    const int32_t* sg = a.seg + a.chunk_seg[c] * GIFB200_JPEG_SEG_INTS;
    unsigned long long o = src[c];
    if (c != sg[JS_FIRST_CHUNK] && src[c - 1] != w.in[c]) {
        int nb;
        w.in[c] = src[c - 1];
        o = chunk_run(a, c, src[c - 1], nb);
        w.nblk[c] = nb;
    }
    dst[c] = o;
}

// 3. the chunks whose start state still differs from their predecessor's end state, per segment: [first, last]
__global__ void __launch_bounds__(256) jpeg_sync_check(JpegArgs a, JpegWs w, const unsigned long long* out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= a.n_chunk) return;
    const int sid = a.chunk_seg[c];
    if (c != a.seg[sid * GIFB200_JPEG_SEG_INTS + JS_FIRST_CHUNK] && out[c - 1] != w.in[c]) {
        atomicMin(w.seg_lo + sid, c);
        atomicMax(w.seg_hi + sid, c);
    }
}

// 4. a segment that is not yet consistent is finished in order from its first inconsistent chunk: past the last one, the
//    chain is consistent from the first chunk whose start state needs no change
__global__ void __launch_bounds__(128) jpeg_sync_fix(JpegArgs a, JpegWs w, unsigned long long* out) {
    const int sid = blockIdx.x * blockDim.x + threadIdx.x;
    if (sid >= a.n_seg || w.seg_hi[sid] < 0) return;
    const int32_t* sg = a.seg + sid * GIFB200_JPEG_SEG_INTS;
    const int end = sg[JS_FIRST_CHUNK] + sg[JS_NCHUNK];
    for (int c = w.seg_lo[sid]; c < end; ++c) {
        if (out[c - 1] == w.in[c]) {
            if (c > w.seg_hi[sid]) break;
            continue;
        }
        int nb;
        w.in[c] = out[c - 1];
        out[c] = chunk_run(a, c, out[c - 1], nb);
        w.nblk[c] = nb;
    }
}

// inclusive scan of one int per thread over a CTA of kScanThreads
__device__ int cta_scan(int v, int* sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < kScanThreads; o <<= 1) {
        const int t = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
        __syncthreads();
        sh[threadIdx.x] += t;
        __syncthreads();
    }
    const int r = sh[threadIdx.x];
    __syncthreads();
    return r;
}

// 5. per segment (one CTA): first decode-order block of every chunk, and the segment's verdict: every chunk decoded and the
//    blocks add up to the segment's MCUs
__global__ void __launch_bounds__(kScanThreads) jpeg_scan_blocks(JpegArgs a, JpegWs w, const unsigned long long* out) {
    __shared__ int sh[kScanThreads];
    const int32_t* sg = a.seg + blockIdx.x * GIFB200_JPEG_SEG_INTS;
    const int32_t* d = a.img + sg[JS_IMG] * GIFB200_JPEG_DESC_INTS;
    const int c0 = sg[JS_FIRST_CHUNK], n = sg[JS_NCHUNK];
    int carry = sg[JS_FIRST_MCU] * d[JD_BPM];
    for (int base = 0; base < n; base += kScanThreads) {
        const int c = c0 + base + threadIdx.x;
        const int v = base + threadIdx.x < n ? w.nblk[c] : 0;
        const int inc = cta_scan(v, sh);
        if (base + threadIdx.x < n) {
            w.first_block[c] = carry + inc - v;
            if (w.in[c] == kInvalid) atomicOr(a.status + sg[JS_IMG], 1);
        }
        sh[threadIdx.x] = inc;
        __syncthreads();
        carry += sh[kScanThreads - 1];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const int want = (sg[JS_FIRST_MCU] + sg[JS_NMCU]) * d[JD_BPM];
        const bool bad_code = out[c0 + n - 1] == kInvalid;
        if (bad_code || carry != want) atomicOr(a.status + sg[JS_IMG], bad_code ? 1 : 2);
    }
}

// 6. every chunk decodes again from its now exact start state, writing coefficients and chunk-local DC sums
__global__ void __launch_bounds__(256) jpeg_decode_chunks(JpegArgs a, JpegWs w) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= a.n_chunk) return;
    const int32_t* sg = a.seg + a.chunk_seg[c] * GIFB200_JPEG_SEG_INTS;
    const int32_t* d = a.img + sg[JS_IMG] * GIFB200_JPEG_DESC_INTS;
    const long long base = d[JD_BLOCK_BASE];
    JpegEmit em;
    em.coef = w.coef + base * 64;
    em.dc_local = w.dc_local + base;
    em.dc_chunk = w.dc_chunk + base;
    em.chunk = c;
    em.first_block = w.first_block[c];
    em.end_block = static_cast<long long>(sg[JS_FIRST_MCU] + sg[JS_NMCU]) * d[JD_BPM];
    const uint32_t nbits = static_cast<uint32_t>(sg[JS_NBYTES]) * 8u;
    const uint32_t cl = static_cast<uint32_t>(c - sg[JS_FIRST_CHUNK]);
    const uint32_t end = cl + 1 == static_cast<uint32_t>(sg[JS_NCHUNK]) ? nbits : (cl + 1) * a.chunk_bits;
    const unsigned long long s = w.in[c] == kInvalid ? pack_state(cl * a.chunk_bits, 0, 0) : w.in[c];
    int nb;
    jpeg_run<true>(d, a.htab + sg[JS_IMG] * 4 * GIFB200_JPEG_HUFF_INTS, a.data + sg[JS_OFF], sg[JS_NBYTES], s, end, nb, &em);
    for (int i = 0; i < 3; ++i) w.dc_sum[c * 3 + i] = em.dc_sum[i];
}

// 7. per segment (one CTA): DC prediction = exclusive scan of the chunks' DC sums per component (restarts reset it)
__global__ void __launch_bounds__(kScanThreads) jpeg_scan_dc(JpegArgs a, JpegWs w) {
    __shared__ int sh[kScanThreads];
    const int32_t* sg = a.seg + blockIdx.x * GIFB200_JPEG_SEG_INTS;
    const int c0 = sg[JS_FIRST_CHUNK], n = sg[JS_NCHUNK];
    for (int comp = 0; comp < 3; ++comp) {
        int carry = 0;
        for (int base = 0; base < n; base += kScanThreads) {
            const int c = c0 + base + threadIdx.x;
            const int v = base + threadIdx.x < n ? w.dc_sum[c * 3 + comp] : 0;
            const int inc = cta_scan(v, sh);
            if (base + threadIdx.x < n) w.dc_off[c * 3 + comp] = carry + inc - v;
            sh[threadIdx.x] = inc;
            __syncthreads();
            carry += sh[kScanThreads - 1];
            __syncthreads();
        }
    }
}

// 8. DC values, then the islow IDCT of every block into the component's sample grid
__global__ void __launch_bounds__(128) jpeg_idct(JpegArgs a, JpegWs w) {
    const int32_t* d = a.img + blockIdx.y * GIFB200_JPEG_DESC_INTS;
    const long long base = d[JD_BLOCK_BASE];
    const int nb = d[JD_NBLOCKS], ncomp = d[JD_NCOMP];
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < nb; p += gridDim.x * blockDim.x) {
        int comp = 0;
        while (comp + 1 < ncomp && p >= d[JD_CBASE0 + comp + 1]) ++comp;
        int16_t blk[64];
        const int16_t* src = w.coef + (base + p) * 64;
        for (int i = 0; i < 64; ++i) blk[i] = src[i];
        const int ch = w.dc_chunk[base + p];
        if (ch >= 0) blk[0] = static_cast<int16_t>(w.dc_local[base + p] + w.dc_off[ch * 3 + comp]);
        idct_islow(blk, a.qtab + (blockIdx.y * 3 + comp) * 64, w.planes + (base + p) * 64);
    }
}

// 9. upsampling + colour conversion -> uint8 RGB (H, W, 3)
__global__ void __launch_bounds__(256) jpeg_color(JpegArgs a, JpegWs w) {
    const int32_t* d = a.img + blockIdx.y * GIFB200_JPEG_DESC_INTS;
    const int W = d[JD_W], H = d[JD_H], ncomp = d[JD_NCOMP];
    const uint8_t* planes = w.planes + static_cast<long long>(d[JD_BLOCK_BASE]) * 64;
    uint8_t* out = a.out + static_cast<unsigned>(d[JD_OUT_OFF]);
    const int hs = d[JD_HMAX], vs = d[JD_VMAX];
    const int cw = (W + hs - 1) / hs, ch = (H + vs - 1) / vs;
    for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < static_cast<long long>(W) * H;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int x = static_cast<int>(e % W), y = static_cast<int>(e / W);
        const int Y = plane_at(planes, d[JD_BW0], x, y);
        uint8_t* o = out + e * 3;
        if (ncomp == 1) {
            o[0] = o[1] = o[2] = static_cast<uint8_t>(Y);
        } else {
            const int cb = chroma_at(planes + d[JD_CBASE0 + 1] * 64ll, d[JD_BW0 + 1], cw, ch, hs, vs, x, y);
            const int cr = chroma_at(planes + d[JD_CBASE0 + 2] * 64ll, d[JD_BW0 + 2], cw, ch, hs, vs, x, y);
            ycc_to_rgb(Y, cb, cr, o);
        }
    }
}

// PNG: one CTA per image reconstructs scanlines in place.  Row r of a band of blockDim rows works on byte tile s - r at
// step s, so the row above (tile t and t-1) is always complete: a diagonal wavefront, one __syncthreads per step.
constexpr int kPngTile = 64;
__global__ void __launch_bounds__(256) png_unfilter_kernel(uint8_t* data, const int32_t* desc, int32_t* status) {
    const int32_t* d = desc + blockIdx.x * GIFB200_PNG_DESC_INTS;
    uint8_t* img = data + static_cast<unsigned>(d[0]);
    const int W = d[1], H = d[2], bpp = d[3];
    const int rowbytes = W * bpp, stride = rowbytes + 1, ntiles = (rowbytes + kPngTile - 1) / kPngTile;
    for (int band = 0; band < H; band += blockDim.x) {
        const int r = band + threadIdx.x;
        uint8_t* cur = img + static_cast<long long>(r) * stride;
        int f = r < H ? cur[0] : 0;
        if (f > 4) {
            atomicOr(status + blockIdx.x, 4);
            f = 0;
        }
        const int nrows = H - band < static_cast<int>(blockDim.x) ? H - band : blockDim.x;
        for (int s = 0; s < ntiles + nrows - 1; ++s) {
            const int t = s - static_cast<int>(threadIdx.x);
            if (r < H && t >= 0 && t < ntiles) {
                const int i1 = (t + 1) * kPngTile < rowbytes ? (t + 1) * kPngTile : rowbytes;
                png_unfilter_span(cur + 1, r > 0 ? cur + 1 - stride : nullptr, f, bpp, t * kPngTile, i1);
            }
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(256) png_to_rgb_kernel(const uint8_t* data, const int32_t* desc, uint8_t* out) {
    const int32_t* d = desc + blockIdx.y * GIFB200_PNG_DESC_INTS;
    const uint8_t* img = data + static_cast<unsigned>(d[0]);
    const int W = d[1], H = d[2], bpp = d[3];
    uint8_t* o = out + static_cast<unsigned>(d[4]);
    for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < static_cast<long long>(W) * H;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int x = static_cast<int>(e % W), y = static_cast<int>(e / W);
        const uint8_t* p = img + static_cast<long long>(y) * (W * bpp + 1) + 1 + x * bpp;
        o[e * 3 + 0] = p[0];
        o[e * 3 + 1] = bpp >= 3 ? p[1] : p[0];
        o[e * 3 + 2] = bpp >= 3 ? p[2] : p[0];
    }
}

// Pillow's two-pass resample: horizontal (B, Hi, Wi, 3) -> tmp (B, Hi, Wo, 3), vertical tmp -> (B, Ho, Wo, 3).
// coef rows: [xmin, n, k_0 .. k_{ks-1}]
__global__ void __launch_bounds__(256) resize_h_kernel(const uint8_t* x, uint8_t* y, const int32_t* coef, int B, int H, int Wi,
                                                      int Wo, int ks) {
    const long long n = static_cast<long long>(B) * H * Wo;
    for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < n;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int xo = static_cast<int>(e % Wo);
        const long long row = e / Wo;
        const int32_t* k = coef + xo * (ks + 2);
        const uint8_t* src = x + (row * Wi + k[0]) * 3;
        for (int c = 0; c < 3; ++c) y[e * 3 + c] = resample_tap(src + c, 3, k + 2, k[1]);
    }
}

__global__ void __launch_bounds__(256) resize_v_kernel(const uint8_t* x, uint8_t* y, const int32_t* coef, int B, int Hi, int Ho,
                                                      int W, int ks) {
    const long long n = static_cast<long long>(B) * Ho * W;
    for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < n;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int xx = static_cast<int>(e % W), yo = static_cast<int>((e / W) % Ho), b = static_cast<int>(e / (static_cast<long long>(W) * Ho));
        const int32_t* k = coef + yo * (ks + 2);
        const uint8_t* src = x + ((static_cast<long long>(b) * Hi + k[0]) * W + xx) * 3;
        for (int c = 0; c < 3; ++c) y[e * 3 + c] = resample_tap(src + c, 3ll * W, k + 2, k[1]);
    }
}

// (v / 255 - 0.5) / 0.5 in IEEE float32, as ToTensor + Normalize compute it; NHWC uint8 -> channel planes of an NCHW batch
__global__ void __launch_bounds__(256) u8_to_unit_kernel(const uint8_t* x, float* y, int B, int HW, long long y_stride) {
    const long long n = static_cast<long long>(B) * HW;
    for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < n;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int p = static_cast<int>(e % HW), b = static_cast<int>(e / HW);
        float* o = y + b * y_stride + p;
        for (int c = 0; c < 3; ++c) o[static_cast<long long>(c) * HW] = __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(x[e * 3 + c]), 255.f), 0.5f), 0.5f);
    }
}

// The inverse direction, as the reference saves generated images (my_utils/generic_utils.py:134-164 after the
// clamp to [-1, 1] of the sampling scripts): uint8(clip(fl(fl(a + 1) * 0.5), 0, 1) * 255) in float32, truncated, with
// a = clamp(x, -1, 1).  The explicit round-to-nearest intrinsics keep nvcc from contracting the steps into an FMA.
// x is any strided (B, 3, H, W) float32 view; y is dense (B, H, W, 3).  NaN inputs are outside the contract.
__global__ void __launch_bounds__(256) image_to_u8_kernel(const float* x, uint8_t* y, int B, int H, int W, long long sb,
                                                          long long sc, long long sh, long long sw) {
    const long long HW = static_cast<long long>(H) * W, n = B * HW;
    for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < n;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long b = e / HW, p = e - b * HW, h = p / W, w = p - h * W;
        const float* src = x + b * sb + h * sh + w * sw;
        for (int c = 0; c < 3; ++c) {
            const float a = fminf(fmaxf(src[c * sc], -1.f), 1.f);
            const float t = fminf(fmaxf(__fmul_rn(__fadd_rn(a, 1.f), 0.5f), 0.f), 1.f);
            y[e * 3 + c] = static_cast<uint8_t>(static_cast<int>(__fmul_rn(t, 255.f)));
        }
    }
}

int grid_for(long long n) {
    int blocks = cdiv(n, 256);
    return blocks > kNumSMs * 16 ? kNumSMs * 16 : (blocks < 1 ? 1 : blocks);
}

}  // namespace
}  // namespace gifb200

using namespace gifb200;

extern "C" size_t gifb200_jpeg_workspace_bytes(int n_chunk, int n_seg, long long n_blocks) {
    if (n_chunk < 1 || n_seg < 1 || n_blocks < 1) return 0;
    return jpeg_ws_layout(n_chunk, n_seg, n_blocks, nullptr, nullptr);
}

extern "C" int gifb200_jpeg_decode(const uint8_t* data, const int32_t* img_desc, const int32_t* seg_desc, const int32_t* chunk_seg,
                                   const int32_t* qtab, const int32_t* htab, int n_img, int n_seg, int n_chunk, long long n_blocks,
                                   int max_blocks, int chunk_bytes, uint8_t* out, int32_t* status, void* ws,
                                   size_t ws_bytes, gifb200_stream_t stream) {
    GIFB200_REQUIRE(n_img > 0 && n_seg >= n_img && n_chunk >= n_seg && n_blocks > 0 && max_blocks > 0, GIFB200_E_SHAPE,
                    "jpeg_decode: needs images, segments (>= 1 per image), chunks (>= 1 per segment) and blocks");
    GIFB200_REQUIRE(chunk_bytes >= 16 && chunk_bytes <= (1 << 20), GIFB200_E_SHAPE, "jpeg_decode: chunk_bytes in [16, 1 MiB]");
    const size_t need = jpeg_ws_layout(n_chunk, n_seg, n_blocks, nullptr, nullptr);
    GIFB200_REQUIRE(ws && ws_bytes >= need, GIFB200_E_WORKSPACE, "jpeg_decode: workspace smaller than gifb200_jpeg_workspace_bytes");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    JpegWs w;
    jpeg_ws_layout(n_chunk, n_seg, n_blocks, static_cast<char*>(ws), &w);
    JpegArgs a{data, img_desc, seg_desc, chunk_seg, qtab, htab, n_img, n_seg, n_chunk, static_cast<uint32_t>(chunk_bytes) * 8u, out, status};
    if (cudaMemsetAsync(w.coef, 0, 128ull * n_blocks, st) != cudaSuccess ||
        cudaMemsetAsync(w.dc_chunk, 0xff, 4ull * n_blocks, st) != cudaSuccess)
        return fail(GIFB200_E_CUDA, "jpeg_decode: cudaMemsetAsync", cudaGetErrorString(cudaGetLastError()));
    const int gc = cdiv(n_chunk, 256);
    jpeg_sync_init<<<gc, 256, 0, st>>>(a, w);
    GIFB200_LAUNCH_CHECK("jpeg_sync_init");
    // a sweep re-decodes only the chunks whose start state changed, so the later sweeps are cheap; whatever is still
    // inconsistent after them (a run of chunks none of which fell into step) is finished in order by jpeg_sync_fix
    unsigned long long *src = w.out_a, *dst = w.out_b;
    for (int i = 0; i < kSweeps; ++i) {
        jpeg_sync_step<<<gc, 256, 0, st>>>(a, w, src, dst);
        GIFB200_LAUNCH_CHECK("jpeg_sync_step");
        unsigned long long* t = src;
        src = dst;
        dst = t;
    }
    jpeg_sync_check<<<gc, 256, 0, st>>>(a, w, src);
    GIFB200_LAUNCH_CHECK("jpeg_sync_check");
    jpeg_sync_fix<<<cdiv(n_seg, 128), 128, 0, st>>>(a, w, src);
    GIFB200_LAUNCH_CHECK("jpeg_sync_fix");
    jpeg_scan_blocks<<<n_seg, kScanThreads, 0, st>>>(a, w, src);
    GIFB200_LAUNCH_CHECK("jpeg_scan_blocks");
    jpeg_decode_chunks<<<gc, 256, 0, st>>>(a, w);
    GIFB200_LAUNCH_CHECK("jpeg_decode_chunks");
    jpeg_scan_dc<<<n_seg, kScanThreads, 0, st>>>(a, w);
    GIFB200_LAUNCH_CHECK("jpeg_scan_dc");
    const int gx = cdiv(max_blocks, 128) < kNumSMs * 4 ? cdiv(max_blocks, 128) : kNumSMs * 4;
    jpeg_idct<<<dim3(gx, n_img), 128, 0, st>>>(a, w);
    GIFB200_LAUNCH_CHECK("jpeg_idct");
    const int gp = cdiv(64ll * max_blocks, 256) < kNumSMs * 4 ? cdiv(64ll * max_blocks, 256) : kNumSMs * 4;
    jpeg_color<<<dim3(gp, n_img), 256, 0, st>>>(a, w);
    GIFB200_LAUNCH_CHECK("jpeg_color");
    return GIFB200_OK;
}

extern "C" int gifb200_png_unfilter(uint8_t* data, const int32_t* desc, int n_img, int max_pixels, uint8_t* out, int32_t* status,
                                    gifb200_stream_t stream) {
    GIFB200_REQUIRE(n_img > 0 && max_pixels > 0, GIFB200_E_SHAPE, "png_unfilter: needs images");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    png_unfilter_kernel<<<n_img, 256, 0, st>>>(data, desc, status);
    GIFB200_LAUNCH_CHECK("png_unfilter_kernel");
    const int gp = cdiv(max_pixels, 256) < kNumSMs * 4 ? cdiv(max_pixels, 256) : kNumSMs * 4;
    png_to_rgb_kernel<<<dim3(gp, n_img), 256, 0, st>>>(data, desc, out);
    GIFB200_LAUNCH_CHECK("png_to_rgb_kernel");
    return GIFB200_OK;
}

extern "C" int gifb200_resize_bicubic_u8(const uint8_t* x, uint8_t* tmp, uint8_t* y, const int32_t* coef_h, const int32_t* coef_v,
                                         int B, int Hi, int Wi, int Ho, int Wo, int ks_h, int ks_v, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B > 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0, GIFB200_E_SHAPE, "resize_bicubic_u8: positive sizes");
    GIFB200_REQUIRE((coef_h ? ks_h > 0 : Wo == Wi) && (coef_v ? ks_v > 0 : Ho == Hi) && (tmp || !coef_h || !coef_v),
                    GIFB200_E_SHAPE, "resize_bicubic_u8: a skipped pass keeps its axis; a pass needs taps; two passes need tmp");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!coef_h && !coef_v) {
        if (cudaMemcpyAsync(y, x, 3ull * B * Hi * Wi, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
            return fail(GIFB200_E_CUDA, "resize_bicubic_u8: cudaMemcpyAsync", cudaGetErrorString(cudaGetLastError()));
        return GIFB200_OK;
    }
    if (coef_h) {
        resize_h_kernel<<<grid_for(static_cast<long long>(B) * Hi * Wo), 256, 0, st>>>(x, coef_v ? tmp : y, coef_h, B, Hi, Wi, Wo, ks_h);
        GIFB200_LAUNCH_CHECK("resize_h_kernel");
    }
    if (coef_v) {
        resize_v_kernel<<<grid_for(static_cast<long long>(B) * Ho * Wo), 256, 0, st>>>(coef_h ? tmp : x, y, coef_v, B, Hi, Ho, Wo, ks_v);
        GIFB200_LAUNCH_CHECK("resize_v_kernel");
    }
    return GIFB200_OK;
}

extern "C" int gifb200_u8_to_unit(const uint8_t* x, float* y, int B, int H, int W, long long y_batch_stride, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B > 0 && H > 0 && W > 0 && y_batch_stride >= 3ll * H * W, GIFB200_E_SHAPE,
                    "u8_to_unit: positive sizes and a batch stride of at least 3*H*W");
    u8_to_unit_kernel<<<grid_for(static_cast<long long>(B) * H * W), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, B, H * W,
                                                                                                                 y_batch_stride);
    GIFB200_LAUNCH_CHECK("u8_to_unit_kernel");
    return GIFB200_OK;
}

extern "C" int gifb200_image_to_u8(const float* x, uint8_t* y, int B, int H, int W, long long stride_b, long long stride_c,
                                   long long stride_h, long long stride_w, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B > 0 && H > 0 && W > 0, GIFB200_E_SHAPE, "image_to_u8: positive sizes");
    image_to_u8_kernel<<<grid_for(static_cast<long long>(B) * H * W), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, y, B, H, W, stride_b, stride_c, stride_h, stride_w);
    GIFB200_LAUNCH_CHECK("image_to_u8_kernel");
    return GIFB200_OK;
}
