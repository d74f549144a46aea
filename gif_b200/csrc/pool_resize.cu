// gifb200_pool2d, gifb200_resize_bilinear and gifb200_resize_bilinear_u8: the pooling layers and the input resize of the FID
// InceptionV3.
#include "common.cuh"

namespace gifb200 {
namespace {

// one thread per output element (b, yo, xo, c); 3x3 window, channels-last in, channel slice [c0, c0+C) of Cy out
__global__ void __launch_bounds__(256) pool2d_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int Hi, int Wi,
                                                     int C, int Ho, int Wo, int stride, int pad, int op, int Cy, int c0,
                                                     int rtf32) {
    const long long n = static_cast<long long>(B) * Ho * Wo * C;
    for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c = static_cast<int>(e % C);
        const long long pix = e / C;
        const int xo = static_cast<int>(pix % Wo), yo = static_cast<int>((pix / Wo) % Ho), b = static_cast<int>(pix / (static_cast<long long>(Wo) * Ho));
        const float* xb = x + static_cast<long long>(b) * Hi * Wi * C + c;
        float acc = op == 0 ? -INFINITY : 0.f;
        int cnt = 0;
        for (int dy = 0; dy < 3; ++dy) {
            const int yi = yo * stride - pad + dy;
            if (yi < 0 || yi >= Hi) continue;
            for (int dx = 0; dx < 3; ++dx) {
                const int xi = xo * stride - pad + dx;
                if (xi < 0 || xi >= Wi) continue;
                const float v = __ldg(xb + (static_cast<long long>(yi) * Wi + xi) * C);
                acc = op == 0 ? fmaxf(acc, v) : acc + v;
                ++cnt;
            }
        }
        if (op == 1) acc /= static_cast<float>(cnt);        // count_include_pad=False: padded cells are not counted
        y[pix * Cy + c0 + c] = rtf32 ? round_tf32(acc) : acc;
    }
}

// torch's source index for align_corners=False: (dst + 0.5) * scale - 0.5, clamped at 0.  In double: a float coordinate
// (torch's float32 kernel) is off by up to 1e-5 of a pixel at 1024 -> 299, which moves the result by ~1e-5.
__device__ __forceinline__ void src_index(int d, double scale, int in, int& i0, int& i1, float& l1) {
    double s = (d + 0.5) * scale - 0.5;
    if (s < 0.0) s = 0.0;
    i0 = static_cast<int>(s);
    if (i0 > in - 1) i0 = in - 1;
    i1 = i0 < in - 1 ? i0 + 1 : i0;
    l1 = static_cast<float>(s - i0);
}

// v / 255 in float32 for every byte, rounded to nearest as numpy's float32 `/= 255` (IEEE division), evaluated at compile
// time: a division in the kernel brings its slow-path call, and with it a stack frame and spills.
struct U8Unit {
    float v[256];
    constexpr U8Unit() : v() {
        for (int i = 0; i < 256; ++i) v[i] = static_cast<float>(i) / 255.f;
    }
};
__device__ constexpr U8Unit kU8Unit{};

// a source sample as the float kernel sees it: fp32 as stored; uint8 as v / 255
__device__ __forceinline__ float load_src(const float* p) { return __ldg(p); }
__device__ __forceinline__ float load_src(const uint8_t* p) { return __ldg(kU8Unit.v + __ldg(p)); }

// x (B,3,H,W) through element strides -> y (B,Ho,Wo,Cy) channels-last, channels 3..Cy-1 zero; v -> a*v + b.  Both source
// types run the same arithmetic after load_src, so the uint8 result is bitwise the float kernel's on x / 255.
template <typename T>
__global__ void __launch_bounds__(256) resize_kernel(const T* __restrict__ x, float* __restrict__ y, int B, int H, int W,
                                                     long long sb, long long sc, long long sh, long long sw, int Ho, int Wo,
                                                     int Cy, float a, float bb, int rtf32) {
    const long long n = static_cast<long long>(B) * Ho * Wo;
    const double sy = static_cast<double>(H) / Ho, sx = static_cast<double>(W) / Wo;
    for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int xo = static_cast<int>(e % Wo), yo = static_cast<int>((e / Wo) % Ho), b = static_cast<int>(e / (static_cast<long long>(Wo) * Ho));
        int y0, y1, x0, x1;
        float ly, lx;
        src_index(yo, sy, H, y0, y1, ly);
        src_index(xo, sx, W, x0, x1, lx);
        float* dst = y + e * Cy;
        for (int c = 0; c < 3; ++c) {
            const T* p = x + b * sb + c * sc;
            const float v00 = load_src(p + y0 * sh + x0 * sw), v01 = load_src(p + y0 * sh + x1 * sw);
            const float v10 = load_src(p + y1 * sh + x0 * sw), v11 = load_src(p + y1 * sh + x1 * sw);
            const float v = (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
            const float o = a * v + bb;
            dst[c] = rtf32 ? round_tf32(o) : o;
        }
        for (int c = 3; c < Cy; ++c) dst[c] = 0.f;
    }
}

}  // namespace
}  // namespace gifb200

using namespace gifb200;

extern "C" int gifb200_pool2d(const float* x, float* y, int B, int Hi, int Wi, int C, int Ho, int Wo, int stride, int pad,
                              int op, int Cy, int c0, int round_tf32, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B > 0 && Hi > 0 && Wi > 0 && C > 0 && Ho > 0 && Wo > 0 && (op == 0 || op == 1) && (stride == 1 || stride == 2) &&
                        (pad == 0 || pad == 1) && c0 >= 0 && c0 + C <= Cy,
                    GIFB200_E_SHAPE, "pool2d: 3x3 window, stride 1 or 2, pad 0 or 1, op 0 (max) or 1 (avg), c0 + C <= Cy");
    GIFB200_REQUIRE((Ho - 1) * stride + 3 <= Hi + 2 * pad && (Wo - 1) * stride + 3 <= Wi + 2 * pad, GIFB200_E_SHAPE,
                    "pool2d: output larger than the padded input allows");
    const long long n = static_cast<long long>(B) * Ho * Wo * C;
    int blocks = cdiv(n, 256);
    if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
    pool2d_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, B, Hi, Wi, C, Ho, Wo, stride, pad, op, Cy, c0,
                                                                        round_tf32);
    GIFB200_LAUNCH_CHECK("pool2d_kernel");
    return GIFB200_OK;
}

extern "C" int gifb200_resize_bilinear(const float* x, float* y, int B, int H, int W, long long stride_b, long long stride_c,
                                       long long stride_h, long long stride_w, int Ho, int Wo, int Cy, float scale, float shift,
                                       int round_tf32, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && Cy >= 3, GIFB200_E_SHAPE,
                    "resize_bilinear: positive sizes and Cy >= 3");
    const long long n = static_cast<long long>(B) * Ho * Wo;
    int blocks = cdiv(n, 256);
    if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
    resize_kernel<float><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, B, H, W, stride_b, stride_c, stride_h,
                                                                               stride_w, Ho, Wo, Cy, scale, shift, round_tf32);
    GIFB200_LAUNCH_CHECK("resize_kernel");
    return GIFB200_OK;
}

extern "C" int gifb200_resize_bilinear_u8(const uint8_t* x, float* y, int B, int H, int W, long long stride_b, int Ho, int Wo,
                                          int Cy, float scale, float shift, int round_tf32, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && Cy >= 3, GIFB200_E_SHAPE,
                    "resize_bilinear_u8: positive sizes and Cy >= 3");
    const long long n = static_cast<long long>(B) * Ho * Wo;
    int blocks = cdiv(n, 256);
    if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
    resize_kernel<uint8_t><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, B, H, W, stride_b, 1, 3ll * W, 3, Ho, Wo,
                                                                                 Cy, scale, shift, round_tf32);
    GIFB200_LAUNCH_CHECK("resize_kernel<u8>");
    return GIFB200_OK;
}
