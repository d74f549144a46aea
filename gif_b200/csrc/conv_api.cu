// gifb200_conv2d / gifb200_conv2d_wgrad: shape checks and dispatch between the tensor-core and the SIMT kernels.
#include "common.cuh"

namespace gifb200 {
int conv2d_simt(const float* x, const float* w, float* y, int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k,
                int mode, int flip, int transposed, const ConvEpilogue& epi, cudaStream_t st);
int conv2d_wgrad_simt(const float* x, const float* gy, float* gw, int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co,
                      int k, int mode, int flip, int transposed, cudaStream_t st);
// conv_tc.cu
bool conv2d_tc_supported(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode);
size_t conv2d_tc_workspace_bytes(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode, int transposed);
int conv2d_tc(const float* x, const float* w, float* y, int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k,
              int mode, int flip, int transposed, const ConvEpilogue& epi, void* ws, size_t ws_bytes, cudaStream_t st,
              bool x3, bool prestaged);
// conv_wgrad_tc.cu
bool conv2d_wgrad_tc_supported(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode);
size_t conv2d_wgrad_tc_workspace_bytes(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode);
int conv2d_wgrad_tc(const float* x, const float* gy, float* gw, int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co,
                    int k, int mode, int flip, int transposed, void* ws, size_t ws_bytes, cudaStream_t st, bool x3);
}  // namespace gifb200

using namespace gifb200;

extern "C" size_t gifb200_conv2d_workspace_bytes(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode,
                                                 int transposed, int impl) {
    impl &= 0xF;
    if (impl == 1) return 0;
    if (!conv2d_tc_supported(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode)) return 0;
    return conv2d_tc_workspace_bytes(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, transposed);
}

extern "C" int gifb200_conv2d(const float* x, const float* w, float* y, int B, int Hi, int Wi, int Ci, int Ho, int Wo,
                              int Co, int k, int mode, int flip, int transposed, int impl, int act, const float* bias,
                              float slope, float gain, int round_tf32, void* workspace, size_t workspace_bytes,
                              gifb200_stream_t stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const ConvEpilogue epi{act, bias, slope, gain, round_tf32};
    const bool prestaged = (impl & GIFB200_CONV_PRESTAGED) != 0;
    impl &= 0xF;
    GIFB200_REQUIRE(impl >= 0 && impl <= 3, GIFB200_E_SHAPE,
                    "conv2d: impl must be 0 (auto), 1 (simt), 2 (wgmma tf32) or 3 (wgmma bf16x3 on split planes)");
    const bool tc_ok = conv2d_tc_supported(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode);
    if (impl >= 2 && !tc_ok) return fail(GIFB200_E_SHAPE, "conv2d: shape not supported by the tensor-core path");
    if (impl != 1 && tc_ok)
        return conv2d_tc(x, w, y, B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, flip, transposed, epi, workspace, workspace_bytes, st,
                         impl == 3, prestaged);
    return conv2d_simt(x, w, y, B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, flip, transposed, epi, st);
}

// > 0 exactly when the tensor-core path will be taken (split-K partial sums live in the workspace)
extern "C" size_t gifb200_conv2d_wgrad_workspace_bytes(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k,
                                                       int mode, int impl) {
    if (impl == 1) return 0;
    return conv2d_wgrad_tc_workspace_bytes(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode);
}

extern "C" int gifb200_conv2d_wgrad_path(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode, int impl) {
    if (impl == 1) return 1;
    if (conv2d_wgrad_tc_supported(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode)) return impl == 3 ? 3 : 2;
    return impl == 0 ? 1 : 0;
}

extern "C" int gifb200_conv2d_wgrad(const float* x, const float* gy, float* gw, int B, int Hi, int Wi, int Ci, int Ho,
                                    int Wo, int Co, int k, int mode, int flip, int transposed, int impl, void* workspace,
                                    size_t workspace_bytes, gifb200_stream_t stream) {
    GIFB200_REQUIRE(impl >= 0 && impl <= 3, GIFB200_E_SHAPE, "conv2d_wgrad: impl must be 0, 1, 2 or 3");
    const bool tc_ok = conv2d_wgrad_tc_supported(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode);
    if (impl >= 2 && !tc_ok) return fail(GIFB200_E_SHAPE, "conv2d_wgrad: shape not supported by the tensor-core path");
    if (impl != 1 && tc_ok)
        return conv2d_wgrad_tc(x, gy, gw, B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, flip, transposed, workspace,
                               workspace_bytes, static_cast<cudaStream_t>(stream), impl == 3);
    return conv2d_wgrad_simt(x, gy, gw, B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, flip, transposed,
                             static_cast<cudaStream_t>(stream));
}
