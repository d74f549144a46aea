/* gifb200.h -- C ABI of libgifb200.so: the H100 (sm_90a) kernels behind GIF's StyleGAN2 / rasteriser hot path.
 *
 * Boundary rules (SURVEY.md 8b):
 *   - plain `extern "C"`, device pointers + int shapes + a `cudaStream_t` (passed as void*); no torch types;
 *   - the caller owns every buffer (inputs, outputs, workspaces); functions never allocate, never synchronise
 *     the stream, never throw; return 0 on success or a negative GIFB200_E_* code, with a human readable
 *     message available from gifb200_last_error() (thread-local);
 *   - all activations are fp32, channels-last: x[b][y][x][c] ("NHWC"), dense.  Weights for the convolution
 *     entry points are "tap-major": w[t][r][s] with t = kh*k + kw (see gifb200_conv2d).
 *   - every entry point cites the reference interface it replaces (paths relative to the reference repo;
 *     cl.py = model/stylegan2_common_layers.py).
 *
 * The reference has no FFI layer of its own for the StyleGAN2 ops (they are Python, cl.py:14-16 has the CUDA op
 * imports commented out); the Python binding a maintainer adds is shown in INTEGRATION.md
 * (gif_b200/_lib.py is that binding).  For the rasteriser the reference binding is pybind11
 * (my_utils/standard_rasterize_cuda/standard_rasterize_cuda.cpp:79-82).
 */
#ifndef GIFB200_H
#define GIFB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GIFB200_OK 0
#define GIFB200_E_SHAPE (-1)     /* unsupported / inconsistent shape argument                       */
#define GIFB200_E_ALIGN (-2)     /* pointer or channel count not aligned as the kernel requires     */
#define GIFB200_E_ARCH (-3)      /* device is not sm_90 / driver entry point missing               */
#define GIFB200_E_CUDA (-4)      /* CUDA runtime / driver error (message has the CUDA error string) */
#define GIFB200_E_WORKSPACE (-5) /* workspace too small                                              */

typedef void* gifb200_stream_t; /* a cudaStream_t */

/* ---- library ------------------------------------------------------------------------------------------ */
int gifb200_version(void);
const char* gifb200_last_error(void);
/* number of kernel launches issued through this library by the calling process since load (bench.py's
 * "gpu_launches" is the difference of this counter across the timed region) */
long long gifb200_launch_count(void);

/* ---- convolution (dense 3x3 / 1x1 contraction) -------------------------------------------------------
 * Replaces: F.conv2d / F.conv_transpose2d inside ModulatedConv2d.forward (cl.py:307-349, in the
 * modulate-input / shared-weight form of SURVEY A3), EqualConv2d.forward (cl.py:175-184), the three
 * nn.Conv2d of NoiseInjection (cl.py:405-414) and their autograd (backward + double backward).
 *
 *   mode 0 (S1): stride 1, zero pad k/2        y[b,yo,xo,o] = sum_{t,i} x[b, yo+kh-k/2, xo+kw-k/2, i] * W[t,o,i]
 *   mode 1 (S2): stride 2, no pad              y[b,yo,xo,o] = sum_{t,i} x[b, 2yo+kh, 2xo+kw, i]     * W[t,o,i]
 *                (Hi >= 2*Ho + k - 2; D's downsampling convs, cl.py:765-786)
 *   mode 2 (T2): transposed stride 2, no pad   y[b,Y,X,o]   = sum_{t,i: Y-kh, X-kw even} x[b,(Y-kh)/2,(X-kw)/2,i] * W[t,o,i]
 *                (Ho = 2*Hi + k - 2; G's upsampling modconv, cl.py:322-331)
 *
 * Logical weights W[t,o,i] are addressed inside the physical buffer w[T][R][S] (T = k*k):
 *     tt = flip ? T-1-t : t;   W[t,o,i] = transposed ? w[tt][i][o] (R = Ci, S = Co) : w[tt][o][i] (R = Co, S = Ci)
 * so that the adjoint (input-gradient) of every mode is another call on the SAME weight buffer:
 *     adj(S1, flip, tr) = (S1, !flip, !tr);  adj(S2, flip, tr) = (T2, flip, !tr);  adj(T2, flip, tr) = (S2, flip, !tr).
 *
 * impl: 0 = auto (tensor-core path when the shape qualifies, else SIMT), 1 = force SIMT fp32,
 *       2 = force the tensor-core path (wgmma tf32, fp32 accumulate; returns GIFB200_E_SHAPE if the shape does not qualify),
 *       3 = tensor-core ERROR-COMPENSATED contraction ("bf16x3", fp32 accumulate): every operand is the two-term bf16
 *           expansion v = hi + lo written by gifb200_split_bf16 and the kernel accumulates hi*hi + hi*lo + lo*hi into the
 *           same fp32 accumulator (16 significant operand bits, ~1e-5 relative; 1.5x the tensor work of tf32).
 *           With impl 3, `x` is NOT an fp32 tensor but the planes buffer of gifb200_split_bf16 for the input
 *           (2 x B*Hi*Wi*Ci bf16 = the same number of bytes); w stays fp32 (split while staging).  Same shapes as impl 2.
 * workspace: gifb200_conv2d_workspace_bytes(...) bytes of device memory (may be 0 / NULL): the staged B operand, followed --
 *   for layers whose output tiles cannot fill the machine (4x4 / 8x8 at batch 32) -- by the partial accumulators of the
 *   split-K schedule (summed in a fixed order by a reduction pass that also applies the epilogue: deterministic).
 * Fused epilogue (ConvLayer = EqualConv2d -> FusedLeakyReLU, cl.py:752-799; nn.Conv2d + ReLU of NoiseInjection):
 *     y = lrelu(acc + bias[o], slope) * gain, optionally rounded to tf32;  act == 0 writes the plain accumulator
 *     (bias / slope / gain / round_tf32 ignored).
 *
 * GIFB200_CONV_PRESTAGED (OR-ed into impl, tensor-core paths only): the workspace still holds what an earlier call with the
 * SAME (w contents, flip, transposed, impl) left there -- the staged B operand -- so the staging pass is skipped.  Weights
 * change once per optimiser step but are used by 3-5 convolutions per step (D runs three forwards and two backwards): the
 * caller keeps one workspace per (weight, variant) and sets the flag while the weight is unchanged. */
#define GIFB200_CONV_PRESTAGED 0x10
size_t gifb200_conv2d_workspace_bytes(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode,
                                      int transposed, int impl);
int gifb200_conv2d(const float* x, const float* w, float* y, int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co,
                   int k, int mode, int flip, int transposed, int impl, int act, const float* bias, float slope,
                   float gain, int round_tf32, void* workspace, size_t workspace_bytes, gifb200_stream_t stream);

/* Weight gradient of gifb200_conv2d for the same (mode, flip, transposed), written in the PHYSICAL layout of w
 * (so it can be accumulated into / compared with the weight buffer directly):
 *     gW[t,o,i] = sum_{b,pixels} gy[b,p_out,o] * x[b,p_in(p_out,t),i]   (p_in as in the mode's formula above)
 * x is the conv input (B,Hi,Wi,Ci), gy the conv output gradient (B,Ho,Wo,Co).  gw is OVERWRITTEN.
 * Replaces autograd's conv weight gradient for the reference modules listed above.
 * impl: 0 auto, 1 SIMT fp32, 2 wgmma tf32 on the channels-last operands (MN-major tiles), 3 = bf16x3 compensated
 * contraction: BOTH x and gy are planes buffers of gifb200_split_bf16 (see gifb200_conv2d). */
size_t gifb200_conv2d_wgrad_workspace_bytes(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode,
                                            int impl);
/* which kernel gifb200_conv2d_wgrad will run for this shape / impl request: 1 or 2 as above (0: request not possible).
 * Path 2 needs tf32-rounded operands (see round_tf32 below); path 1 is exact fp32. */
int gifb200_conv2d_wgrad_path(int B, int Hi, int Wi, int Ci, int Ho, int Wo, int Co, int k, int mode, int impl);
int gifb200_conv2d_wgrad(const float* x, const float* gy, float* gw, int B, int Hi, int Wi, int Ci, int Ho, int Wo,
                         int Co, int k, int mode, int flip, int transposed, int impl, void* workspace,
                         size_t workspace_bytes, gifb200_stream_t stream);

/* Two-term bf16 expansion of an fp32 tensor (B, P pixels, C channels, channels-last), optionally fused with the style
 * modulation of ModulatedConv2d (cl.py:311-313 in the modulate-input form): v = x[b,p,c] * (s ? s[b,c] : 1);
 *     planes[0][b,p,c] = bf16_rn(v);   planes[1][b,p,c] = bf16_rn(v - planes[0][b,p,c])
 * planes: 2 * B*P*C bf16 (16-byte aligned).  The operand format of impl 3 above.  C % 4 == 0. */
int gifb200_split_bf16(const float* x, const float* s, void* planes, int B, int P, int C, gifb200_stream_t stream);

/* ---- upfirdn2d ---------------------------------------------------------------------------------------
 * Replaces upfirdn2d (cl.py:42-72) and through it Blur (cl.py:136-152), Upsample (cl.py:94-112),
 * Downsample (cl.py:115-133); its adjoint is the same entry point (SURVEY A1):
 *     out[b,y,x,c] = sum_{a,b'} K[a,b'] * U[y*down + (kh-1-a) - pad_y0, x*down + (kw-1-b') - pad_x0]
 * with U = input with (up-1) zeros inserted after every sample, zero outside; K = flip ? kernel reversed in
 * both axes : kernel.  Negative pads crop.  The output size (Ho,Wo) is given by the caller
 * (forward: (H*up + pad0 + pad1 - kh)/down + 1; adjoint: the forward's input size).
 * kernel: kh*kw floats on the device, kh,kw <= 8.  C % 4 == 0 takes the vectorised path. */
int gifb200_upfirdn2d(const float* x, const float* kernel, float* y, int B, int Hi, int Wi, int C, int Ho, int Wo,
                      int kh, int kw, int up, int down, int pad_y0, int pad_x0, int flip, int round_tf32,
                      gifb200_stream_t stream);

/* ---- fused bias / demodulation / noise-add / leaky-ReLU -----------------------------------------------
 * Replaces FusedLeakyReLU.forward (cl.py:32-39), the tail of StyledConv.forward (cl.py:479-486: demodulate,
 * NoiseInjection add, bias, activation), ScaledLeakyReLU (cl.py:238-247) and plain bias adds:
 *     t = x[b,p,c] * rowscale[b,c] + add[b,p,c] + bias[c];   y = (t > 0 ? t : slope*t) * gain
 * rowscale, add, bias may each be NULL.  rows = B*P pixels in total, P pixels per sample.
 * round_tf32 (here and below): != 0 rounds the OUTPUT to tf32 (round-to-nearest-away, cvt.rna) -- set by the caller
 * when the consumer is a wgmma tf32 contraction, which truncates its operands: pre-rounded operands make
 * that truncation exact and the contraction unbiased. */
int gifb200_bias_act(const float* x, const float* rowscale, const float* add, const float* bias, float* y, int B,
                     int P, int C, float slope, float gain, int round_tf32, gifb200_stream_t stream);
/* Backward of the activation given the OUTPUT y:  gx = gy * gain * (y > 0 ? 1 : slope)  (second derivative is
 * zero a.e., so this is also its own double-backward rule, SURVEY A4). n = number of elements. */
int gifb200_act_bwd(const float* gy, const float* y, float* gx, long long n, float slope, float gain,
                    int round_tf32, gifb200_stream_t stream);
/* out[g,c] = sum_{r<rows} x[g,r,c]  (bias gradients: G = 1; per-sample reductions: G = B). out is OVERWRITTEN. */
int gifb200_rows_sum(const float* x, float* out, int G, int rows, int C, gifb200_stream_t stream);
/* y[b,p,c] = x[b,p,c] * s[b,c]  -- style modulation of the conv INPUT (cl.py:311-312 moved to the activation),
 * demodulation of the conv OUTPUT (cl.py:315-316).  round_tf32 != 0 rounds y to tf32 (round-to-nearest) so that
 * the wgmma tf32 contraction, which truncates, sees exactly representable operands. */
int gifb200_chan_scale(const float* x, const float* s, float* y, int B, int P, int C, int round_tf32,
                       gifb200_stream_t stream);
/* Fused first-order backward passes (used when no second derivative is requested; the composable primitives above remain
 * the definition).  tail_bwd: backward of t = acc*d[b,c] + add + bias[c], y = lrelu(t)*gain given (gy, y, acc):
 *   gt = gy*gain*(y>0?1:slope) (= grad of add, of the noise branch), gacc = gt*d (may be NULL), gb[c] = sum gt (may be
 *   NULL), gd[b,c] = sum_p gt*acc (may be NULL; d == NULL means d = 1).  Replaces act_bwd + chan_scale + spatial_dot +
 *   rows_sum (autograd of cl.py:479-486).  scale_bwd: backward of y = x*s[b,c]: gx = gy*s, gs[b,c] = sum_p gy*x. */
int gifb200_tail_bwd(const float* gy, const float* y, const float* acc, const float* d, float* gt, float* gacc, float* gb,
                     float* gd, int B, int P, int C, float slope, float gain, int round_tf32, gifb200_stream_t stream);
int gifb200_scale_bwd(const float* gy, const float* x, const float* s, float* gx, float* gs, int B, int P, int C,
                      int round_tf32, gifb200_stream_t stream);
/* gifb200_tail_bwd for the bf16x3 mode: gt_planes / gacc_planes (each may be NULL) receive the two-term bf16 expansion
 * (the layout of gifb200_split_bf16) of gt / gacc in the SAME pass -- the operands of the convolution input-gradient and
 * weight-gradient that follow -- and the fp32 outputs gt / gacc may then be NULL (one of gt / gt_planes / gacc is required).
 * C % 32 == 0. */
int gifb200_tail_bwd_planes(const float* gy, const float* y, const float* acc, const float* d, float* gt, float* gacc,
                            float* gb, float* gd, int B, int P, int C, float slope, float gain, void* gt_planes,
                            void* gacc_planes, gifb200_stream_t stream);
/* Second-order pass of tail_bwd / scale_bwd (the path-length regulariser differentiates a recorded first-order backward;
 * reference rule: losses.py:102-124 through cl.py:479-486 / cl.py:311-316).  With m = gain*(y>0 ? 1 : slope) (y == NULL:
 * m = 1, the modulation variant) the first-order map is gacc = gy*m*d[b,c], gd[b,c] = sum_p gy*m*acc; given the upstream
 * gradients gg (of gacc; may be NULL) and ggd (of gd, (B,C); may be NULL) this writes in one pass
 *   ggy = m*(gg*d + ggd*acc)  (may be NULL),  gx2 = gy*m*ggd  (w.r.t. acc; may be NULL),  gdd[b,c] = sum_p gg*gy*m  (w.r.t.
 *   d; may be NULL; OVERWRITTEN).  ggy_planes (may be NULL; C % 32 == 0): the bf16x3 expansion of ggy in the same pass. */
int gifb200_tail_bwd2(const float* gg, const float* ggd, const float* gy, const float* y, const float* acc, const float* d,
                      float* ggy, float* gx2, float* gdd, int B, int P, int C, float slope, float gain, void* ggy_planes,
                      gifb200_stream_t stream);
/* One Adam step (torch.optim.Adam, no weight decay / amsgrad: train.py:365-382, stepped at train.py:160 and :246) over
 * ``count`` fp32 tensors given as HOST arrays of device pointers (read during the call): params, grads, first and second
 * moments, per-tensor step counters (0-d device floats, the layout of torch's capturable Adam), element counts.  Each
 * counter is incremented on the device first, then used for the bias corrections (a captured CUDA graph advances it on
 * replay).  The hyper-parameters are doubles (python floats in torch: 1 - beta2 must not be taken from a float beta2).
 * Two launches per 64 tensors.  The caller owns autograd's version counters of the parameters (raw pointer writes). */
int gifb200_adam_step(float* const* params, const float* const* grads, float* const* exp_avg, float* const* exp_avg_sq,
                      float* const* steps, const long long* numel, int count, double lr, double beta1, double beta2, double eps,
                      gifb200_stream_t stream);
/* out[b,c] = sum_p a[b,p,c] * b2[b,p,c]  (gradient of chan_scale w.r.t. s). out is OVERWRITTEN. */
int gifb200_spatial_dot(const float* a, const float* b2, float* out, int B, int P, int C, gifb200_stream_t stream);
/* y = alpha*a + beta*b (b may be NULL): residual merge (a+b)/sqrt2 of ResBlock.forward (cl.py:817-818),
 * skip accumulation of ToRGB (cl.py:509), noise add. */
int gifb200_axpby(const float* a, const float* b, float* y, long long n, float alpha, float beta, int round_tf32,
                  gifb200_stream_t stream);
/* d[b,o] = rsqrt(sum_i s[b,i]^2 * q[o,i] + eps): style-vector demodulation coefficients (cl.py:315; q[o,i] =
 * sum_taps W~[o,i,.,.]^2), one warp per (b,o) with a shuffle reduction. */
int gifb200_demod(const float* s, const float* q, float* d, int B, int Ci, int Co, float eps, gifb200_stream_t stream);

/* ---- ToRGB: per-sample 1x1 convolution to 3 channels (no demodulation) ----------------------------------
 * Replaces ToRGB.forward's ModulatedConv2d(k=1, demodulate=False) (cl.py:498-504). ws[b,3,C] = W~rgb[c3,i]*s[b,i]
 * is computed by the caller (tiny).  y[b,p,3] = sum_i x[b,p,i] * ws[b,:,i]. */
int gifb200_torgb_fwd(const float* x, const float* ws, float* y, int B, int P, int C, gifb200_stream_t stream);
int gifb200_torgb_bwd_x(const float* gy, const float* ws, float* gx, int B, int P, int C, gifb200_stream_t stream);
int gifb200_torgb_bwd_w(const float* gy, const float* x, float* gws, int B, int P, int C, gifb200_stream_t stream);

/* ---- small dense GEMM (EqualLinear) -------------------------------------------------------------------
 * Replaces F.linear in EqualLinear.forward (cl.py:212-230) and its gradients. Row-major:
 *     C[M,N] = alpha * op(A) * op(B),  op(A) is M x K (A stored K x M if transA), op(B) is K x N (N x K if transB). */
int gifb200_sgemm(int transA, int transB, int M, int N, int K, float alpha, const float* A, int lda, const float* B,
                  int ldb, float* C, int ldc, gifb200_stream_t stream);

/* ---- condition pyramid ----------------------------------------------------------------------------------
 * Replaces F.interpolate(cond, (r,r), 'bilinear', align_corners=False) for power-of-two reductions
 * (stg2_generator.py:309-314; SURVEY A2: mean of the central 2x2 of each s x s block). x (B,H,W,C) -> y (B,H/s,W/s,C).
 * adjoint != 0 computes the transpose map (y given, x produced, zeros elsewhere). */
int gifb200_cond_down(float* x, float* y, int B, int H, int W, int C, int s, int adjoint,
                      gifb200_stream_t stream);

/* ---- rasteriser ---------------------------------------------------------------------------------------
 * Replaces standard_rasterize / standard_rasterize_colors
 * (my_utils/standard_rasterize_cuda/standard_rasterize_cuda.cpp:26-40,59-75; kernels
 * standard_rasterize_cuda_kernel.cu:112-233).  Same contract: face_vertices (B,F,3,3) fp32 in pixel space,
 * caller-initialised depth (B,h,w) / triangle (B,h,w) int32 / bary-or-image (B,h,w,3) buffers updated IN PLACE.
 * Deterministic: exact depth ties are won by the lowest face index; fp32 arithmetic is evaluated without FMA
 * contraction (bit-exact against oracle/rasterize_oracle.c).  face_colors == NULL selects standard_rasterize
 * (out3 = barycentric weights), otherwise standard_rasterize_colors (out3 = interpolated colours). */
size_t gifb200_rasterize_workspace_bytes(int B, int F, int h, int w);
int gifb200_rasterize_fwd(const float* face_vertices, const float* face_colors, float* depth, int32_t* triangle,
                          float* out3, int B, int F, int h, int w, void* workspace, size_t workspace_bytes,
                          gifb200_stream_t stream);
/* Extended form.  convention 0 = the in-repo standard_rasterize semantics above.  convention 1 = pytorch3d's
 * rasterize_meshes as Pytorch3dRasterizer.forward calls it (my_utils/photometric_optimization/renderer.py:35-67:
 * image_size, blur_radius 0, faces_per_pixel 1, perspective_correct False) -- the rasteriser the reference's conditioning
 * maps are made with: face_vertices in NDC with x, y already negated by the caller (renderer.py:55), +X left / +Y up,
 * pixel (yi,xi) samples NDC (-1 + (2(W-1-xi)+1)/W, -1 + (2(H-1-yi)+1)/H), edge-function barycentrics over (area + 1e-8),
 * no back-face culling, strictly-inside test, linear depth sum w_i z_i >= 0; depth/triangle/out3 = zbuf / face index within
 * the mesh / barycentrics, still updated in place (initialise depth to +inf; the binding maps empty pixels to the -1 that
 * pytorch3d returns).  The fork the reference pins is absent (requirements.txt:36): parity unpinned, checked against the
 * restatement in oracle/rasterize_oracle.c.
 * face_colors2 / out3b (both may be NULL): a second per-corner attribute set interpolated in the same pass, e.g. vertex
 * colours and vertex normals of BASELINE.json configs[3] ("texture+normal render") from ONE rasterisation. */
int gifb200_rasterize_fwd_ex(const float* face_vertices, const float* face_colors, const float* face_colors2, float* depth,
                             int32_t* triangle, float* out3, float* out3b, int B, int F, int h, int w, int convention,
                             void* workspace, size_t workspace_bytes, gifb200_stream_t stream);
/* Backward (absent in the reference for standard_rasterize, SURVEY R5; provided by pytorch3d for convention 1): given the
 * forward's triangle buffer and upstream gradients of the barycentric weights g_bary (B,h,w,3) and/or interpolated
 * colours g_img (B,h,w,3) and/or depth g_depth (B,h,w) (each may be NULL), writes g_face_vertices (B,F,3,3) and
 * g_face_colors (B,F,3,3) (may be NULL).  Outputs are OVERWRITTEN (one thread per face gathers the pixels it owns: no
 * atomics, no zero-initialisation needed, deterministic). */
int gifb200_rasterize_bwd(const float* face_vertices, const float* face_colors, const int32_t* triangle,
                          const float* g_bary, const float* g_img, const float* g_depth, float* g_face_vertices,
                          float* g_face_colors, int B, int F, int h, int w, gifb200_stream_t stream);
int gifb200_rasterize_bwd_ex(const float* face_vertices, const float* face_colors, const float* face_colors2,
                             const int32_t* triangle, const float* g_bary, const float* g_img, const float* g_img2,
                             const float* g_depth, float* g_face_vertices, float* g_face_colors, float* g_face_colors2,
                             int B, int F, int h, int w, int convention, gifb200_stream_t stream);

/* Fused shading epilogue of the FLAME conditioning render: from the rasteriser's (triangle, bary) buffers to the textured
 * image tex (B,h,w,3) = albedo(uv) * SH-shading(normal) * alpha, the normal image nrm (B,h,w,3), and the quantised
 * 6-channel condition map cond (B,h,w,6) in [-1,1] (each output may be NULL).
 * Replaces the attribute interpolation of Pytorch3dRasterizer.forward (photometric_optimization/renderer.py:69-84),
 * Renderer.forward's grid_sample / add_SHlight / composition (renderer.py:152-221), Renderer.render_normal (:291-305),
 * OverLayViz.get_rendered_mesh's quantisation (my_utils/visualize_flame_overlay.py:29-31) and the consumer's mapping
 * to [-1,1] (loss_functions/losses.py:213-214).  face_uv (F,3,2) grid coordinates in [-1,1] (shared by the batch),
 * face_normals (B,F,3,3) world-space vertex normals per face corner, albedo (B,3,T,T), sh (B,9,3). */
int gifb200_render_shade(const int32_t* triangle, const float* bary, const float* face_uv, const float* face_normals,
                         const float* albedo, const float* sh, float* tex, float* nrm, float* cond, int B, int F, int h,
                         int w, int T, gifb200_stream_t stream);

/* FLAME decoder: linear blend skinning, lbs() of my_utils/photometric_optimization/models/lbs.py:141-228 as called by
 * FLAME.forward (models/FLAME.py:175-216).  betas (B,NB) = [shape | expression], pose (B,NJ*3) axis-angle per joint
 * (FLAME: NJ = 5 = global, neck, jaw, 2 eyes).  Model tensors prepared once by the host binding: v_template (V,3);
 * shapedirs_t (NB, V*3) = the reference's shapedirs (V,3,NB) with the coefficient axis first; posedirs ((NJ-1)*9, V*3) as
 * in the reference; j_template (NJ,3) = J_regressor @ v_template and j_shapedirs (NB, NJ*3) = J_regressor contracted
 * with shapedirs (the reference regresses the joints from the shaped mesh on every call, lbs.py:180 -- same value, one
 * reduction over the mesh less); parents (NJ) int32 kinematic tree (entry 0 ignored); lbs_weights (V,NJ).
 * Outputs: verts (B,V,3); joints (B,NJ,3) posed joint locations (may be NULL).  NJ <= 8, NB <= 1024. */
size_t gifb200_flame_lbs_workspace_bytes(int B, int NJ);
int gifb200_flame_lbs(const float* betas, const float* pose, const float* v_template, const float* shapedirs_t,
                      const float* posedirs, const float* j_template, const float* j_shapedirs, const int32_t* parents,
                      const float* lbs_weights, float* verts, float* joints, int B, int V, int NB, int NJ, void* ws,
                      size_t ws_bytes, gifb200_stream_t stream);

/* Texture stealing, FlameTextureSpace.compute_texture_map (model/stg2_generator.py:376-421): for every texel of the T x T
 * FLAME UV atlas, bilinear sample (zeros padding, align_corners = False) of the image src (B,H,W,C) channels-last at the
 * weak-perspective projection (cam (B,3) = scale, tx, ty; y flipped) of the texel's 3-D point on the posed mesh verts
 * (B,V,3).  Table (shared by the batch): texel_to_valid (T*T) int32, index n into vid / bary or -1; vid (N,3) int32 mesh
 * vertex ids; bary (N,3).  Texels with n < 0 sample grid (0,0), the image centre, like the reference's zero-initialised
 * grid.  Outputs tex (B,T,T,C) and, if mask != NULL, mask (B,T,T) uint8 = interpolated normal z < 0 on valid texels
 * (normals (B,V,3) of the projected mesh) else 0.  _bwd: the adjoint w.r.t. src (g_src (B,H,W,C) is overwritten). */
int gifb200_texture_steal_fwd(const float* src, const float* verts, const float* normals, const float* cam,
                              const int32_t* texel_to_valid, const int32_t* vid, const float* bary, float* tex,
                              unsigned char* mask, int B, int H, int W, int C, int V, int T, gifb200_stream_t stream);
int gifb200_texture_steal_bwd(const float* g_tex, const float* verts, const float* cam, const int32_t* texel_to_valid,
                              const int32_t* vid, const float* bary, float* g_src, int B, int H, int W, int C, int V, int T,
                              gifb200_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* GIFB200_H */
