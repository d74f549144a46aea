// Multi-tensor Adam for the two optimisers of the loop body (train.py:365-382: torch.optim.Adam on the generator and the
// discriminator, betas (0, 0.99^ratio), no weight decay, no amsgrad), one launch per 64 parameter tensors instead of
// torch's capturable foreach implementation (~600 launches per optimiser step for the ~210 tensors of the generator: its
// per-parameter step counters and bias corrections are 0-d tensors, each handled by its own elementwise kernel).
//
// Arithmetic: torch/optim/adam.py::_single_tensor_adam in the order the reference's (non-capturable) optimiser runs it:
//   m = lerp(m, g, 1-b1);  v = b2*v + (1-b2)*g*g;  bc1 = 1-b1^t;  bc2 = 1-b2^t  (double, like the host floats there)
//   p = p + (-(lr/bc1)) * (m / (sqrt(v)/sqrt(bc2) + eps))
// HBM-bound: 16 bytes read + 12 written per parameter; 59 M parameters -> 1.7 GB per iteration.
#include "common.cuh"

namespace gifb200 {

constexpr int kAdamPack = 64;

struct AdamPack {
    float* p[kAdamPack];
    const float* g[kAdamPack];
    float* m[kAdamPack];
    float* v[kAdamPack];
    float* s[kAdamPack];      // per-tensor step counters (0-d device floats, torch's capturable layout)
    long long n[kAdamPack];
};

__global__ void adam_tick_kernel(const AdamPack pk, int k) {
    if (threadIdx.x < k) *pk.s[threadIdx.x] += 1.f;
}

__device__ __forceinline__ void adam_one(float& p, float g, float& m, float& v, float w1, float beta2, float omb2, float neg_step_size,
                                         float bc2_sqrt, float eps) {
    const float diff = __fsub_rn(g, m);
    m = (w1 < 0.5f) ? __fadd_rn(m, __fmul_rn(w1, diff)) : __fsub_rn(g, __fmul_rn(diff, __fsub_rn(1.f, w1)));   // at::lerp
    v = __fadd_rn(__fmul_rn(v, beta2), __fmul_rn(omb2, __fmul_rn(g, g)));                  // mul_(b2).addcmul_(g, g, 1-b2)
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);
    p = __fadd_rn(p, __fmul_rn(neg_step_size, __fdiv_rn(m, denom)));                        // addcdiv_(m, denom, -step_size)
}

__global__ void __launch_bounds__(256) adam_multi_kernel(const AdamPack pk, double lr, double beta1, double beta2_d, float eps) {
    const int t = blockIdx.y;
    const long long n = pk.n[t];
    float* __restrict__ p = pk.p[t];
    const float* __restrict__ g = pk.g[t];
    float* __restrict__ m = pk.m[t];
    float* __restrict__ v = pk.v[t];
    const double st = static_cast<double>(*pk.s[t]);
    // the hyper-parameters arrive as doubles (python floats in torch): 1 - beta2 taken from a float beta2 is off by 4e-6
    const double bc1 = 1.0 - pow(beta1, st);
    const double bc2 = 1.0 - pow(beta2_d, st);
    const float neg_step_size = static_cast<float>(-(lr / bc1));
    const float bc2_sqrt = static_cast<float>(sqrt(bc2));
    const float w1 = static_cast<float>(1.0 - beta1);
    const float omb2 = static_cast<float>(1.0 - beta2_d);
    const float beta2 = static_cast<float>(beta2_d);
    const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long nth = static_cast<long long>(gridDim.x) * blockDim.x;
    const bool vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                       reinterpret_cast<uintptr_t>(v)) & 15u) == 0;
    long long done = 0;
    if (vec) {
        const long long n4 = n / 4;
        for (long long i = tid; i < n4; i += nth) {
            float4 pv = reinterpret_cast<float4*>(p)[i];
            const float4 gv = __ldcs(reinterpret_cast<const float4*>(g) + i);
            float4 mv = reinterpret_cast<float4*>(m)[i];
            float4 vv = reinterpret_cast<float4*>(v)[i];
            adam_one(pv.x, gv.x, mv.x, vv.x, w1, beta2, omb2, neg_step_size, bc2_sqrt, eps);
            adam_one(pv.y, gv.y, mv.y, vv.y, w1, beta2, omb2, neg_step_size, bc2_sqrt, eps);
            adam_one(pv.z, gv.z, mv.z, vv.z, w1, beta2, omb2, neg_step_size, bc2_sqrt, eps);
            adam_one(pv.w, gv.w, mv.w, vv.w, w1, beta2, omb2, neg_step_size, bc2_sqrt, eps);
            reinterpret_cast<float4*>(p)[i] = pv;
            reinterpret_cast<float4*>(m)[i] = mv;
            reinterpret_cast<float4*>(v)[i] = vv;
        }
        done = n4 * 4;
    }
    for (long long i = done + tid; i < n; i += nth) {
        float pv = p[i], mv = m[i], vv = v[i];
        adam_one(pv, g[i], mv, vv, w1, beta2, omb2, neg_step_size, bc2_sqrt, eps);
        p[i] = pv; m[i] = mv; v[i] = vv;
    }
}

}  // namespace gifb200

using namespace gifb200;

extern "C" int gifb200_adam_step(float* const* params, const float* const* grads, float* const* exp_avg, float* const* exp_avg_sq,
                                 float* const* steps, const long long* numel, int count, double lr, double beta1, double beta2,
                                 double eps, gifb200_stream_t stream) {
    GIFB200_REQUIRE(count >= 0, GIFB200_E_SHAPE, "adam_step: bad arguments");
    GIFB200_REQUIRE(count == 0 || (params && grads && exp_avg && exp_avg_sq && steps && numel), GIFB200_E_SHAPE,
                    "adam_step: null table");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int base = 0; base < count; base += kAdamPack) {
        AdamPack pk;
        memset(&pk, 0, sizeof(pk));
        const int k = (count - base < kAdamPack) ? count - base : kAdamPack;
        long long nmax = 0;
        for (int i = 0; i < k; ++i) {
            GIFB200_REQUIRE(params[base + i] && grads[base + i] && exp_avg[base + i] && exp_avg_sq[base + i] && steps[base + i] &&
                                numel[base + i] >= 0, GIFB200_E_SHAPE, "adam_step: null tensor");
            pk.p[i] = params[base + i]; pk.g[i] = grads[base + i]; pk.m[i] = exp_avg[base + i]; pk.v[i] = exp_avg_sq[base + i];
            pk.s[i] = steps[base + i];
            pk.n[i] = numel[base + i];
            if (pk.n[i] > nmax) nmax = pk.n[i];
        }
        adam_tick_kernel<<<1, kAdamPack, 0, st>>>(pk, k);
        GIFB200_LAUNCH_CHECK("adam_tick_kernel");
        if (nmax == 0) continue;
        long long bx = (nmax + 256LL * 4 * 8 - 1) / (256LL * 4 * 8);      // ~8 float4 per thread on the largest tensor
        if (bx < 1) bx = 1;
        if (bx > 128) bx = 128;
        adam_multi_kernel<<<dim3(static_cast<unsigned>(bx), k), 256, 0, st>>>(pk, lr, beta1, beta2, static_cast<float>(eps));
        GIFB200_LAUNCH_CHECK("adam_multi_kernel");
    }
    return GIFB200_OK;
}
