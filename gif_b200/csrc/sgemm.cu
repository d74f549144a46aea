// Small dense fp32 GEMM for EqualLinear (mapping network 512x512, modulation 512xCi, D head 8192x512):
// C[M,N] = alpha * op(A) op(B).  32x32 tiles, 256 threads, 2x2 micro-tiles.  These GEMMs are tiny
// (<= 0.3 GFLOP per step in total) so a SIMT kernel is the right tool; the tensor cores are reserved for the convolutions.
#include "common.cuh"

namespace gifb200 {

__global__ void __launch_bounds__(256) sgemm_kernel(int transA, int transB, int M, int N, int K, float alpha,
                                                    const float* __restrict__ A, int lda, const float* __restrict__ B,
                                                    int ldb, float* __restrict__ C, int ldc, int k_per_split) {
    __shared__ float As[32][33];  // [k][m]
    __shared__ float Bs[32][33];  // [k][n]
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int m0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
    float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
    const int k_begin = blockIdx.z * k_per_split;
    const int k_end = min(K, k_begin + k_per_split);
    for (int k0 = k_begin; k0 < k_end; k0 += 32) {
        for (int e = threadIdx.x; e < 1024; e += 256) {
            // read along the contiguous dimension of each operand
            int kk, mm;
            if (transA) { mm = e & 31; kk = e >> 5; } else { kk = e & 31; mm = e >> 5; }
            const int gm = m0 + mm, gk = k0 + kk;
            float v = 0.f;
            if (gm < M && gk < k_end) v = transA ? A[static_cast<long long>(gk) * lda + gm] : A[static_cast<long long>(gm) * lda + gk];
            As[kk][mm] = v;
            int kb, nn;
            if (transB) { kb = e & 31; nn = e >> 5; } else { nn = e & 31; kb = e >> 5; }
            const int gn = n0 + nn, gkb = k0 + kb;
            float w = 0.f;
            if (gn < N && gkb < k_end) w = transB ? B[static_cast<long long>(gn) * ldb + gkb] : B[static_cast<long long>(gkb) * ldb + gn];
            Bs[kb][nn] = w;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 32; ++k) {
            const float a0 = As[k][ty * 2], a1 = As[k][ty * 2 + 1];
            const float b0 = Bs[k][tx * 2], b1 = Bs[k][tx * 2 + 1];
            acc[0][0] += a0 * b0; acc[0][1] += a0 * b1; acc[1][0] += a1 * b0; acc[1][1] += a1 * b1;
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int gm = m0 + ty * 2 + i, gn = n0 + tx * 2 + j;
            if (gm < M && gn < N) {
                if (gridDim.z == 1) C[static_cast<long long>(gm) * ldc + gn] = alpha * acc[i][j];
                else C[(static_cast<long long>(blockIdx.z) * M + gm) * N + gn] = alpha * acc[i][j];   // split-K: C = slots
            }
        }
}

}  // namespace gifb200

using namespace gifb200;

extern "C" int gifb200_sgemm(int transA, int transB, int M, int N, int K, float alpha, const float* A, int lda,
                             const float* B, int ldb, float* C, int ldc, gifb200_stream_t stream) {
    GIFB200_REQUIRE(M >= 0 && N >= 0 && K >= 0, GIFB200_E_SHAPE, "sgemm: bad shape");
    if (M == 0 || N == 0) return GIFB200_OK;
    GIFB200_REQUIRE(cdiv(M, 32) <= 65535, GIFB200_E_SHAPE, "sgemm: M too large");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // few output tiles and a long K (the 8192 -> 512 discriminator head, its gradients): split K across CTAs
    const long long tiles = static_cast<long long>(cdiv(N, 32)) * cdiv(M, 32);
    int splits = 1;
    // ... and the batch-32 style / mapping-network GEMMs (M = 32, N = K = 512: 16 output tiles of 16 serial k-tiles each are
    // latency-bound, 250 launches per step): at least two k-tiles per split
    if (tiles < kNumSMs && K >= 128 && ldc == N) {
        splits = static_cast<int>((2LL * kNumSMs + tiles - 1) / tiles);
        const int max_splits = K >= 1024 ? K / 256 : K / 64;
        if (splits > max_splits) splits = max_splits;
        if (splits < 1) splits = 1;
    }
    int kps = ((K + splits - 1) / splits + 31) / 32 * 32;
    splits = (K + kps - 1) / kps;
    Slots sl;      // split-K: one partial product per split, added in split order
    if (splits > 1) {
        GIFB200_REQUIRE(ldc == N, GIFB200_E_SHAPE, "sgemm: split-K needs a dense C");
        if (int rc = slots_take(sl, C, splits, static_cast<long long>(M) * N, st)) return rc;
    }
    sgemm_kernel<<<dim3(cdiv(N, 32), cdiv(M, 32), splits), 256, 0, st>>>(transA, transB, M, N, K, alpha, A, lda, B, ldb, C,
                                                                         ldc, kps);
    GIFB200_LAUNCH_CHECK("sgemm_kernel");
    return sl.part ? slots_reduce(sl, st) : GIFB200_OK;
}
