// FLAME decoder: linear blend skinning (reference: my_utils/photometric_optimization/models/lbs.py:141-228, called from
// FLAME.forward, FLAME.py:175-216) as two kernels, so that random FLAME parameters become the vertices the rasteriser
// consumes without leaving the GPU (SURVEY 8f.1).
//
//   flame_pose_kernel  (one warp per sample; a few hundred FLOPs): joints from the shape coefficients through the
//       PRE-CONTRACTED regressor  J = Jr T + (Jr S) beta  (the reference regresses them from all V shaped vertices,
//       lbs.py:180; contracting Jr with the basis once at model-load time removes a reduction over the mesh from every
//       call), Rodrigues rotations (lbs.py:247-279, incl. its +1e-8 on every component), the pose feature
//       (R_j - I, lbs.py:189), the kinematic chain and the rest-pose-relative transforms A_j (lbs.py:296-349).
//   flame_skin_kernel  (HBM/L2-bound over the bases: (NB + P) x 3V floats, read once per group of 8 samples): one thread
//       per vertex, 8 samples in registers; v = T + S beta + P feat; skinning transform sum_j w_vj A_j applied to [v;1].
// Algorithmic bytes per call: bases (NB+P)*3V*4 (2.2 MB for FLAME: 150+36, V=5023) + weights + B*V*12 out.
#include "common.cuh"

namespace gifb200 {

constexpr int kFlameMaxJoints = 8;
constexpr int kFlameSB = 8;            // samples per CTA of the skinning kernel

__global__ void __launch_bounds__(32) flame_pose_kernel(const float* __restrict__ betas, const float* __restrict__ pose,
                                                        const float* __restrict__ j_template,
                                                        const float* __restrict__ j_shapedirs,
                                                        const int* __restrict__ parents, float* __restrict__ feat,
                                                        float* __restrict__ amat, float* __restrict__ joints_out, int NB,
                                                        int NJ) {
    __shared__ float J[kFlameMaxJoints][3];
    __shared__ float R[kFlameMaxJoints][9];
    __shared__ float C[kFlameMaxJoints][12];     // chain transforms, rows of [Rc | tc]
    const int b = blockIdx.x, lane = threadIdx.x;
    if (lane < NJ * 3) {
        float a = j_template[lane];
        const float* bt = betas + static_cast<long long>(b) * NB;
        for (int l = 0; l < NB; ++l) a = fmaf(bt[l], j_shapedirs[l * NJ * 3 + lane], a);
        J[lane / 3][lane % 3] = a;
    }
    if (lane < NJ) {
        const float* r = pose + (static_cast<long long>(b) * NJ + lane) * 3;
        const float rx = r[0], ry = r[1], rz = r[2];
        const float ex = rx + 1e-8f, ey = ry + 1e-8f, ez = rz + 1e-8f;
        const float angle = sqrtf(ex * ex + ey * ey + ez * ez);
        const float dx = rx / angle, dy = ry / angle, dz = rz / angle;
        const float s = sinf(angle), c1 = 1.f - cosf(angle);
        // K = [[0,-dz,dy],[dz,0,-dx],[-dy,dx,0]];  R = I + s K + (1-c) K K
        const float kk[9] = {-(dy * dy + dz * dz), dx * dy, dx * dz, dx * dy, -(dx * dx + dz * dz), dy * dz,
                             dx * dz, dy * dz, -(dx * dx + dy * dy)};
        const float k1[9] = {0.f, -dz, dy, dz, 0.f, -dx, -dy, dx, 0.f};
#pragma unroll
        for (int i = 0; i < 9; ++i) R[lane][i] = ((i % 4 == 0) ? 1.f : 0.f) + s * k1[i] + c1 * kk[i];
    }
    __syncwarp();
    const int P = (NJ - 1) * 9;
    for (int i = lane; i < P; i += 32) {
        const int j = i / 9 + 1, e = i % 9;
        feat[static_cast<long long>(b) * P + i] = R[j][e] - ((e % 4 == 0) ? 1.f : 0.f);
    }
    if (lane == 0) {
        for (int i = 0; i < NJ; ++i) {
            const int par = i == 0 ? -1 : parents[i];
            float rel[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) rel[k] = par < 0 ? J[i][k] : J[i][k] - J[par][k];
            if (par < 0) {
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    C[i][r * 4 + 0] = R[i][r * 3 + 0]; C[i][r * 4 + 1] = R[i][r * 3 + 1]; C[i][r * 4 + 2] = R[i][r * 3 + 2];
                    C[i][r * 4 + 3] = rel[r];
                }
            } else {
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const float p0 = C[par][r * 4 + 0], p1 = C[par][r * 4 + 1], p2 = C[par][r * 4 + 2], p3 = C[par][r * 4 + 3];
#pragma unroll
                    for (int cc = 0; cc < 3; ++cc) C[i][r * 4 + cc] = p0 * R[i][cc] + p1 * R[i][3 + cc] + p2 * R[i][6 + cc];
                    C[i][r * 4 + 3] = p0 * rel[0] + p1 * rel[1] + p2 * rel[2] + p3;
                }
            }
        }
        for (int i = 0; i < NJ; ++i) {
            float* a = amat + (static_cast<long long>(b) * NJ + i) * 12;
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const float c0 = C[i][r * 4 + 0], c1 = C[i][r * 4 + 1], c2 = C[i][r * 4 + 2];
                a[r * 4 + 0] = c0; a[r * 4 + 1] = c1; a[r * 4 + 2] = c2;
                a[r * 4 + 3] = C[i][r * 4 + 3] - (c0 * J[i][0] + c1 * J[i][1] + c2 * J[i][2]);
                if (joints_out) joints_out[(static_cast<long long>(b) * NJ + i) * 3 + r] = C[i][r * 4 + 3];
            }
        }
    }
}

__global__ void __launch_bounds__(128) flame_skin_kernel(const float* __restrict__ betas, const float* __restrict__ feat,
                                                         const float* __restrict__ amat,
                                                         const float* __restrict__ v_template,
                                                         const float* __restrict__ shapedirs_t,
                                                         const float* __restrict__ posedirs,
                                                         const float* __restrict__ lbs_weights, float* __restrict__ verts,
                                                         int B, int V, int NB, int NJ) {
    extern __shared__ float sm[];
    const int P = (NJ - 1) * 9;
    float* sb = sm;                              // [NB + P][SB] coefficients (betas then pose feature), sample-minor
    float* sa = sm + (NB + P) * kFlameSB;        // [SB][NJ][12]
    const int b0 = blockIdx.y * kFlameSB;
    for (int i = threadIdx.x; i < (NB + P) * kFlameSB; i += blockDim.x) {
        const int l = i / kFlameSB, s = i % kFlameSB, b = b0 + s;
        float v = 0.f;
        if (b < B) v = l < NB ? betas[static_cast<long long>(b) * NB + l] : feat[static_cast<long long>(b) * P + (l - NB)];
        sb[i] = v;
    }
    for (int i = threadIdx.x; i < kFlameSB * NJ * 12; i += blockDim.x) {
        const int s = i / (NJ * 12), b = b0 + s;
        sa[i] = b < B ? amat[static_cast<long long>(b) * NJ * 12 + (i - s * NJ * 12)] : 0.f;
    }
    __syncthreads();
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    float acc[kFlameSB][3];
    {
        const float t0 = v_template[v * 3 + 0], t1 = v_template[v * 3 + 1], t2 = v_template[v * 3 + 2];
#pragma unroll
        for (int s = 0; s < kFlameSB; ++s) { acc[s][0] = t0; acc[s][1] = t1; acc[s][2] = t2; }
    }
    const long long row = static_cast<long long>(V) * 3;
#pragma unroll 2
    for (int l = 0; l < NB + P; ++l) {
        const float* basis = (l < NB ? shapedirs_t + l * row : posedirs + (l - NB) * row) + v * 3;
        const float d0 = __ldg(basis), d1 = __ldg(basis + 1), d2 = __ldg(basis + 2);
        const float4 c0 = *reinterpret_cast<const float4*>(sb + l * kFlameSB);
        const float4 c1 = *reinterpret_cast<const float4*>(sb + l * kFlameSB + 4);
        const float cs[kFlameSB] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
#pragma unroll
        for (int s = 0; s < kFlameSB; ++s) {
            acc[s][0] = fmaf(cs[s], d0, acc[s][0]);
            acc[s][1] = fmaf(cs[s], d1, acc[s][1]);
            acc[s][2] = fmaf(cs[s], d2, acc[s][2]);
        }
    }
    float w[kFlameMaxJoints];
#pragma unroll
    for (int j = 0; j < kFlameMaxJoints; ++j) w[j] = j < NJ ? lbs_weights[static_cast<long long>(v) * NJ + j] : 0.f;
#pragma unroll
    for (int s = 0; s < kFlameSB; ++s) {
        if (b0 + s >= B) break;
        float T[12];
#pragma unroll
        for (int e = 0; e < 12; ++e) T[e] = 0.f;
#pragma unroll
        for (int j = 0; j < kFlameMaxJoints; ++j) {
            if (j < NJ) {
                const float* a = sa + (s * NJ + j) * 12;
#pragma unroll
                for (int e = 0; e < 12; ++e) T[e] = fmaf(w[j], a[e], T[e]);
            }
        }
        float* o = verts + (static_cast<long long>(b0 + s) * V + v) * 3;
#pragma unroll
        for (int r = 0; r < 3; ++r)
            o[r] = T[r * 4 + 0] * acc[s][0] + T[r * 4 + 1] * acc[s][1] + T[r * 4 + 2] * acc[s][2] + T[r * 4 + 3];
    }
}

}  // namespace gifb200

using namespace gifb200;

extern "C" size_t gifb200_flame_lbs_workspace_bytes(int B, int NJ) {
    if (B <= 0 || NJ <= 0) return 0;
    return sizeof(float) * static_cast<size_t>(B) * ((NJ - 1) * 9 + NJ * 12);
}

extern "C" int gifb200_flame_lbs(const float* betas, const float* pose, const float* v_template, const float* shapedirs_t,
                                 const float* posedirs, const float* j_template, const float* j_shapedirs,
                                 const int* parents, const float* lbs_weights, float* verts, float* joints, int B, int V,
                                 int NB, int NJ, void* ws, size_t ws_bytes, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && V > 0 && NB > 0 && NB <= 1024, GIFB200_E_SHAPE, "flame_lbs: bad shape (NB <= 1024)");
    GIFB200_REQUIRE(NJ >= 1 && NJ <= kFlameMaxJoints, GIFB200_E_SHAPE, "flame_lbs: 1..8 joints");
    GIFB200_REQUIRE(static_cast<long long>(V) * 3 * (NB + (NJ - 1) * 9) < 2147483647LL, GIFB200_E_SHAPE, "flame_lbs: basis too large");
    if (B == 0) return GIFB200_OK;
    GIFB200_REQUIRE(ws && ws_bytes >= gifb200_flame_lbs_workspace_bytes(B, NJ), GIFB200_E_WORKSPACE,
                    "flame_lbs: workspace too small (see gifb200_flame_lbs_workspace_bytes)");
    GIFB200_REQUIRE(B <= 65535 * kFlameSB, GIFB200_E_SHAPE, "flame_lbs: batch too large");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int P = (NJ - 1) * 9;
    float* feat = static_cast<float*>(ws);
    float* amat = feat + static_cast<size_t>(B) * P;
    flame_pose_kernel<<<B, 32, 0, st>>>(betas, pose, j_template, j_shapedirs, parents, feat, amat, joints, NB, NJ);
    GIFB200_LAUNCH_CHECK("flame_pose_kernel");
    const int smem = static_cast<int>(sizeof(float)) * ((NB + P) * kFlameSB + kFlameSB * NJ * 12);
    static bool attr = false;
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(flame_skin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
        if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "flame_lbs smem attribute", cudaGetErrorString(e));
        attr = true;
    }
    flame_skin_kernel<<<dim3(cdiv(V, 128), cdiv(B, kFlameSB)), 128, smem, st>>>(betas, feat, amat, v_template, shapedirs_t,
                                                                                 posedirs, lbs_weights, verts, B, V, NB, NJ);
    GIFB200_LAUNCH_CHECK("flame_skin_kernel");
    return GIFB200_OK;
}

// ---------------------------------------------------------------------------------------------- eye-centred camera
// position_to_given_location (my_utils/eye_centering.py:35-66): the weak-perspective camera (s, bx, by) that puts the two
// eye vertices at fixed image positions.  The reference solves  d = (s, s bx, s by) M  with  M = [[e1x e2x e1y e2y],
// [1 1 0 0], [0 0 1 1]]  by a float32 pseudo-inverse per row; for a full-rank M that least-squares solution is
//     s = (dex dx + dey dy) / (dex^2 + dey^2),  s bx = (x1 + x2)/2 - s (e1x + e2x)/2,  s by likewise,
// with dex = e1x - e2x, dx = x1 - x2 (y likewise), evaluated here in float64 and rounded once.  cam = (-s, bx, by).
// A row whose eyes coincide in x and y has no unique camera: 0/0 makes it NaN (the reference divides by zero there too).
__global__ void __launch_bounds__(128) eye_camera_kernel(const float* __restrict__ verts, float* __restrict__ cam, int B, int V,
                                                         int i1, int i2, double x1, double x2, double y1, double y2) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float* v = verts + static_cast<long long>(b) * V * 3;
    const double e1x = v[i1 * 3 + 0], e1y = v[i1 * 3 + 1], e2x = v[i2 * 3 + 0], e2y = v[i2 * 3 + 1];
    const double dex = e1x - e2x, dey = e1y - e2y;
    const double s = (dex * (x1 - x2) + dey * (y1 - y2)) / (dex * dex + dey * dey);
    const double sbx = 0.5 * (x1 + x2) - s * (0.5 * (e1x + e2x));
    const double sby = 0.5 * (y1 + y2) - s * (0.5 * (e1y + e2y));
    cam[b * 3 + 0] = static_cast<float>(-s);
    cam[b * 3 + 1] = static_cast<float>(sbx / s);
    cam[b * 3 + 2] = static_cast<float>(sby / s);
}

extern "C" int gifb200_eye_camera(const float* verts, float* cam, int B, int V, int i1, int i2, float x1, float x2, float y1,
                                  float y2, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && V > 0, GIFB200_E_SHAPE, "eye_camera: bad shape");
    GIFB200_REQUIRE(i1 >= 0 && i1 < V && i2 >= 0 && i2 < V, GIFB200_E_SHAPE, "eye_camera: eye vertex index outside 0..V-1");
    if (B == 0) return GIFB200_OK;
    eye_camera_kernel<<<cdiv(B, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(verts, cam, B, V, i1, i2, x1, x2, y1, y2);
    GIFB200_LAUNCH_CHECK("eye_camera_kernel");
    return GIFB200_OK;
}

// ------------------------------------------------------------------------------------------------------------ FLAMETex
// FLAMETex.forward (models/FLAME.py:237-242): mean + basis . texcode, reshaped to side x side x 3, F.interpolate to T x T in
// the default nearest mode (source index min(floor(dst * side / T), side - 1)), RGB -> BGR -- evaluated only at the texels
// the nearest sampling keeps (a quarter of the basis at side 512, T 256).  One CTA per (64 output texels of one row): it
// stages the 192 basis rows of its texels in shared memory once and runs every texcode of the batch against them, 32 at a
// time (coefficient-major, read as float4 broadcasts), so the basis is read from HBM once per batch.
// Algorithmic bytes per call: T*T*3*(n+1)*4 of basis + mean (39 MB at n 50, T 256) + B*n*4 + B*3*T*T*4 out.
constexpr int kTexX = 64;
constexpr int kTexBC = 32;
constexpr int kTexMaxN = 200;

__global__ void __launch_bounds__(kTexX * 3) flametex_kernel(const float* __restrict__ texcode, const float* __restrict__ mean,
                                                             const float* __restrict__ basis, float* __restrict__ albedo,
                                                             int B, int n, int side, int T, float scale) {
    extern __shared__ __align__(16) float tex_smem[];
    float* sB = tex_smem;                          // (kTexX*3, n): basis rows of this CTA's texels, texel-major
    float* sT = tex_smem + kTexX * 3 * n;          // (n, kTexBC): texcodes, coefficient-major
    const int y = blockIdx.y, x0 = blockIdx.x * kTexX, tid = threadIdx.x;
    const int nx = min(kTexX, T - x0);
    const int sy = min(static_cast<int>(floorf(static_cast<float>(y) * scale)), side - 1);
    const int rowlen = 3 * n;
    for (int i = tid; i < nx * rowlen; i += blockDim.x) {
        const int xl = i / rowlen, e = i - xl * rowlen;
        const int sx = min(static_cast<int>(floorf(static_cast<float>(x0 + xl) * scale)), side - 1);
        sB[i] = __ldg(basis + (static_cast<long long>(sy) * side + sx) * rowlen + e);
    }
    const int c = tid / kTexX, xl = tid - c * kTexX;       // consecutive threads: consecutive x of one channel plane
    const bool active = xl < nx;
    const int sx = min(static_cast<int>(floorf(static_cast<float>(x0 + xl) * scale)), side - 1);
    const float m = active ? __ldg(mean + (static_cast<long long>(sy) * side + sx) * 3 + c) : 0.f;
    const float* brow = sB + (xl * 3 + c) * n;
    const long long plane = static_cast<long long>(T) * T;
    float* out = albedo + (2 - c) * plane + static_cast<long long>(y) * T + x0 + xl;
    for (int b0 = 0; b0 < B; b0 += kTexBC) {
        const int nb = min(kTexBC, B - b0);
        __syncthreads();                           // sB staged / the previous pass is done with sT
        for (int i = tid; i < n * kTexBC; i += blockDim.x) {
            const int j = i / kTexBC, bb = i - j * kTexBC;
            sT[i] = bb < nb ? __ldg(texcode + static_cast<long long>(b0 + bb) * n + j) : 0.f;
        }
        __syncthreads();
        if (!active) continue;
        for (int g = 0; g < nb; g += 8) {
            float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            for (int j = 0; j < n; ++j) {
                const float bv = brow[j];
                const float4 t0 = *reinterpret_cast<const float4*>(sT + j * kTexBC + g);
                const float4 t1 = *reinterpret_cast<const float4*>(sT + j * kTexBC + g + 4);
                acc[0] = fmaf(bv, t0.x, acc[0]);
                acc[1] = fmaf(bv, t0.y, acc[1]);
                acc[2] = fmaf(bv, t0.z, acc[2]);
                acc[3] = fmaf(bv, t0.w, acc[3]);
                acc[4] = fmaf(bv, t1.x, acc[4]);
                acc[5] = fmaf(bv, t1.y, acc[5]);
                acc[6] = fmaf(bv, t1.z, acc[6]);
                acc[7] = fmaf(bv, t1.w, acc[7]);
            }
#pragma unroll
            for (int q = 0; q < 8; ++q)
                if (g + q < nb) out[static_cast<long long>(b0 + g + q) * 3 * plane] = m + acc[q];
        }
    }
}

extern "C" int gifb200_flametex(const float* texcode, const float* mean, const float* basis, float* albedo, int B, int n,
                                int side, int T, gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && n >= 1 && n <= kTexMaxN && side > 0 && T > 0 && T <= 65535, GIFB200_E_SHAPE,
                    "flametex: bad shape (1 <= n <= 200 coefficients, T <= 65535)");
    if (B == 0) return GIFB200_OK;
    const int smem = static_cast<int>(sizeof(float)) * (kTexX * 3 + kTexBC) * n;
    static bool attr = false;
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(flametex_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             static_cast<int>(sizeof(float)) * (kTexX * 3 + kTexBC) * kTexMaxN);
        if (e != cudaSuccess) return fail(GIFB200_E_CUDA, "flametex smem attribute", cudaGetErrorString(e));
        attr = true;
    }
    flametex_kernel<<<dim3(cdiv(T, kTexX), T), kTexX * 3, smem, static_cast<cudaStream_t>(stream)>>>(
        texcode, mean, basis, albedo, B, n, side, T, static_cast<float>(side) / static_cast<float>(T));
    GIFB200_LAUNCH_CHECK("flametex_kernel");
    return GIFB200_OK;
}
