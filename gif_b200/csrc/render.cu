// Fused shading epilogue of the FLAME conditioning render (SURVEY 7.7): per pixel, from the rasteriser's (triangle, bary)
// buffers, interpolate the UV coordinates and the world-space vertex normals of the owning face, fetch the albedo with
// grid_sample semantics (bilinear, align_corners=False, zero padding), evaluate the 9-term spherical-harmonics shading,
// and write the textured image, the normal image and (optionally) the quantised 6-channel condition map that the
// generator consumes -- one pass, nothing but the final maps goes to HBM.
// Replaces the attribute gather + interpolation of Pytorch3dRasterizer.forward (renderer.py:69-84), Renderer.forward's
// albedo lookup / add_SHlight / image composition (renderer.py:152-221), Renderer.render_normal (renderer.py:291-305)
// and the quantisation of OverLayViz.get_rendered_mesh (visualize_flame_overlay.py:29-31) + the consumer's mapping to
// [-1,1] (loss_functions/losses.py:213-214).
#include "common.cuh"

namespace gifb200 {

struct ShadeParams {
    int B, F, h, w, T;
};

__device__ __forceinline__ float tex_fetch(const float* __restrict__ plane, int T, int x, int y) {
    return (x >= 0 && x < T && y >= 0 && y < T) ? __ldg(plane + y * T + x) : 0.f;
}

__global__ void __launch_bounds__(256) render_shade_kernel(const int* __restrict__ tri, const float* __restrict__ bary,
                                                           const float* __restrict__ face_uv,       // (F,3,2) shared
                                                           const float* __restrict__ face_normals,  // (B,F,3,3)
                                                           const float* __restrict__ albedo,        // (B,3,T,T)
                                                           const float* __restrict__ sh,            // (B,9,3)
                                                           float* __restrict__ tex, float* __restrict__ nrm,
                                                           float* __restrict__ cond, uint8_t* __restrict__ cond_u8,
                                                           ShadeParams p) {
    const long long pix = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long npix = static_cast<long long>(p.B) * p.h * p.w;
    if (pix >= npix) return;
    const int b = static_cast<int>(pix / (static_cast<long long>(p.h) * p.w));
    const int f = tri[pix];
    float t3[3] = {0.f, 0.f, 0.f}, n3[3] = {0.f, 0.f, 0.f};
    if (f >= 0) {
        const float w0 = bary[pix * 3], w1 = bary[pix * 3 + 1], w2 = bary[pix * 3 + 2];
        const float* uv = face_uv + static_cast<long long>(f) * 6;
        const float gu = w0 * uv[0] + w1 * uv[2] + w2 * uv[4];
        const float gv = w0 * uv[1] + w1 * uv[3] + w2 * uv[5];
        const float* fn = face_normals + (static_cast<long long>(b) * p.F + f) * 9;
#pragma unroll
        for (int k = 0; k < 3; ++k) n3[k] = w0 * fn[k] + w1 * fn[3 + k] + w2 * fn[6 + k];
        // F.grid_sample(albedo, grid, mode='bilinear', padding_mode='zeros', align_corners=False)
        const float ix = ((gu + 1.f) * p.T - 1.f) * 0.5f, iy = ((gv + 1.f) * p.T - 1.f) * 0.5f;
        const float fx = floorf(ix), fy = floorf(iy);
        const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
        const float ax = ix - fx, ay = iy - fy;
        // SH basis (renderer.py:207-221) with the constant factors of renderer.py:119-126
        const float pi = 3.14159265358979323846f;
        const float c0 = 1.f / sqrtf(4.f * pi), c1 = (2.f * pi / 3.f) * sqrtf(3.f / (4.f * pi));
        const float c2 = (pi / 4.f) * 3.f * sqrtf(5.f / (12.f * pi)), c3 = (pi / 4.f) * 1.5f * sqrtf(5.f / (12.f * pi));
        const float c4 = (pi / 4.f) * 0.5f * sqrtf(5.f / (4.f * pi));
        const float nx = n3[0], ny = n3[1], nz = n3[2];
        const float basis[9] = {c0, c1 * nx, c1 * ny, c1 * nz, c2 * nx * ny, c2 * nx * nz, c2 * ny * nz,
                                c3 * (nx * nx - ny * ny), c4 * (3.f * nz * nz - 1.f)};
        const float* shb = sh + static_cast<long long>(b) * 27;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float* plane = albedo + (static_cast<long long>(b) * 3 + c) * p.T * p.T;
            const float a = (1.f - ay) * ((1.f - ax) * tex_fetch(plane, p.T, x0, y0) + ax * tex_fetch(plane, p.T, x0 + 1, y0)) +
                            ay * ((1.f - ax) * tex_fetch(plane, p.T, x0, y0 + 1) + ax * tex_fetch(plane, p.T, x0 + 1, y0 + 1));
            float shade = 0.f;
#pragma unroll
            for (int k = 0; k < 9; ++k) shade += shb[k * 3 + c] * basis[k];
            t3[c] = a * shade;            // * alpha (= 1 on covered pixels)
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        if (tex) tex[pix * 3 + c] = t3[c];
        if (nrm) nrm[pix * 3 + c] = n3[c];
    }
    if (cond) {
        // texture: floor(clamp(x,0,255))/255 ; normals: floor(clamp(n,0,1)*255)/255 ; then clamp(0,1)*2-1
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float tq = floorf(fminf(fmaxf(t3[c], 0.f), 255.f)) / 255.f;
            const float nq = floorf(fminf(fmaxf(n3[c], 0.f), 1.f) * 255.f) / 255.f;
            cond[pix * 6 + c] = fminf(fmaxf(tq, 0.f), 1.f) * 2.f - 1.f;
            cond[pix * 6 + 3 + c] = fminf(fmaxf(nq, 0.f), 1.f) * 2.f - 1.f;
        }
    }
    if (cond_u8) {
        // the bytes create_deca_rendered_lmdb.py stores: (floor(clamp(t,0,255))/255*255).astype(uint8) == floor(clamp(t,0,255)),
        // (floor(clamp(n,0,1)*255)/255*255).astype(uint8) == floor(clamp(n,0,1)*255); texture plane b, normal plane B + b
        uint8_t* tq = cond_u8 + pix * 3;
        uint8_t* nq = cond_u8 + (npix + pix) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            tq[c] = static_cast<uint8_t>(floorf(fminf(fmaxf(t3[c], 0.f), 255.f)));
            nq[c] = static_cast<uint8_t>(floorf(__fmul_rn(fminf(fmaxf(n3[c], 0.f), 1.f), 255.f)));
        }
    }
}

// util.vertex_normals (util.py:156-189) without atomics: every vertex sums the cross products of its face corners in the
// fixed order of a CSR adjacency (ascending face, then corner), so the result does not depend on scheduling or on the
// batch position.  Corner k of face (v0,v1,v2) contributes cross(v[k+1] - v[k], v[k+2] - v[k]) (indices mod 3), as the
// reference's three index_add calls do; then n / max(|n|, 1e-6) (F.normalize).
__device__ __forceinline__ void vertex_normal(const float* __restrict__ vb, const int* __restrict__ faces,
                                              const int* __restrict__ adj_off, const int* __restrict__ adj, int v,
                                              float* __restrict__ o) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    const int e1 = __ldg(adj_off + v + 1);
    for (int e = __ldg(adj_off + v); e < e1; ++e) {
        const int fc = __ldg(adj + e), f = fc / 3, k = fc - 3 * f;
        const int ia = __ldg(faces + f * 3 + (k + 1) % 3), ib = __ldg(faces + f * 3 + (k + 2) % 3);
        const float px = __ldg(vb + v * 3), py = __ldg(vb + v * 3 + 1), pz = __ldg(vb + v * 3 + 2);
        const float ux = __ldg(vb + ia * 3) - px, uy = __ldg(vb + ia * 3 + 1) - py, uz = __ldg(vb + ia * 3 + 2) - pz;
        const float wx = __ldg(vb + ib * 3) - px, wy = __ldg(vb + ib * 3 + 1) - py, wz = __ldg(vb + ib * 3 + 2) - pz;
        s0 += uy * wz - uz * wy;
        s1 += uz * wx - ux * wz;
        s2 += ux * wy - uy * wx;
    }
    const float d = fmaxf(sqrtf(s0 * s0 + s1 * s1 + s2 * s2), 1e-6f);
    o[0] = s0 / d;
    o[1] = s1 / d;
    o[2] = s2 / d;
}

// items [0, B*V): normals (B,V,3); items [B*V, B*V + B*F*3): face_normals (B,F,3,3), the normal of each face corner's vertex
__global__ void __launch_bounds__(256) vertex_normals_kernel(const float* __restrict__ verts, const int* __restrict__ faces,
                                                             const int* __restrict__ adj_off, const int* __restrict__ adj,
                                                             float* __restrict__ normals, float* __restrict__ face_normals,
                                                             int B, int V, int F) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long nv = normals ? static_cast<long long>(B) * V : 0;
    const long long nf = face_normals ? static_cast<long long>(B) * F * 3 : 0;
    if (i >= nv + nf) return;
    int b, v;
    float* o;
    if (i < nv) {
        b = static_cast<int>(i / V);
        v = static_cast<int>(i - static_cast<long long>(b) * V);
        o = normals + i * 3;
    } else {
        const long long j = i - nv;
        b = static_cast<int>(j / (3LL * F));
        v = __ldg(faces + (j - 3LL * F * b));
        o = face_normals + j * 3;
    }
    vertex_normal(verts + static_cast<long long>(b) * V * 3, faces, adj_off, adj, v, o);
}

}  // namespace gifb200

using namespace gifb200;

extern "C" int gifb200_render_shade(const int32_t* triangle, const float* bary, const float* face_uv,
                                    const float* face_normals, const float* albedo, const float* sh, float* tex,
                                    float* nrm, float* cond, uint8_t* cond_u8, int B, int F, int h, int w, int T,
                                    gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && F > 0 && h > 0 && w > 0 && T > 0, GIFB200_E_SHAPE, "render_shade: bad shape");
    if (B == 0) return GIFB200_OK;
    ShadeParams p{B, F, h, w, T};
    const long long npix = static_cast<long long>(B) * h * w;
    render_shade_kernel<<<cdiv(npix, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(triangle, bary, face_uv, face_normals,
                                                                                        albedo, sh, tex, nrm, cond, cond_u8, p);
    GIFB200_LAUNCH_CHECK("render_shade_kernel");
    return GIFB200_OK;
}

extern "C" int gifb200_vertex_normals(const float* verts, const int32_t* faces, const int32_t* adj_offsets,
                                      const int32_t* adj_corners, float* normals, float* face_normals, int B, int V, int F,
                                      gifb200_stream_t stream) {
    GIFB200_REQUIRE(B >= 0 && V > 0 && F > 0 && static_cast<long long>(V) * 3 < 2147483647LL &&
                    static_cast<long long>(F) * 3 < 2147483647LL, GIFB200_E_SHAPE, "vertex_normals: bad shape");
    const long long n = (normals ? static_cast<long long>(B) * V : 0) + (face_normals ? static_cast<long long>(B) * F * 3 : 0);
    if (n == 0) return GIFB200_OK;
    vertex_normals_kernel<<<cdiv(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(verts, faces, adj_offsets, adj_corners,
                                                                                    normals, face_normals, B, V, F);
    GIFB200_LAUNCH_CHECK("vertex_normals_kernel");
    return GIFB200_OK;
}
