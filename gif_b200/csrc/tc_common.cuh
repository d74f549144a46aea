// Shared wgmma / TMA / mbarrier plumbing for the sm_90a tensor-core kernels (conv_tc.cu, conv_wgrad_tc.cu).
#pragma once
#include <cuda.h>

#include <mutex>

#include "common.cuh"

namespace gifb200 {

// ----------------------------------------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}
// ----------------------------------------------------------------------------------------------- wgmma (sm_90a)
// Warpgroup MMA: D (registers of the 128 threads of a warpgroup, m64nN fp32) (+)= A[smem desc] * B[smem desc].
// Accumulator fragment of thread t (warp w = t / 32 of the warpgroup, lane l): d[4j + 2h + e] is row 16w + l/4 + 8h,
// column 8j + 2(l%4) + e.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_regs(float* d) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int V>
struct Trans {};
// kind tf32: both operands K-major (the only layout wgmma accepts for 32-bit types); K = 8 per instruction
template <int N>
__device__ __forceinline__ void wgmma_tf32(float* d, uint64_t da, uint64_t db, int scale_d);
// bf16 operands, fp32 accumulate, K = 16 per instruction; Trans<1>: both operands MN-major (transposed)
template <int N, int T>
__device__ __forceinline__ void wgmma_bf16(float* d, uint64_t da, uint64_t db, int scale_d, Trans<T>);
// operand lists of the accumulator fragment: N/2 "+f" registers, and the matching "%0, %1, ..." of the PTX template
#define GIF_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define GIF_F16 GIF_F8(0), GIF_F8(8)
#define GIF_F32 GIF_F16, GIF_F8(16), GIF_F8(24)
#define GIF_F64 GIF_F32, GIF_F8(32), GIF_F8(40), GIF_F8(48), GIF_F8(56)
#define GIF_R8(a, b, c, d, e, f, g, h) "%" #a ", %" #b ", %" #c ", %" #d ", %" #e ", %" #f ", %" #g ", %" #h
#define GIF_R16 GIF_R8(0, 1, 2, 3, 4, 5, 6, 7) ", " GIF_R8(8, 9, 10, 11, 12, 13, 14, 15)
#define GIF_R32 GIF_R16 ", " GIF_R8(16, 17, 18, 19, 20, 21, 22, 23) ", " GIF_R8(24, 25, 26, 27, 28, 29, 30, 31)
#define GIF_R64 GIF_R32 ", " GIF_R8(32, 33, 34, 35, 36, 37, 38, 39) ", " GIF_R8(40, 41, 42, 43, 44, 45, 46, 47) ", " \
    GIF_R8(48, 49, 50, 51, 52, 53, 54, 55) ", " GIF_R8(56, 57, 58, 59, 60, 61, 62, 63)
// operands after the accumulators: descriptors %R, %R+1, scale-d %R+2 (, transpose immediates %R+3, %R+4)
#define GIF_WGMMA_TF32(N, R, S0, S1, S2) \
    template <> \
    __device__ __forceinline__ void wgmma_tf32<N>(float* d, uint64_t da, uint64_t db, int scale_d) { \
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #S2 ", 0;\n" \
                     "wgmma.mma_async.sync.aligned.m64n" #N "k8.f32.tf32.tf32 {" GIF_R##R "}, %" #S0 ", %" #S1 \
                     ", p, 1, 1;\n}\n" \
                     : GIF_F##R \
                     : "l"(da), "l"(db), "r"(scale_d)); \
    }
#define GIF_WGMMA_BF16(N, R, S0, S1, S2, T0, T1, TR) \
    template <> \
    __device__ __forceinline__ void wgmma_bf16<N>(float* d, uint64_t da, uint64_t db, int scale_d, Trans<TR>) { \
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #S2 ", 0;\n" \
                     "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 {" GIF_R##R "}, %" #S0 ", %" #S1 \
                     ", p, 1, 1, %" #T0 ", %" #T1 ";\n}\n" \
                     : GIF_F##R \
                     : "l"(da), "l"(db), "r"(scale_d), "n"(TR), "n"(TR)); \
    }
GIF_WGMMA_TF32(32, 16, 16, 17, 18)
GIF_WGMMA_TF32(64, 32, 32, 33, 34)
GIF_WGMMA_TF32(128, 64, 64, 65, 66)
GIF_WGMMA_BF16(32, 16, 16, 17, 18, 19, 20, 0)
GIF_WGMMA_BF16(64, 32, 32, 33, 34, 35, 36, 0)
GIF_WGMMA_BF16(128, 64, 64, 65, 66, 67, 68, 0)
GIF_WGMMA_BF16(32, 16, 16, 17, 18, 19, 20, 1)
GIF_WGMMA_BF16(64, 32, 32, 33, 34, 35, 36, 1)

// warp-level tensor-core MMA, m16n8k8, tf32 operands, fp32 accumulate (the weight-gradient kernel's tf32 mode: its operands
// are MN-major in shared memory, which wgmma does not accept for 32-bit types, so the fragments are gathered with lds)
__device__ __forceinline__ void mma_tf32_m16n8k8(float* c, const uint32_t* a, const uint32_t* b) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// Shared-memory matrix descriptor (sm_90 GMMA): start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | base_offset [49,52) |
// layout [62,64): 1 = SWIZZLE_128B, 2 = SWIZZLE_64B
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
    d |= static_cast<uint64_t>(lbo_bytes >> 4) << 16;
    d |= static_cast<uint64_t>(sbo_bytes >> 4) << 32;
    d |= static_cast<uint64_t>(layout) << 62;
    return d;
}
// K-major, SWIZZLE_128B (rows of 128 bytes = 32 fp32; 8-row atoms of 1024 B)
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr) { return make_smem_desc(smem_addr, 16, 1024, 1); }
// K-major, SWIZZLE_64B (rows of 64 bytes = 32 bf16; 8-row atoms of 512 B)
__device__ __forceinline__ uint64_t make_kmajor_sw64_desc(uint32_t smem_addr) { return make_smem_desc(smem_addr, 16, 512, 2); }

// ----------------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn get_encode() {
    static EncodeTiledFn g_encode = nullptr;
    static std::once_flag g_encode_once;
    std::call_once(g_encode_once, [] {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            g_encode = reinterpret_cast<EncodeTiledFn>(fn);
    });
    return g_encode;
}

inline int encode_map(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                      const cuuint32_t* box, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B,
                      CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT32, const cuuint32_t* elem_strides = nullptr) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return fail(GIFB200_E_ARCH, "cuTensorMapEncodeTiled driver entry point not available");
    // elem_strides: traversal stride per dimension (a box of n elements with stride s loads ceil(n / s) of them)
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    if (elem_strides)
        for (int i = 0; i < rank; ++i) estr[i] = elem_strides[i];
    CUresult r = enc(map, dtype, rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char msg[64];
        snprintf(msg, sizeof(msg), "CUresult %d", static_cast<int>(r));
        return fail(GIFB200_E_CUDA, "cuTensorMapEncodeTiled failed", msg);
    }
    return GIFB200_OK;
}


}  // namespace gifb200
