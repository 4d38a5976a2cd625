// rsb_tc.cuh -- thin inline-PTX wrappers for the Hopper (sm_90a) tensor-core path shared by the encoder GEMM
// (rsb_bert.cu, f16 / bf16) and the coarse-quantizer GEMM (rsb_tf32.cu, tf32): mbarrier, TMA tensor loads, warpgroup
// MMAs (wgmma.mma_async) and the K-major 128B-swizzle shared-memory descriptor.
#ifndef RSB_TC_CUH_
#define RSB_TC_CUH_

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace rsbtc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// ---- wgmma (sm_90a): D[64 x 128] (fp32 registers of one warpgroup) += A[64 x K] . B[128 x K]^T, both operands K-major in
// shared memory with the 128-byte swizzle.  Accumulator fragment of thread t of the warpgroup: d[4 j + 2 h + c] holds
// row 16 (t / 32) + (t % 32) / 4 + 8 h, column 8 j + 2 (t % 4) + c.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
__device__ __forceinline__ void acc_fence(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define RSB_WG_D64                                                                                                    \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "   \
    "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, " \
    "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define RSB_WG_OUT64(d)                                                                                                \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),         \
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),          \
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),         \
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),         \
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),         \
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),         \
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),         \
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])

// K = 16 f16 elements (32 bytes of each operand row)
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " RSB_WG_D64 ", %64, %65, p, 1, 1, 0, 0;\n}\n"
                 : RSB_WG_OUT64(d)
                 : "l"(adesc), "l"(bdesc), "r"(1));
}
// K = 16 bf16 elements (32 bytes of each operand row)
__device__ __forceinline__ void wgmma_bf16_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " RSB_WG_D64 ", %64, %65, p, 1, 1, 0, 0;\n}\n"
                 : RSB_WG_OUT64(d)
                 : "l"(adesc), "l"(bdesc), "r"(1));
}
// K = 8 tf32 elements (32 bytes of each operand row)
__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " RSB_WG_D64 ", %64, %65, p, 1, 1;\n}\n"
                 : RSB_WG_OUT64(d)
                 : "l"(adesc), "l"(bdesc), "r"(1));
}
#undef RSB_WG_D64
#undef RSB_WG_OUT64

// named barrier over `count` threads (the warpgroups of a kernel that do not include the producer)
__device__ __forceinline__ void named_sync(uint32_t id, uint32_t count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ uint64_t make_sw128_kmajor_desc(uint32_t smem_addr) {
    // wgmma matrix descriptor: start >> 4 in [0,14) | LBO >> 4 in [16,30) = 1 (unused for swizzled K-major)
    // | SBO >> 4 in [32,46) = 1024 B between 8-row groups | base offset [49,52) = 0 (1024-byte aligned tiles)
    // | layout [62,64) = 1 (SWIZZLE_128B).  Advancing K by 32 bytes inside the swizzle row adds 2 to the start field.
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// ---- host: tensor-map encoding through the driver entry point (no link-time dependency on libcuda) ----------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && p)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}
// row-major [rows, cols] matrix of 2-byte (f16, or bf16 with bf16 set) or 4-byte (f32) elements; box = one 128-byte
// swizzle row of columns x box_rows; rows beyond `rows` read as zero
inline bool make_map_2d(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows, int elem_bytes,
                        bool bf16 = false) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    const cuuint64_t dims[2] = {cols, rows};
    const cuuint64_t strides[1] = {cols * (uint64_t)elem_bytes};
    const cuuint32_t box[2] = {(cuuint32_t)(128 / elem_bytes), box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUtensorMapDataType dt = elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                   : bf16         ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                  : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    return enc(m, dt, 2,
               const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace rsbtc
#endif
