// Hopper (sm_90a) building blocks of the wgmma kernels of this library: mbarrier, bulk-copy TMA, the wgmma shared-memory
// descriptor and the m64n128k8 tf32 wgmma with its A operand in registers.  Everything is inline PTX; there is no CUTLASS
// dependency.  The descriptor bit layout follows the PTX ISA's "matrix descriptor" table for wgmma.  mbar_init,
// mbar_arrive_expect_tx, smem_u32 and split_tf32 are shared with the other kernels and live in common.cuh.
#pragma once
#include "common.cuh"

namespace wg {

// ---- mbarrier ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init_fence() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t a = smem_u32(bar);
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}\n" ::"r"(a), "r"(parity) : "memory");
}

// ---- bulk copy (TMA engine, 1-D): global -> shared, completion counted on an mbarrier ------------------------------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// ---- operand layout ------------------------------------------------------------------------------------------------
// B tiles are K-major ("row n holds consecutive k") with 32 fp32/tf32 elements = 128 bytes of k per row, stored as the
// canonical SWIZZLE_128B layout: row n at byte n*128, its 16-byte chunk c at position (c ^ (n & 7)); 8-row groups are 1024
// bytes apart (= the descriptor's stride byte offset).  Tile bases must be 1024-byte aligned.  One wgmma of tf32 consumes
// k = 8 (32 bytes): k-slice s of the tile is addressed by advancing the start address by 32*s bytes.
constexpr uint32_t ROW_BYTES = 128;

// byte offset of element (n, k) of a K-major SWIZZLE_128B tile, k in [0, 32)
__host__ __device__ __forceinline__ uint32_t sw128_off(uint32_t n, uint32_t k) {
    return n * ROW_BYTES + ((((k >> 2) ^ (n & 7u)) & 7u) << 4) + ((k & 3u) << 2);
}

__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFFu);          // [0,14)  start address >> 4
    d |= (uint64_t)1 << 16;                           // [16,30) leading byte offset >> 4 (unused: one swizzle atom along k)
    d |= (uint64_t)(1024u >> 4) << 32;                // [32,46) stride byte offset >> 4: 8 rows x 128 B
    d |= (uint64_t)1 << 62;                           // [62,64) layout: SWIZZLE_128B
    return d;
}

// ---- wgmma ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// keeps the compiler from moving accesses of an accumulator across the asynchronous wgmma that owns it
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] (+)= A[64 x 8] * B[128 x 8]^T for the whole warpgroup.  A in registers: thread (warp w, lane l) holds rows
// 16w + l/4 (a0, a2) and 16w + l/4 + 8 (a1, a3) at k = l%4 (a0, a1) and l%4 + 4 (a2, a3).  D: d[4i + {0,1}] = row
// 16w + l/4, columns 8i + 2(l%4) + {0,1}; d[4i + {2,3}] = the same columns of row 16w + l/4 + 8.
__device__ __forceinline__ void wgmma_m64n128k8_tf32_rs(float (&d)[64], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                        uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(desc_b), "r"(accumulate)
        : "memory");
}

}  // namespace wg
