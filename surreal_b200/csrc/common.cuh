// Shared device/host helpers for libsurreal_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/surreal_b200.h"

#define SB200_THREADS 256

// c + a * b on a pair of fp32 lanes: two IEEE fmas (sm_90 has no packed fp32 fma)
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

extern unsigned long long g_sb200_launches;     // kernels launched by this library (api.cu)

static inline int sb200_launch_status(int kernels = 1) {
    g_sb200_launches += (unsigned long long)kernels;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) return SB200_OK;
    fprintf(stderr, "[surreal_b200] CUDA launch error: %s\n", cudaGetErrorString(e));
    return SB200_ERR_CUDA;
}

#define SB200_REQUIRE(cond)                                                             \
    do {                                                                                \
        if (!(cond)) {                                                                  \
            fprintf(stderr, "[surreal_b200] invalid argument: %s (%s:%d)\n", #cond,     \
                    __FILE__, __LINE__);                                                \
            return SB200_ERR_ARG;                                                       \
        }                                                                               \
    } while (0)

#define SB200_CUDA(call)                                                                \
    do {                                                                                \
        cudaError_t e__ = (call);                                                       \
        if (e__ != cudaSuccess) {                                                       \
            fprintf(stderr, "[surreal_b200] %s failed: %s\n", #call,                    \
                    cudaGetErrorString(e__));                                           \
            return SB200_ERR_CUDA;                                                      \
        }                                                                               \
    } while (0)

// Does the descriptor carry a LayerNorm (sb200_mlp.ln_g / ln_b)?  Entries that do not implement it reject such nets.
static inline bool sb200_mlp_has_ln(const sb200_mlp* net) {
    for (int l = 0; l < SB200_MAX_LAYERS; ++l)
        if (net->ln_g[l] != nullptr || net->ln_b[l] != nullptr) return true;
    return false;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Block-wide sum of doubles (all threads get the result). `sh` needs >= 32 doubles.
__device__ __forceinline__ double block_sum(double v, double* sh) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();                 // protect sh from a previous use
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    double t = (lane < nw) ? sh[lane] : 0.0;
    t = warp_sum(t);
    return t;
}

// "Last block done" ticket: returns true in exactly one block, after every other block's prior
// global writes are visible to it.  `counter` must be 0 on entry and is reset to 0 by the winner.
__device__ __forceinline__ bool last_block_ticket(unsigned int* counter, unsigned int nblocks) {
    __shared__ bool is_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned int t = atomicAdd(counter, 1u);
        is_last = (t == nblocks - 1);
        if (is_last) *counter = 0u;
    }
    __syncthreads();
    if (is_last) __threadfence();
    return is_last;
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src, int src_bytes) {
    unsigned int d = (unsigned int)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(gmem_src), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ float4 ld_stream4(const float* p) {   // read-once data: bypass L1 allocation
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}

// Philox4x32-10 counter-based generator (Salmon et al. 2011), written from the published round
// function; one call yields 4 x 32 random bits for (key, counter).
struct Philox4 { unsigned int x, y, z, w; };
__device__ __forceinline__ Philox4 philox4x32_10(unsigned long long seed, unsigned long long ctr_lo,
                                                 unsigned long long ctr_hi) {
    unsigned int k0 = (unsigned int)seed, k1 = (unsigned int)(seed >> 32);
    unsigned int c0 = (unsigned int)ctr_lo, c1 = (unsigned int)(ctr_lo >> 32);
    unsigned int c2 = (unsigned int)ctr_hi, c3 = (unsigned int)(ctr_hi >> 32);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        unsigned int hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        unsigned int hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        unsigned int n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    Philox4 o = {c0, c1, c2, c3};
    return o;
}
// two N(0,1) from two 32-bit words (Box-Muller, fp32)
__device__ __forceinline__ float2 box_muller(unsigned int a, unsigned int b) {
    float u1 = ((float)a + 1.0f) * 2.3283064365386963e-10f;     // (0,1]
    float u2 = (float)b * 2.3283064365386963e-10f;               // [0,1)
    float rad = sqrtf(-2.0f * logf(u1));
    float s, c;
    sincosf(6.283185307179586f * u2, &s, &c);
    return make_float2(rad * c, rad * s);
}
