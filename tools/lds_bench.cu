// Micro-benchmark (dev tool, not shipped): cycles per warp-wide shared-memory load as a function of width and of the
// number of DISTINCT addresses in the warp -- decides the register-tile shape of the persistent rollout kernel.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/lds_bench tools/lds_bench.cu
#include <cstdio>
#include <cuda_runtime.h>

template <int W>   // W = floats per load (1, 2, 4)
__global__ void k(const int* __restrict__ offs, long long* out, float* sink, int iters) {
    extern __shared__ __align__(16) float sm[];
    for (int i = threadIdx.x; i < 8192; i += blockDim.x) sm[i] = (float)i;
    __syncthreads();
    int o = offs[threadIdx.x & 31];
    float acc = 0.f;
    long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int u = 0; u < 16; ++u) {
            const float* p = sm + ((o + u * 64 + (it & 1) * 32) & 8191 & ~3);
            if (W == 4) { float4 v = *reinterpret_cast<const float4*>(p); acc += v.x + v.y + v.z + v.w; }
            else if (W == 2) { float2 v = *reinterpret_cast<const float2*>(p); acc += v.x + v.y; }
            else acc += *p;
        }
    }
    long long t1 = clock64();
    if (threadIdx.x == 0) out[blockIdx.x] = t1 - t0;
    if (acc == 12345.678f) sink[0] = acc;
}

int main() {
    int* d_offs; long long* d_out; float* d_sink;
    cudaMalloc(&d_offs, 32 * 4); cudaMalloc(&d_out, 8); cudaMalloc(&d_sink, 4);
    struct Pat { const char* name; int (*f)(int); };
    Pat pats[] = {
        {"all lanes same address", [](int l) { return 0; }},
        {"2 distinct 16B (lane>>4), stride 260 floats", [](int l) { return (l >> 4) * 260; }},
        {"4 distinct 16B (lane>>3), stride 260", [](int l) { return (l >> 3) * 260; }},
        {"8 distinct 16B (lane>>2), stride 68", [](int l) { return (l >> 2) * 68; }},
        {"8 distinct contiguous 16B (lane&7)", [](int l) { return (l & 7) * 4; }},
        {"16 distinct contiguous 16B (lane&15)", [](int l) { return (l & 15) * 4; }},
        {"32 distinct contiguous 16B", [](int l) { return l * 4; }},
        {"32 distinct contiguous 4B", [](int l) { return l; }},
        {"8 distinct contiguous 4B x4 bcast (lane&7)", [](int l) { return (l & 7); }},
    };
    const int iters = 2000;
    for (int nw : {1, 4, 16}) {
        printf("---- %d warps per CTA (1 CTA), cycles per warp-load instruction (issue-side, CTA total / loads per warp)\n", nw);
        for (auto& p : pats) {
            int h[32];
            for (int l = 0; l < 32; ++l) h[l] = p.f(l);
            cudaMemcpy(d_offs, h, sizeof(h), cudaMemcpyHostToDevice);
            for (int W : {4, 2, 1}) {
                long long c = 0;
                for (int rep = 0; rep < 2; ++rep) {
                    if (W == 4) k<4><<<1, nw * 32, 32768>>>(d_offs, d_out, d_sink, iters);
                    if (W == 2) k<2><<<1, nw * 32, 32768>>>(d_offs, d_out, d_sink, iters);
                    if (W == 1) k<1><<<1, nw * 32, 32768>>>(d_offs, d_out, d_sink, iters);
                    cudaDeviceSynchronize();
                    cudaMemcpy(&c, d_out, 8, cudaMemcpyDeviceToHost);
                }
                // all nw warps run concurrently: SM-level cycles per warp-load = c / (iters*16) / nw
                printf("  %-46s W=%d  %6.2f cyc/warp-load (per SM: %5.2f)\n", p.name, W, (double)c / (iters * 16.0), (double)c / (iters * 16.0) / nw);
            }
        }
    }
    cudaError_t e = cudaGetLastError();
    printf("status %s\n", cudaGetErrorString(e));
    return 0;
}
