// One-shot all-reduce over NVLink peer memory for the SMALL, latency-bound exchanges of the data-parallel learner
// (SURVEY §8e: the ~330 KB flat gradient of every optimiser step, the KL scalar, advantage moments, z-filter sums).
//
// Every rank owns a "symmetric" buffer allocated with cudaMalloc and exported through CUDA IPC; all ranks of the box map
// each other's buffers (NVSwitch: every peer at full NVLink bandwidth).  One kernel launch per all-reduce:
//
//   1. each CTA copies its slice of the local input into the rank's own slot (double-buffered by call parity),
//   2. publishes "slice b of call k is ready" by storing k into flag[rank][b] of EVERY peer (system-scope release),
//   3. waits until the same flag from every peer has reached k (acquire),
//   4. reads the slice from every rank's slot in RANK ORDER, sums (bit-identical result on all ranks: no replica
//      drift), scales, writes the output and -- optionally -- accumulates the squared norm for the gradient clip
//      (the work of sb200_grad_reduce_norm_f32, fused), finishing with a last-CTA ticket.
//
// No second barrier is needed: slot (k & 1) is rewritten at call k+2, and a rank can only get there after every peer has
// signalled call k+1, i.e. has finished reading call k.  A ~330 KB gradient costs one NVLink round trip plus 8 x 330 KB of
// peer reads instead of an NCCL launch + ring/tree protocol (~30-40 us on this box for messages this small).
// The call counter lives in device memory, so the launch can be captured in a CUDA graph and replayed.
#include "common.cuh"
#include "optim_dev.cuh"
#include "peer_dev.cuh"
#include <string.h>

namespace {

using namespace peer_dev;

constexpr int PAR_T = 256;

__global__ void __launch_bounds__(PAR_T) par_allreduce_kernel(const __grid_constant__ sb200_par c, const float* __restrict__ x,
                                                              float* __restrict__ out, long long n, float scale, int bump_step,
                                                              optim_dev::OptWs* ws, const int* __restrict__ stop) {
    ParHeader* me = header_of(c, c.rank);
    __shared__ double sh[32];
    const int b = blockIdx.x, G = gridDim.x, tid = threadIdx.x;
    // NOTE: the exchange itself is unconditional (every rank must take part in every call); `stop` only gates the norm /
    // step bookkeeping, exactly like sb200_grad_reduce_norm_f32
    const unsigned int k = me->counter + 1u;
    const unsigned int parity = k & 1u;
    long long per = (n + G - 1) / G;
    per = (per + 3) & ~3ll;                                   // 16-byte aligned slices
    const long long lo = (long long)b * per;
    const long long hi = (lo + per < n) ? lo + per : n;
    float* mine = slot_of(c, c.rank, parity);
    const bool vec = ((((uintptr_t)x) | ((uintptr_t)out)) & 15) == 0;
    // 1. local slice -> own slot
    if (vec) {
        for (long long i = lo + 4 * tid; i + 3 < hi; i += 4 * PAR_T)
            *reinterpret_cast<float4*>(mine + i) = *reinterpret_cast<const float4*>(x + i);
        const long long tail = lo + ((hi - lo) & ~3ll);
        for (long long i = tail + tid; i < hi; i += PAR_T) mine[i] = x[i];
    } else {
        for (long long i = lo + tid; i < hi; i += PAR_T) mine[i] = x[i];
    }
    __threadfence_system();
    // 2. publish, 3. wait
    publish_and_wait(c, me, b, k);
    // 4. sum in rank order
    double sq = 0.0;
    const float* slots[PAR_MAX_WORLD];
#pragma unroll
    for (int p = 0; p < PAR_MAX_WORLD; ++p) slots[p] = (p < c.world) ? slot_of(c, p, parity) : nullptr;
    if (vec) {
        for (long long i = lo + 4 * tid; i + 3 < hi; i += 4 * PAR_T) {
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int p = 0; p < PAR_MAX_WORLD; ++p) {
                if (p < c.world) {
                    const float4 v = ld_sys4(slots[p] + i);
                    a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
                }
            }
            if (scale != 1.0f) { a.x = __fmul_rn(a.x, scale); a.y = __fmul_rn(a.y, scale); a.z = __fmul_rn(a.z, scale); a.w = __fmul_rn(a.w, scale); }
            *reinterpret_cast<float4*>(out + i) = a;
            sq += (double)a.x * a.x + (double)a.y * a.y + (double)a.z * a.z + (double)a.w * a.w;
        }
        const long long tail = lo + ((hi - lo) & ~3ll);
        for (long long i = tail + tid; i < hi; i += PAR_T) {
            float a = 0.f;
            for (int p = 0; p < c.world; ++p) a += ld_sys1(slots[p] + i);
            if (scale != 1.0f) a = __fmul_rn(a, scale);
            out[i] = a;
            sq += (double)a * a;
        }
    } else {
        for (long long i = lo + tid; i < hi; i += PAR_T) {
            float a = 0.f;
            for (int p = 0; p < c.world; ++p) a += ld_sys1(slots[p] + i);
            if (scale != 1.0f) a = __fmul_rn(a, scale);
            out[i] = a;
            sq += (double)a * a;
        }
    }
    const double t = block_sum(sq, sh);
    if (tid == 0) me->partial[b] = t;
    if (last_block_ticket(&me->ticket, G)) {
        if (tid == 0) {
            me->counter = k;                                   // this rank has completed call k
            if (ws != nullptr && !(stop != nullptr && *stop)) optim_dev::finish_norm(ws, me->partial, G, bump_step);
        }
    }
}

// float64 variant for the scalar exchanges (KL, advantage moments): a handful of elements, one CTA, same protocol
__global__ void __launch_bounds__(64) par_allreduce_f64_kernel(const __grid_constant__ sb200_par c, const double* __restrict__ x,
                                                               double* __restrict__ out, int n, double scale) {
    ParHeader* me = header_of(c, c.rank);
    const int tid = threadIdx.x;
    const unsigned int k = me->counter + 1u;
    const unsigned int parity = k & 1u;
    double* mine = reinterpret_cast<double*>(slot_of(c, c.rank, parity));
    for (int i = tid; i < n; i += 64) mine[i] = x[i];
    __threadfence_system();
    publish_and_wait(c, me, 0, k);
    for (int i = tid; i < n; i += 64) {
        double a = 0.0;
        for (int p = 0; p < c.world; ++p) a += ld_sys_f64(reinterpret_cast<const double*>(slot_of(c, p, parity)) + i);
        out[i] = a * scale;
    }
    __syncthreads();
    if (tid == 0) me->counter = k;
}

}  // namespace

extern "C" size_t sb200_par_buffer_bytes(int64_t max_floats) {
    return sizeof(ParHeader) + 2 * (size_t)max_floats * sizeof(float);
}

// cudaMalloc + zero + IPC export of a symmetric buffer (the caching allocators of frameworks sub-allocate, which CUDA IPC
// cannot export: this buffer is a whole allocation of its own).  handle_out: 64 bytes.
extern "C" int sb200_par_alloc(int64_t max_floats, void** ptr_out, void* handle_out) {
    SB200_REQUIRE(ptr_out && handle_out && max_floats >= 4 && max_floats % 4 == 0);
    void* p = nullptr;
    SB200_CUDA(cudaMalloc(&p, sb200_par_buffer_bytes(max_floats)));
    SB200_CUDA(cudaMemset(p, 0, sb200_par_buffer_bytes(max_floats)));
    SB200_CUDA(cudaDeviceSynchronize());
    cudaIpcMemHandle_t h;
    SB200_CUDA(cudaIpcGetMemHandle(&h, p));
    memcpy(handle_out, &h, sizeof(h));
    *ptr_out = p;
    return SB200_OK;
}

extern "C" int sb200_par_open(const void* handle, void** ptr_out) {
    SB200_REQUIRE(handle && ptr_out);
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    SB200_CUDA(cudaIpcOpenMemHandle(ptr_out, h, cudaIpcMemLazyEnablePeerAccess));
    return SB200_OK;
}

extern "C" int sb200_par_close(void* ptr, int own) {
    if (ptr == nullptr) return SB200_OK;
    if (own) { SB200_CUDA(cudaFree(ptr)); } else { SB200_CUDA(cudaIpcCloseMemHandle(ptr)); }
    return SB200_OK;
}

// out[i] = scale * sum_p x_p[i] over the ranks of `ctx`, identical bits on every rank; optionally the gradient-norm / step
// bookkeeping of sb200_grad_reduce_norm_f32 on the result (opt_workspace may be NULL).
extern "C" int sb200_par_allreduce_f32(const sb200_par* ctx, const float* x, float* out, int64_t n, double scale, int bump_step,
                                       void* opt_workspace, const int* stop_flag, void* stream) {
    SB200_REQUIRE(x && out && n >= 1);
    if (const int e = sb200_par_check(ctx, n)) return e;
    int G = (int)((n + 16383) / 16384);                        // ~64 KB of fp32 per CTA
    if (G < 1) G = 1;
    if (G > PAR_MAX_CTAS) G = PAR_MAX_CTAS;
    par_allreduce_kernel<<<G, PAR_T, 0, (cudaStream_t)stream>>>(*ctx, x, out, n, (float)scale, bump_step,
                                                                (optim_dev::OptWs*)opt_workspace, stop_flag);
    return sb200_launch_status();
}

extern "C" int sb200_par_allreduce_f64(const sb200_par* ctx, const double* x, double* out, int n, double scale, void* stream) {
    SB200_REQUIRE(x && out && n >= 1);
    if (const int e = sb200_par_check(ctx, 2ll * n)) return e;
    par_allreduce_f64_kernel<<<1, 64, 0, (cudaStream_t)stream>>>(*ctx, x, out, n, scale);
    return sb200_launch_status();
}
