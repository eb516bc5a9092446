// Optimiser step over ONE flat parameter buffer: deterministic slab reduction + global grad norm,
// then clip (by global norm, ppo.py:244-246,349-351; or by value, ddpg.py:309,332) + Adam.
//
// Replaces nn.utils.clip_grad_norm_ / clip_grad_value_ and torch.optim.Adam.step() (default betas/eps,
// L2 weight decay; surreal/learner/ppo.py:159-168, ddpg.py:145-165).  The arithmetic follows torch's
// single-tensor Adam (lerp_ / mul_.addcmul_ / sqrt./.add_ / addcdiv_) operation by operation so that
// fp32 results agree with the reference to rounding.  The step counter lives on the device so that the
// whole update can be replayed from a CUDA graph.
#include "common.cuh"
#include "optim_dev.cuh"

namespace {

using optim_dev::OptWs;

constexpr int OT = 256;

__global__ void __launch_bounds__(OT) grad_reduce_norm_kernel(const float* __restrict__ slabs, long long slab_stride,
                                                              int splits, float* __restrict__ grad, long long n,
                                                              float scale, int bump_step, OptWs* ws,
                                                              const int* __restrict__ stop) {
    if (stop != nullptr && *stop) return;
    __shared__ double sh[32];
    double sq = 0.0;
    for (long long i = (long long)blockIdx.x * OT + threadIdx.x; i < n; i += (long long)gridDim.x * OT) {
        float g = slabs[i];
        for (int z = 1; z < splits; ++z) g += slabs[(long long)z * slab_stride + i];   // fixed order
        if (scale != 1.0f) g = __fmul_rn(g, scale);
        grad[i] = g;
        sq += (double)g * (double)g;
    }
    const double t = block_sum(sq, sh);
    if (threadIdx.x == 0) ws->partial[blockIdx.x] = t;
    if (last_block_ticket(&ws->counter, gridDim.x) && threadIdx.x == 0)
        optim_dev::finish_norm(ws, ws->partial, gridDim.x, bump_step);
}

__global__ void __launch_bounds__(OT) clip_adam_kernel(float* __restrict__ p, const float* __restrict__ grad,
                                                       float* __restrict__ m, float* __restrict__ v, long long n,
                                                       const double* __restrict__ lr_ptr, double beta1, double beta2,
                                                       double eps, double weight_decay, int clip_mode,
                                                       double clip_value, const OptWs* __restrict__ ws,
                                                       float* __restrict__ norm_out, const int* __restrict__ stop) {
    if (stop != nullptr && *stop) return;
    const optim_dev::AdamCoef c = optim_dev::adam_coef(ws->step, lr_ptr[0], beta1, beta2, eps, weight_decay, clip_mode,
                                                       clip_value, ws->total_norm);
    if (norm_out != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *norm_out = ws->total_norm;
    for (long long i = (long long)blockIdx.x * OT + threadIdx.x; i < n; i += (long long)gridDim.x * OT) {
        float pi = p[i], mi = m[i], vi = v[i];
        optim_dev::adam_apply(c, grad[i], pi, mi, vi);
        p[i] = pi;
        m[i] = mi;
        v[i] = vi;
    }
}

__global__ void __launch_bounds__(OT) soft_update_kernel(float* __restrict__ target, const float* __restrict__ src,
                                                         long long n, float tau, const int* __restrict__ stop) {
    if (stop != nullptr && *stop) return;
    const float keep = 1.0f - tau;
    for (long long i = (long long)blockIdx.x * OT + threadIdx.x; i < n; i += (long long)gridDim.x * OT)
        target[i] = __fadd_rn(__fmul_rn(target[i], keep), __fmul_rn(tau, src[i]));
}

// Hard target update on the device, PeriodicTracker(period).track_increment(incr) on a device counter (ddpg.py:419-428
// counts updates, incr = 1; dqn.py:84-86 counts samples, incr = batch size), so that several learner updates, and the
// ones among them that copy, fit in one CUDA graph.  `tick` adds incr; the copy runs when the count crossed a multiple
// of the period, floor(c / period) > floor((c - incr) / period) -- for incr = 1 and c >= 1 that is c % period == 0.
// Both leave everything alone when *stop != 0.
__global__ void hard_update_tick_kernel(long long* counter, long long incr, const int* __restrict__ stop) {
    if (stop != nullptr && *stop) return;
    *counter += incr;
}

__global__ void __launch_bounds__(OT) hard_update_kernel(float* __restrict__ target, const float* __restrict__ src,
                                                         long long n, const long long* __restrict__ counter,
                                                         long long period, long long incr, const int* __restrict__ stop) {
    if (stop != nullptr && *stop) return;
    const long long c = *counter;
    if (c / period <= (c - incr) / period) return;
    for (long long i = (long long)blockIdx.x * OT + threadIdx.x; i < n; i += (long long)gridDim.x * OT)
        target[i] = src[i];
}

inline int grid_for(long long n) {
    long long b = (n + 4 * OT - 1) / (4 * OT);   // >= 4 elements per thread: small nets finish in one short wave
    if (b > 264) b = 264;          // 2 x 132 SMs, grid-stride
    if (b < 1) b = 1;
    return (int)b;
}

}  // namespace

extern "C" size_t sb200_optim_workspace_bytes(void) { return sizeof(OptWs); }

extern "C" int sb200_grad_reduce_norm_f32(const float* slabs, int64_t slab_stride, int splits, float* grad, int64_t n,
                                          double scale, int bump_step, void* workspace, const int* stop_flag,
                                          void* stream) {
    SB200_REQUIRE(slabs && grad && workspace && splits >= 1 && n >= 1);
    grad_reduce_norm_kernel<<<grid_for(n), OT, 0, (cudaStream_t)stream>>>(slabs, slab_stride, splits, grad, n,
                                                                          (float)scale, bump_step, (OptWs*)workspace,
                                                                          stop_flag);
    return sb200_launch_status();
}

extern "C" int sb200_clip_adam_f32(float* params, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                                   const double* lr, double beta1, double beta2, double eps, double weight_decay,
                                   int clip_mode, double clip_value, void* workspace, float* norm_out,
                                   const int* stop_flag, void* stream) {
    SB200_REQUIRE(params && grad && exp_avg && exp_avg_sq && lr && workspace && n >= 1);
    SB200_REQUIRE(clip_mode >= 0 && clip_mode <= 2);
    clip_adam_kernel<<<grid_for(n), OT, 0, (cudaStream_t)stream>>>(params, grad, exp_avg, exp_avg_sq, n, lr, beta1,
                                                                   beta2, eps, weight_decay, clip_mode, clip_value,
                                                                   (const OptWs*)workspace, norm_out, stop_flag);
    return sb200_launch_status();
}

extern "C" int sb200_soft_update_f32(float* target, const float* src, int64_t n, double tau, const int* stop_flag,
                                     void* stream) {
    SB200_REQUIRE(target && src && n >= 1);
    soft_update_kernel<<<grid_for(n), OT, 0, (cudaStream_t)stream>>>(target, src, n, (float)tau, stop_flag);
    return sb200_launch_status();
}

extern "C" int sb200_hard_update_f32(float* target, const float* src, int64_t n, int64_t* counter, int64_t period,
                                     int64_t incr, int tick, const int* stop_flag, void* stream) {
    SB200_REQUIRE(target && src && counter && n >= 1 && period >= 1 && incr >= 0);
    if (tick) hard_update_tick_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((long long*)counter, incr, stop_flag);
    hard_update_kernel<<<grid_for(n), OT, 0, (cudaStream_t)stream>>>(target, src, n, (const long long*)counter, period,
                                                                     incr, stop_flag);
    return sb200_launch_status(tick ? 2 : 1);
}
