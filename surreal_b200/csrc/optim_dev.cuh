// Optimiser pieces shared by the stand-alone kernels (optim.cu, peer_allreduce.cu) and the persistent learner kernel
// (epoch2.cu): the device-resident workspace and torch's single-tensor Adam, operation by operation.
#pragma once
#include "common.cuh"

namespace optim_dev {

constexpr int MAX_BLOCKS = 1024;

struct OptWs {                           // sb200_optim_workspace_bytes() bytes
    unsigned int counter;
    int step;
    float total_norm;
    float pad;
    double partial[MAX_BLOCKS];
};

// The single thread that finishes a squared-norm reduction: total_norm = sqrt(sum of the n partials in order), and the
// step bump of the Adam update that follows.
__device__ __forceinline__ void finish_norm(OptWs* ws, const double* partial, unsigned int n, int bump_step) {
    double acc = 0.0;
    for (unsigned int k = 0; k < n; ++k) acc += partial[k];
    ws->total_norm = (float)sqrt(acc);
    if (bump_step) ws->step += 1;
}

struct AdamCoef {
    float neg_step, bc2_sqrt, w1, b2, a2, eps, coef, cv, wd;
    int clip_mode;
};

// t = step count AFTER the bump (>= 1).  clip_mode 1: clip_grad_norm_ (coef from the global norm), 2: clip_grad_value_.
__device__ __forceinline__ AdamCoef adam_coef(int t, double lr, double beta1, double beta2, double eps, double weight_decay,
                                              int clip_mode, double clip_value, float total_norm) {
    AdamCoef c;
    const double bc1 = 1.0 - pow(beta1, (double)t);
    const double bc2 = 1.0 - pow(beta2, (double)t);
    c.neg_step = (float)(-(lr / bc1));
    c.bc2_sqrt = (float)sqrt(bc2);
    c.w1 = (float)(1.0 - beta1);
    c.b2 = (float)beta2;
    c.a2 = (float)(1.0 - beta2);
    c.eps = (float)eps;
    c.coef = 1.0f;
    if (clip_mode == 1) c.coef = fminf((float)clip_value / (total_norm + 1e-6f), 1.0f);      // clip_grad_norm_
    c.cv = (float)clip_value;
    c.wd = (float)weight_decay;
    c.clip_mode = clip_mode;
    return c;
}

__device__ __forceinline__ void adam_apply(const AdamCoef& c, float g, float& pi, float& mi, float& vi) {
    if (c.clip_mode == 1) g = __fmul_rn(g, c.coef);
    else if (c.clip_mode == 2) g = fminf(fmaxf(g, -c.cv), c.cv);
    if (c.wd != 0.0f) g = __fadd_rn(g, __fmul_rn(c.wd, pi));
    mi = fmaf(c.w1, __fsub_rn(g, mi), mi);                                   // exp_avg.lerp_(grad, 1-beta1)
    vi = __fadd_rn(__fmul_rn(vi, c.b2), __fmul_rn(__fmul_rn(c.a2, g), g));   // mul_(beta2).addcmul_(g, g, 1-beta2)
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vi), c.bc2_sqrt), c.eps);
    pi = __fadd_rn(pi, __fdiv_rn(__fmul_rn(c.neg_step, mi), denom));         // addcdiv_(exp_avg, denom, -step_size)
}

}  // namespace optim_dev
