// The PPO loss algebra that depends neither on the policy distribution nor on how rows map to threads (ppo.py:194-225
// clip, 250-285 adapt, 311-332 value, 568-575 closing statistics), and the workspace of the launch-chain loss kernels.
// The Gaussian loss kernels (ppo_loss.cu, a thread per row), the categorical ones (ppo_cat.cu, a warp per row) and the
// one-launch learner (epoch2.cu, a warp per row) all take these pieces from here, so that every path evaluates the same
// arithmetic in the same order; each keeps only its likelihoods, their gradients and its row mapping.  A function takes
// a sum and 1/B where its callers multiply them, never a precomputed mean: nvcc contracts a*b + c*d into an FMA, so a
// mean formed first would round differently.
#pragma once
#include "common.cuh"

namespace ppo_dev {

constexpr int MAX_A = 64;
constexpr int LT = 256;      // threads per block of the loss kernels, and batch rows per block (workspace sizing)

// Workspace of the loss / KL / statistics kernels of both policy distributions (sb200_ppo_loss_workspace_bytes).
struct LossWs {
    unsigned int counter;
    unsigned int pad;
    double kl_mean;          // written by the KL kernel, consumed by the adapt loss
    double partial[1];       // [blocks][slots]
};

// This block's sum of v (one value per thread, every thread calls) into slot `slot` of its `nslots` partials.
__device__ __forceinline__ void put_partial(LossWs* ws, int nslots, int slot, double v, double* sh) {
    const double t = block_sum(v, sh);
    if (threadIdx.x == 0) ws->partial[(size_t)blockIdx.x * nslots + slot] = t;
}

// In the last block (last_block_ticket): s[q] = the grid sum of slot `slot + q`, each in block order.  Any thread may sum
// any slots.
template <int N>
__device__ __forceinline__ void grid_sums(const LossWs* ws, int nslots, int slot, double (&s)[N]) {
#pragma unroll
    for (int q = 0; q < N; ++q) s[q] = 0.0;
    for (unsigned int k = 0; k < gridDim.x; ++k)
#pragma unroll
        for (int q = 0; q < N; ++q) s[q] += ws->partial[(size_t)k * nslots + slot + q];
}

// Last block of a KL kernel: mean KL `klm` (the fp32 .mean()) -> ws->kl_mean, stats[slot], the early-stop flag above
// stop_threshold (> 0) and the epoch count (ppo.py:553-557).  defer: data-parallel, leave the local mean for kl_apply.
__device__ __forceinline__ void kl_publish(float klm, LossWs* ws, float* stats, int slot, double stop_threshold, int* stop,
                                           int defer) {
    ws->kl_mean = (double)klm;
    if (defer) return;
    if (stats != nullptr && slot >= 0) stats[slot] = klm;
    if (stop != nullptr && stop_threshold > 0.0 && (double)klm > stop_threshold) *stop = 1;
    if (stats != nullptr && slot == SB200_STAT_KL_POST) stats[SB200_STAT_EPOCHS] += 1.0f;
}

// Surrogate of one batch row from the current and behaviour likelihoods P and Pb (before their 1e-5 clamps) and the
// advantage ad: surr and the loss row for the statistics, and g_ll = d loss / d log P (zero where the clamp binds).
// mode 0: clip (hyper[0] = clip_epsilon)   mode 1: adapt (its KL term enters the gradient through adapt_ckl).
struct Surrogate {
    float surr, rowloss, g_ll;
};
__device__ __forceinline__ Surrogate surrogate(int mode, float P, float Pb, float ad, double invB, const double* hyper) {
    Surrogate o;
    const float Ll = fmaxf(P, 1e-5f);
    const bool live = P >= 1e-5f;                                     // clamp(min) passes grad where x >= min
    const float Lb = fmaxf(Pb, 1e-5f);
    if (mode == 0) {
        const float lo = (float)(1.0 - hyper[0]), hi = (float)(1.0 + hyper[0]);
        const float ratio = Ll / Lb;
        const float cr = fminf(fmaxf(ratio, lo), hi);
        o.surr = -ratio * ad;
        const float cs = -cr * ad;
        o.rowloss = fmaxf(o.surr, cs);
        const float g_ratio = (o.surr >= cs) ? -ad : 0.0f;            // max(1) routes grad to the first max
        o.g_ll = live ? (float)((double)g_ratio * invB) * (P / Lb) : 0.0f;
    } else {
        const float den = fmaxf(Lb, 1e-2f);
        o.surr = -ad * (Ll / den);
        o.rowloss = o.surr;
        o.g_ll = live ? (float)((double)(-ad / den) * invB) * P : 0.0f;
    }
    return o;
}

// Adapt mode: the weight of a row's d KL(ref || current) in the loss gradient, (beta + 2 eta max(0, kl - 2 kl_target)) / B
// with beta = hyper[1] and kl the batch-mean KL.
__device__ __forceinline__ float adapt_ckl(double kl, double invB, const double* hyper, double eta, double kl_target) {
    double ck = hyper[1];
    if (kl - 2.0 * kl_target > 0.0) ck += 2.0 * eta * (kl - 2.0 * kl_target);
    return (float)(ck * invB);
}

// Statistics of policy-loss slot s from its grid sum: slot 0 (surr) -> SURR, and in adapt mode the penalised LOSS and
// KL_PRE = kl; slot 1 (loss rows) -> the clip-mode LOSS.
__device__ __forceinline__ void loss_stats(int mode, int s, double sum, double invB, const double* hyper, double eta,
                                           double kl_target, double kl, float* stats) {
    if (s == 0) stats[SB200_STAT_SURR] = (float)(sum * invB);
    if (s == 1 && mode == 0) stats[SB200_STAT_LOSS] = (float)(sum * invB);
    if (s == 0 && mode == 1) {
        double loss = sum * invB + hyper[1] * kl;
        if (kl - 2.0 * kl_target > 0.0) loss += eta * (kl - 2.0 * kl_target) * (kl - 2.0 * kl_target);
        stats[SB200_STAT_LOSS] = (float)loss;
        stats[SB200_STAT_KL_PRE] = (float)kl;
    }
}

// ENTROPY of the diagonal Gaussian with std s_sig[0..A) (ppo_net.py:72)
__device__ __forceinline__ float gauss_entropy(const float* s_sig, int A) {
    float slog = 0.0f;
    for (int j = 0; j < A; ++j) slog += logf(s_sig[j]);
    return 0.5f * slog + (float)(0.5 * 2.8378770664093453 * (double)A);
}

// One row of the value loss mean((v - ret)^2): dpre = d loss / d v, and d = ret - v, r = ret, whose sums and sums of
// squares are the moments value_stats takes.
struct ValueRow {
    float dpre;
    double d, r;
};
__device__ __forceinline__ ValueRow value_row(float v, float ret, int B) {
    ValueRow o;
    o.dpre = (float)(2.0 * (double)(v - ret) / (double)B);
    o.d = (double)(ret - v);
    o.r = (double)ret;
    return o;
}

// Value statistics (ppo.py:323-331) from s = the grid sums of {d, d^2, r, r^2} over n rows
__device__ __forceinline__ void value_stats(const double* s, double n, float* stats) {
    const double var_d = (s[1] - s[0] * s[0] / n) / (n - 1.0);
    const double var_r = (s[3] - s[2] * s[2] / n) / (n - 1.0);
    stats[SB200_STAT_VAL_LOSS] = (float)(s[1] / n);
    stats[SB200_STAT_EXPLAINED_VAR] = (float)(1.0 - var_d / var_r);
    stats[SB200_STAT_RETURN_MEAN] = (float)(s[2] / n);
    // raw moments as (hi, lo) float pairs: a data-parallel learner averages them over ranks and recomputes the explained
    // variance of the GLOBAL batch (a mean of per-rank ratios is not the ratio of the global moments)
    for (int q = 0; q < 4; ++q) {
        const double m = s[q] / n;
        const float hi = (float)m;
        stats[SB200_STAT_VAL_MOMENTS + 2 * q] = hi;
        stats[SB200_STAT_VAL_MOMENTS + 2 * q + 1] = (float)(m - (double)hi);
    }
}

// Closing statistics (ppo.py:568-575) from s = the grid sums of the clamped behaviour likelihood, the importance weight
// and KL(ref || behave) over B rows
__device__ __forceinline__ void closing_stats(const double* s, int B, float* stats) {
    stats[SB200_STAT_BEHAVE_LIK] = (float)(s[0] / B);
    stats[SB200_STAT_IS_WEIGHT] = (float)(s[1] / B);
    stats[SB200_STAT_REF_BEHAVE_KL] = (float)(s[2] / B);
}

}  // namespace ppo_dev
