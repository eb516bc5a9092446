// Per-row pieces of the PPO losses (ppo.py:194-225 clip, 250-285 adapt; DiagGauss of ppo_net.py:29-72), shared by the
// stand-alone loss kernels (ppo_loss.cu) and the persistent learner kernel (epoch2.cu) so that both evaluate the same
// arithmetic in the same order.
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

__device__ __forceinline__ float row_loglik(const float* a, const float* mu, const float* sg, int A, float c0,
                                            float* quad_out) {
    // ppo_net.py:39-40:  -0.5*sum(((a-mu)/std)^2) - 0.5*log(2pi)*d - sum(log std)
    float quad = 0.0f, slog = 0.0f;
    for (int j = 0; j < A; ++j) {
        const float z = (a[j] - mu[j]) / sg[j];
        quad += z * z;
        slog += logf(sg[j]);
    }
    if (quad_out) *quad_out = quad;
    return -0.5f * quad - c0 - slog;
}

__device__ __forceinline__ float row_kl(const float* m0, const float* s0, const float* m1, const float* s1, int A) {
    // ppo_net.py:61-62: KL(p0 || p1)
    float t1 = 0.0f, t2 = 0.0f;
    for (int j = 0; j < A; ++j) {
        t1 += logf(s1[j] / s0[j]);
        const float d = m0[j] - m1[j];
        t2 += (s0[j] * s0[j] + d * d) / (2.0f * s1[j] * s1[j]);
    }
    return t1 + t2 - 0.5f * (float)A;
}


struct PolicyRow {
    float surr, rowloss, klrow, g_ll, c_kl;
};

// One batch row of the policy loss and its gradient w.r.t. the pre-tanh head output (dpre_row[0..ldd), zero padded).
// mode 0: clip (hyper[0] = clip_epsilon)   mode 1: adapt (hyper[1] = beta; kl_mean = mean KL(ref || current)).
__device__ __forceinline__ PolicyRow policy_row(int mode, const float* mu, const float* act, const float* s_sig,
                                                const float* bp, const float* rp, float ad, int A, float c0, double invB,
                                                const double* hyper, double eta, double kl_target, double kl_mean,
                                                float* dpre_row, int ldd) {
    PolicyRow o = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    const float ll = row_loglik(act, mu, s_sig, A, c0, nullptr);
    const float Pl = expf(ll);
    const float Ll = fmaxf(Pl, 1e-5f);
    const bool live = Pl >= 1e-5f;                                    // clamp(min) passes grad where x >= min
    const float llb = row_loglik(act, bp, bp + A, A, c0, nullptr);
    const float Lb = fmaxf(expf(llb), 1e-5f);
    if (mode == 0) {
        const float lo = (float)(1.0 - hyper[0]), hi = (float)(1.0 + hyper[0]);
        const float ratio = Ll / Lb;
        const float cr = fminf(fmaxf(ratio, lo), hi);
        o.surr = -ratio * ad;
        const float cs = -cr * ad;
        o.rowloss = fmaxf(o.surr, cs);
        const float g_ratio = (o.surr >= cs) ? -ad : 0.0f;            // max(1) routes grad to the first max
        o.g_ll = live ? (float)((double)g_ratio * invB) * (Pl / Lb) : 0.0f;
    } else {
        o.klrow = row_kl(rp, rp + A, mu, s_sig, A);
        const float den = fmaxf(Lb, 1e-2f);
        o.surr = -ad * (Ll / den);
        o.rowloss = o.surr;
        o.g_ll = live ? (float)((double)(-ad / den) * invB) * Pl : 0.0f;
        double ck = hyper[1];
        if (kl_mean - 2.0 * kl_target > 0.0) ck += 2.0 * eta * (kl_mean - 2.0 * kl_target);
        o.c_kl = (float)(ck * invB);
    }
    // gradient w.r.t. the pre-tanh output (mean = tanh(pre))
    for (int j = 0; j < A; ++j) {
        const float z = (act[j] - mu[j]) / s_sig[j];
        float dmu = o.g_ll * z / s_sig[j];
        if (mode == 1) dmu += o.c_kl * (-(rp[j] - mu[j]) / (s_sig[j] * s_sig[j]));
        dpre_row[j] = dmu * (1.0f - mu[j] * mu[j]);
    }
    for (int j = A; j < ldd; ++j) dpre_row[j] = 0.0f;
    return o;
}

// this row's contribution to d loss / d log_var[j]
__device__ __forceinline__ float policy_dlogvar(int mode, int j, const float* mu, const float* act, const float* s_sig,
                                                const float* rp, const PolicyRow& o, int A) {
    const float z = (act[j] - mu[j]) / s_sig[j];
    float dl = o.g_ll * (z * z - 1.0f);
    if (mode == 1) {
        const float d = rp[j] - mu[j];
        dl += o.c_kl * (1.0f - (rp[A + j] * rp[A + j] + d * d) / (s_sig[j] * s_sig[j]));
    }
    return dl;
}

}  // namespace ppo_dev
