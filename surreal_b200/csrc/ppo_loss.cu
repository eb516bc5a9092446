// PPO losses, fused forward + gradient w.r.t. the actor's pre-tanh output and log_var in one pass.
//
// Replaces surreal/learner/ppo.py:194-225 (_clip_loss), 250-285 (_adapt_loss), 311-332 (_value_loss),
// 553-556 (post-epoch KL check), 568-575 (reporting stats) and the DiagGauss math of
// surreal/model/ppo_net.py:29-72, plus torch autograd through them.  One thread per batch row;
// block partials are reduced in fixed order by the last block (deterministic).
//
// stats[] slots (fp32): see SB200_STAT_* in the header.
#include "common.cuh"
#include "ppo_loss_dev.cuh"
#include <math.h>
#include <stddef.h>

namespace {

using ppo_dev::LT;
using ppo_dev::MAX_A;
using ppo_dev::row_loglik;
using ppo_dev::row_kl;
using ppo_dev::LossWs;

// ------------------------------------------------------------------------------------------------
// mode 0: clip   mode 1: adapt (needs ws->kl_mean from kl_kernel(ref, learn))
__global__ void __launch_bounds__(LT) policy_loss_kernel(int mode, const float* __restrict__ mean, long long ldm,
                                                         const float* __restrict__ log_var,
                                                         const float* __restrict__ actions, long long lda,
                                                         const float* __restrict__ adv,
                                                         const float* __restrict__ behave, long long ldb,
                                                         const float* __restrict__ ref, long long ldr, int B, int A,
                                                         const double* __restrict__ hyper, double eta,
                                                         double kl_target, float* __restrict__ dpre, long long ldd,
                                                         float* __restrict__ dlog_var, float* __restrict__ stats,
                                                         LossWs* ws, const int* __restrict__ stop) {
    if (stop != nullptr && *stop) return;
    __shared__ double sh[32];
    __shared__ float s_sig[MAX_A];
    const int tid = threadIdx.x;
    const int b = blockIdx.x * LT + tid;
    const int nslots = 3 + A;
    for (int j = tid; j < A; j += LT) s_sig[j] = expf(log_var[j]);       // builders.py:127: std = exp(log_var)
    __syncthreads();
    const float c0 = (float)(0.5 * 1.8378770664093453 * (double)A);      // 0.5*log(2*pi)*d
    const double invB = 1.0 / (double)B;

    float mu[MAX_A], act[MAX_A];
    ppo_dev::PolicyRow pr = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    const bool live_row = b < B;
    if (live_row) {
        for (int j = 0; j < A; ++j) {
            mu[j] = mean[(long long)b * ldm + j];
            act[j] = actions[(long long)b * lda + j];
        }
        pr = ppo_dev::policy_row(mode, mu, act, s_sig, behave + (long long)b * ldb, ref + (long long)b * ldr, adv[b], A, c0,
                                 invB, hyper, eta, kl_target, ws->kl_mean, dpre + (long long)b * ldd, (int)ldd);
    }
    const float surr = pr.surr, rowloss = pr.rowloss, klrow = pr.klrow;
    // ---- block partials: [surr, rowloss, kl] + dlog_var[A]
    double* part = ws->partial + (size_t)blockIdx.x * nslots;
    double t;
    t = block_sum(live_row ? (double)surr : 0.0, sh);
    if (tid == 0) part[0] = t;
    t = block_sum(live_row ? (double)rowloss : 0.0, sh);
    if (tid == 0) part[1] = t;
    t = block_sum(live_row ? (double)klrow : 0.0, sh);
    if (tid == 0) part[2] = t;
    for (int j = 0; j < A; ++j) {
        float dl = 0.0f;
        if (live_row) dl = ppo_dev::policy_dlogvar(mode, j, mu, act, s_sig, ref + (long long)b * ldr, pr, A);
        t = block_sum((double)dl, sh);
        if (tid == 0) part[3 + j] = t;
    }
    if (last_block_ticket(&ws->counter, gridDim.x)) {
        for (int s = tid; s < nslots; s += LT) {
            double acc = 0.0;
            for (unsigned int k = 0; k < gridDim.x; ++k) acc += ws->partial[(size_t)k * nslots + s];
            if (s >= 3) dlog_var[s - 3] = (float)acc;
            if (s == 0) stats[SB200_STAT_SURR] = (float)(acc * invB);
            if (s == 1 && mode == 0) stats[SB200_STAT_LOSS] = (float)(acc * invB);
            if (s == 2 && mode == 1) stats[SB200_STAT_KL_PRE] = (float)ws->kl_mean;
        }
        if (tid == 0) {
            float slog = 0.0f;
            for (int j = 0; j < A; ++j) slog += logf(s_sig[j]);
            stats[SB200_STAT_ENTROPY] = 0.5f * slog + (float)(0.5 * 2.8378770664093453 * (double)A);   // ppo_net.py:72
            if (mode == 1) {
                double surr_sum = 0.0;
                for (unsigned int k = 0; k < gridDim.x; ++k) surr_sum += ws->partial[(size_t)k * nslots + 0];
                const double kl = ws->kl_mean;
                double loss = surr_sum * invB + hyper[1] * kl;
                if (kl - 2.0 * kl_target > 0.0) loss += eta * (kl - 2.0 * kl_target) * (kl - 2.0 * kl_target);
                stats[SB200_STAT_LOSS] = (float)loss;
            }
        }
    }
}

// mean KL(p0 || cur) with cur = (mean, exp(log_var)); writes ws->kl_mean and stats[slot]; optionally raises
// the early-stop flag when kl > stop_threshold (ppo.py:553-557).
__global__ void __launch_bounds__(LT) kl_kernel(const float* __restrict__ p0, long long ld0,
                                                const float* __restrict__ mean, long long ldm,
                                                const float* __restrict__ log_var, int B, int A,
                                                float* __restrict__ stats, int slot, double stop_threshold,
                                                int* __restrict__ stop, LossWs* ws, int defer) {
    if (stop != nullptr && *stop) return;
    __shared__ double sh[32];
    __shared__ float s_sig[MAX_A];
    const int tid = threadIdx.x, b = blockIdx.x * LT + tid;
    for (int j = tid; j < A; j += LT) s_sig[j] = expf(log_var[j]);
    __syncthreads();
    float kl = 0.0f;
    if (b < B) kl = row_kl(p0 + (long long)b * ld0, p0 + (long long)b * ld0 + A, mean + (long long)b * ldm, s_sig, A);
    const double t = block_sum((double)kl, sh);
    if (tid == 0) ws->partial[blockIdx.x] = t;
    if (last_block_ticket(&ws->counter, gridDim.x)) {
        if (tid == 0) {
            double acc = 0.0;
            for (unsigned int k = 0; k < gridDim.x; ++k) acc += ws->partial[k];
            // .mean() in fp32; data-parallel (defer): all-reduce ws->kl_mean, then kl_apply
            ppo_dev::kl_publish((float)(acc / (double)B), ws, stats, slot, stop_threshold, stop, defer);
        }
    }
}

// second half of kl_kernel for the data-parallel learner (after the KL scalar was averaged over ranks)
__global__ void kl_apply_kernel(LossWs* ws, float* __restrict__ stats, int slot, double stop_threshold,
                                int* __restrict__ stop) {
    if (stop != nullptr && *stop) return;
    ppo_dev::kl_publish((float)ws->kl_mean, ws, stats, slot, stop_threshold, stop, 0);
}

// value loss: mean((v - ret)^2), dv = 2(v-ret)/B, explained variance (ppo.py:323-331)
__global__ void __launch_bounds__(LT) value_loss_kernel(const float* __restrict__ v, long long ldv,
                                                        const float* __restrict__ ret, int B,
                                                        float* __restrict__ dpre, long long ldd,
                                                        float* __restrict__ stats, LossWs* ws) {
    __shared__ double sh[32];
    const int tid = threadIdx.x, b = blockIdx.x * LT + tid;
    double d = 0.0, r = 0.0;
    if (b < B) {
        const float vv = v[(long long)b * ldv], rr = ret[b];
        const float df = vv - rr;
        d = (double)(rr - vv);
        r = (double)rr;
        dpre[(long long)b * ldd] = (float)(2.0 * (double)df / (double)B);
        for (int j = 1; j < (int)ldd; ++j) dpre[(long long)b * ldd + j] = 0.0f;
    }
    double* part = ws->partial + (size_t)blockIdx.x * 4;
    double t;
    t = block_sum(d, sh);       if (tid == 0) part[0] = t;
    t = block_sum(d * d, sh);   if (tid == 0) part[1] = t;
    t = block_sum(r, sh);       if (tid == 0) part[2] = t;
    t = block_sum(r * r, sh);   if (tid == 0) part[3] = t;
    if (last_block_ticket(&ws->counter, gridDim.x)) {
        if (tid == 0) {
            double s[4] = {0, 0, 0, 0};
            for (unsigned int k = 0; k < gridDim.x; ++k)
                for (int q = 0; q < 4; ++q) s[q] += ws->partial[(size_t)k * 4 + q];
            const double n = (double)B;
            const double var_d = (s[1] - s[0] * s[0] / n) / (n - 1.0);
            const double var_r = (s[3] - s[2] * s[2] / n) / (n - 1.0);
            stats[SB200_STAT_VAL_LOSS] = (float)(s[1] / n);
            stats[SB200_STAT_EXPLAINED_VAR] = (float)(1.0 - var_d / var_r);
            stats[SB200_STAT_RETURN_MEAN] = (float)(s[2] / n);
            // raw moments as (hi, lo) float pairs: a data-parallel learner averages them over ranks and recomputes the
            // explained variance of the GLOBAL batch (a mean of per-rank ratios is not the ratio of the global moments)
            for (int q = 0; q < 4; ++q) {
                const double m = s[q] / n;
                const float hi = (float)m;
                stats[SB200_STAT_VAL_MOMENTS + 2 * q] = hi;
                stats[SB200_STAT_VAL_MOMENTS + 2 * q + 1] = (float)(m - (double)hi);
            }
        }
    }
}

// end-of-learn reporting (ppo.py:568-575)
__global__ void __launch_bounds__(LT) final_stats_kernel(const float* __restrict__ mean, long long ldm,
                                                         const float* __restrict__ log_var,
                                                         const float* __restrict__ actions, long long lda,
                                                         const float* __restrict__ behave, long long ldb,
                                                         const float* __restrict__ ref, long long ldr, int B, int A,
                                                         float* __restrict__ stats, LossWs* ws) {
    __shared__ double sh[32];
    __shared__ float s_sig[MAX_A];
    const int tid = threadIdx.x, b = blockIdx.x * LT + tid;
    for (int j = tid; j < A; j += LT) s_sig[j] = expf(log_var[j]);
    __syncthreads();
    const float c0 = (float)(0.5 * 1.8378770664093453 * (double)A);
    double lb = 0.0, isw = 0.0, kd = 0.0;
    if (b < B) {
        const float* a = actions + (long long)b * lda;
        const float* bp = behave + (long long)b * ldb;
        const float* rp = ref + (long long)b * ldr;
        const float Lb = fmaxf(expf(row_loglik(a, bp, bp + A, A, c0, nullptr)), 1e-5f);
        const float Lc = fmaxf(expf(row_loglik(a, mean + (long long)b * ldm, s_sig, A, c0, nullptr)), 1e-5f);
        lb = (double)Lb;
        isw = (double)(Lc / (Lb + 1e-4f));
        kd = (double)row_kl(rp, rp + A, bp, bp + A, A);
    }
    double* part = ws->partial + (size_t)blockIdx.x * 3;
    double t;
    t = block_sum(lb, sh);  if (tid == 0) part[0] = t;
    t = block_sum(isw, sh); if (tid == 0) part[1] = t;
    t = block_sum(kd, sh);  if (tid == 0) part[2] = t;
    if (last_block_ticket(&ws->counter, gridDim.x)) {
        if (tid == 0) {
            double s[3] = {0, 0, 0};
            for (unsigned int k = 0; k < gridDim.x; ++k)
                for (int q = 0; q < 3; ++q) s[q] += ws->partial[(size_t)k * 3 + q];
            stats[SB200_STAT_BEHAVE_LIK] = (float)(s[0] / B);
            stats[SB200_STAT_IS_WEIGHT] = (float)(s[1] / B);
            stats[SB200_STAT_REF_BEHAVE_KL] = (float)(s[2] / B);
            float lv = 0.0f;
            for (int j = 0; j < A; ++j) lv += log_var[j];
            stats[SB200_STAT_LOG_SIG] = lv / (float)A;
        }
    }
}

inline int nblocks(int B) { return (B + LT - 1) / LT; }

}  // namespace

extern "C" size_t sb200_ppo_loss_workspace_bytes(int B, int A) {
    return sizeof(LossWs) + (size_t)nblocks(B) * (size_t)(4 + A) * sizeof(double);
}

extern "C" int sb200_ppo_policy_loss_f32(int mode, const float* mean, int64_t ldm, const float* log_var,
                                         const float* actions, int64_t lda, const float* adv, const float* behave_pd,
                                         int64_t ldb, const float* ref_pd, int64_t ldr, int B, int A,
                                         const double* hyper, double eta, double kl_target, float* dpre, int64_t ldd,
                                         float* dlog_var, float* stats, void* workspace, const int* stop_flag,
                                         void* stream) {
    SB200_REQUIRE(mode == 0 || mode == 1);
    SB200_REQUIRE(mean && log_var && actions && adv && behave_pd && hyper && dpre && dlog_var && stats && workspace);
    SB200_REQUIRE(mode == 0 || ref_pd != nullptr);
    SB200_REQUIRE(B >= 1 && A >= 1 && A <= MAX_A && ldd >= A && ldm >= A && lda >= A && ldb >= 2 * A);
    if (ref_pd == nullptr) { ref_pd = behave_pd; ldr = ldb; }
    policy_loss_kernel<<<nblocks(B), LT, 0, (cudaStream_t)stream>>>(mode, mean, ldm, log_var, actions, lda, adv,
                                                                   behave_pd, ldb, ref_pd, ldr, B, A, hyper, eta,
                                                                   kl_target, dpre, ldd, dlog_var, stats,
                                                                   (LossWs*)workspace, stop_flag);
    return sb200_launch_status();
}

extern "C" int sb200_ppo_kl_f32(const float* p0, int64_t ld0, const float* mean, int64_t ldm, const float* log_var,
                                int B, int A, float* stats, int stat_slot, double stop_threshold, int* stop_flag,
                                int defer, void* workspace, void* stream) {
    SB200_REQUIRE(p0 && mean && log_var && workspace && B >= 1 && A >= 1 && A <= MAX_A);
    SB200_REQUIRE(stat_slot < SB200_STAT_COUNT);
    kl_kernel<<<nblocks(B), LT, 0, (cudaStream_t)stream>>>(p0, ld0, mean, ldm, log_var, B, A, stats, stat_slot,
                                                          stop_threshold, stop_flag, (LossWs*)workspace, defer);
    return sb200_launch_status();
}

extern "C" int sb200_ppo_kl_apply(void* workspace, float* stats, int stat_slot, double stop_threshold, int* stop_flag,
                                  void* stream) {
    SB200_REQUIRE(workspace && stat_slot < SB200_STAT_COUNT);
    kl_apply_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((LossWs*)workspace, stats, stat_slot, stop_threshold, stop_flag);
    return sb200_launch_status();
}

extern "C" size_t sb200_ppo_loss_kl_offset(void) { return offsetof(LossWs, kl_mean); }

extern "C" int sb200_value_loss_f32(const float* values, int64_t ldv, const float* returns, int B, float* dpre,
                                    int64_t ldd, float* stats, void* workspace, void* stream) {
    SB200_REQUIRE(values && returns && dpre && stats && workspace && B >= 1 && ldd >= 1 && ldv >= 1);
    value_loss_kernel<<<nblocks(B), LT, 0, (cudaStream_t)stream>>>(values, ldv, returns, B, dpre, ldd, stats,
                                                                  (LossWs*)workspace);
    return sb200_launch_status();
}

extern "C" int sb200_ppo_final_stats_f32(const float* mean, int64_t ldm, const float* log_var, const float* actions,
                                         int64_t lda, const float* behave_pd, int64_t ldb, const float* ref_pd,
                                         int64_t ldr, int B, int A, float* stats, void* workspace, void* stream) {
    SB200_REQUIRE(mean && log_var && actions && behave_pd && ref_pd && stats && workspace);
    SB200_REQUIRE(B >= 1 && A >= 1 && A <= MAX_A);
    final_stats_kernel<<<nblocks(B), LT, 0, (cudaStream_t)stream>>>(mean, ldm, log_var, actions, lda, behave_pd, ldb,
                                                                   ref_pd, ldr, B, A, stats, (LossWs*)workspace);
    return sb200_launch_status();
}
