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
using ppo_dev::LossWs;
using ppo_dev::put_partial;
using ppo_dev::grid_sums;

__device__ __forceinline__ float row_loglik(const float* a, const float* mu, const float* sg, int A, float c0) {
    // ppo_net.py:39-40:  -0.5*sum(((a-mu)/std)^2) - 0.5*log(2pi)*d - sum(log std)
    float quad = 0.0f, slog = 0.0f;
    for (int j = 0; j < A; ++j) {
        const float z = (a[j] - mu[j]) / sg[j];
        quad += z * z;
        slog += logf(sg[j]);
    }
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

// One batch row of the policy loss and its gradient w.r.t. the pre-tanh head output (dpre_row[0..ldd), zero padded).
// c_kl: adapt mode's ppo_dev::adapt_ckl.
__device__ __forceinline__ ppo_dev::Surrogate policy_row(int mode, const float* mu, const float* act, const float* s_sig,
                                                         const float* bp, const float* rp, float ad, int A, float c0,
                                                         double invB, const double* hyper, float c_kl, float* dpre_row,
                                                         int ldd) {
    const float P = expf(row_loglik(act, mu, s_sig, A, c0));
    const float Pb = expf(row_loglik(act, bp, bp + A, A, c0));
    const ppo_dev::Surrogate o = ppo_dev::surrogate(mode, P, Pb, ad, invB, hyper);
    // gradient w.r.t. the pre-tanh output (mean = tanh(pre))
    for (int j = 0; j < A; ++j) {
        const float z = (act[j] - mu[j]) / s_sig[j];
        float dmu = o.g_ll * z / s_sig[j];
        if (mode == 1) dmu += c_kl * (-(rp[j] - mu[j]) / (s_sig[j] * s_sig[j]));
        dpre_row[j] = dmu * (1.0f - mu[j] * mu[j]);
    }
    for (int j = A; j < ldd; ++j) dpre_row[j] = 0.0f;
    return o;
}

// this row's contribution to d loss / d log_var[j]
__device__ __forceinline__ float policy_dlogvar(int mode, int j, const float* mu, const float* act, const float* s_sig,
                                                const float* rp, float g_ll, float c_kl, int A) {
    const float z = (act[j] - mu[j]) / s_sig[j];
    float dl = g_ll * (z * z - 1.0f);
    if (mode == 1) {
        const float d = rp[j] - mu[j];
        dl += c_kl * (1.0f - (rp[A + j] * rp[A + j] + d * d) / (s_sig[j] * s_sig[j]));
    }
    return dl;
}

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
    const int nslots = 3 + A;                                            // [surr, rowloss, unused] + dlog_var[A]
    for (int j = tid; j < A; j += LT) s_sig[j] = expf(log_var[j]);       // builders.py:127: std = exp(log_var)
    __syncthreads();
    const float c0 = (float)(0.5 * 1.8378770664093453 * (double)A);      // 0.5*log(2*pi)*d
    const double invB = 1.0 / (double)B;
    const float c_kl = (mode == 1) ? ppo_dev::adapt_ckl(ws->kl_mean, invB, hyper, eta, kl_target) : 0.0f;

    float mu[MAX_A], act[MAX_A];
    ppo_dev::Surrogate pr = {0.0f, 0.0f, 0.0f};
    const bool live_row = b < B;
    const float* rp = ref + (long long)b * ldr;
    if (live_row) {
        for (int j = 0; j < A; ++j) {
            mu[j] = mean[(long long)b * ldm + j];
            act[j] = actions[(long long)b * lda + j];
        }
        pr = policy_row(mode, mu, act, s_sig, behave + (long long)b * ldb, rp, adv[b], A, c0, invB, hyper, c_kl,
                        dpre + (long long)b * ldd, (int)ldd);
    }
    put_partial(ws, nslots, 0, live_row ? (double)pr.surr : 0.0, sh);
    put_partial(ws, nslots, 1, live_row ? (double)pr.rowloss : 0.0, sh);
    for (int j = 0; j < A; ++j) {
        float dl = 0.0f;
        if (live_row) dl = policy_dlogvar(mode, j, mu, act, s_sig, rp, pr.g_ll, c_kl, A);
        put_partial(ws, nslots, 3 + j, (double)dl, sh);
    }
    if (last_block_ticket(&ws->counter, gridDim.x)) {
        for (int s = tid; s < nslots; s += LT) {
            if (s == 2) continue;
            double acc[1];
            grid_sums(ws, nslots, s, acc);
            if (s >= 3) dlog_var[s - 3] = (float)acc[0];
            else ppo_dev::loss_stats(mode, s, acc[0], invB, hyper, eta, kl_target, ws->kl_mean, stats);
        }
        if (tid == 0) stats[SB200_STAT_ENTROPY] = ppo_dev::gauss_entropy(s_sig, A);
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
    put_partial(ws, 1, 0, (double)kl, sh);
    // .mean() in fp32; data-parallel (defer): all-reduce ws->kl_mean, then kl_apply
    if (last_block_ticket(&ws->counter, gridDim.x) && tid == 0) {
        double s[1];
        grid_sums(ws, 1, 0, s);
        ppo_dev::kl_publish((float)(s[0] / (double)B), ws, stats, slot, stop_threshold, stop, defer);
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
        const ppo_dev::ValueRow vr = ppo_dev::value_row(v[(long long)b * ldv], ret[b], B);
        d = vr.d;
        r = vr.r;
        dpre[(long long)b * ldd] = vr.dpre;
        for (int j = 1; j < (int)ldd; ++j) dpre[(long long)b * ldd + j] = 0.0f;
    }
    put_partial(ws, 4, 0, d, sh);
    put_partial(ws, 4, 1, d * d, sh);
    put_partial(ws, 4, 2, r, sh);
    put_partial(ws, 4, 3, r * r, sh);
    if (last_block_ticket(&ws->counter, gridDim.x) && tid == 0) {
        double s[4];
        grid_sums(ws, 4, 0, s);
        ppo_dev::value_stats(s, (double)B, stats);
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
        const float Lb = fmaxf(expf(row_loglik(a, bp, bp + A, A, c0)), 1e-5f);
        const float Lc = fmaxf(expf(row_loglik(a, mean + (long long)b * ldm, s_sig, A, c0)), 1e-5f);
        lb = (double)Lb;
        isw = (double)(Lc / (Lb + 1e-4f));
        kd = (double)row_kl(rp, rp + A, bp, bp + A, A);
    }
    put_partial(ws, 3, 0, lb, sh);
    put_partial(ws, 3, 1, isw, sh);
    put_partial(ws, 3, 2, kd, sh);
    if (last_block_ticket(&ws->counter, gridDim.x) && tid == 0) {
        double s[3];
        grid_sums(ws, 3, 0, s);
        ppo_dev::closing_stats(s, B, stats);
        float lv = 0.0f;
        for (int j = 0; j < A; ++j) lv += log_var[j];
        stats[SB200_STAT_LOG_SIG] = lv / (float)A;
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
