// Categorical policy of PPO for discrete action spaces: sampling, pd rows, the clip / adapt losses with their gradient
// w.r.t. the logits, the KL early-stop test and the closing statistics (semantics: tests/cat_ref.py).
//
// pd row of a batch row = [p_0 .. p_{K-1} | log p_0 .. log p_{K-1}] (2K floats, the window records' [2A] width with
// A = K), from a max-subtracted log-softmax of the K logits; actions are one-hot rows [K].  One warp per row, lanes
// striding over K.  The loss / KL / statistics kernels take LT rows per block (eight warps of 32 rows each), so that
// they share the Gaussian kernels' workspace (sb200_ppo_loss_workspace_bytes) and its fixed-order block partials.
#include "common.cuh"
#include "ppo_loss_dev.cuh"
#include "rollout_dev.cuh"
#include <math.h>

namespace {

using ppo_dev::LossWs;
using ppo_dev::LT;
using ppo_dev::put_partial;
using ppo_dev::grid_sums;
constexpr int WARPS = LT / 32;
constexpr int ROWS_PER_WARP = LT / WARPS;

// max-subtracted log-softmax of one row, on every lane: log p_j = (l_j - m) - log_s, p_j = exp(l_j - m) / s
struct RowSoftmax {
    float m, s, log_s;
    __device__ __forceinline__ float logp(float l) const { return (l - m) - log_s; }
    __device__ __forceinline__ float p(float l) const { return expf(l - m) / s; }
};

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ RowSoftmax row_softmax(const float* __restrict__ l, int K, int lane) {
    float m = -INFINITY;
    for (int j = lane; j < K; j += 32) m = fmaxf(m, l[j]);
    m = warp_max(m);
    float s = 0.0f;
    for (int j = lane; j < K; j += 32) s += expf(l[j] - m);
    s = warp_sum(s);
    RowSoftmax r = {m, s, logf(s)};
    return r;
}

// argmax of a row, the lowest index among ties (NaN entries never win)
__device__ __forceinline__ int row_argmax(const float* __restrict__ l, int K, int lane) {
    float best = -INFINITY;
    int bi = K;
    for (int j = lane; j < K; j += 32)
        if (l[j] > best || (bi == K && l[j] == best)) { best = l[j]; bi = j; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    return bi < K ? bi : 0;
}

// The uniform of actor i's draw: the first word of Philox4x32-10 keyed exactly as ppo_sample keys its normals
// (action_noise4: seed, step counter, actor << 16), as u = (x >> 8) * 2^-24, exact in fp32 and in [0, 1).
__device__ __forceinline__ float cat_uniform(unsigned long long seed, unsigned long long ctr, unsigned long long actor) {
    const Philox4 r = philox4x32_10(seed, ctr, actor << 16);
    return (float)(r.x >> 8) * 5.9604644775390625e-8f;
}

// Inverse CDF: the first j with u < c_j, c_j the fp32 running sum of p_0..p_j in index order (a warp scan per chunk of
// 32, carried from chunk to chunk), or K - 1 when u is not below c_{K-1}.
__device__ __forceinline__ int row_inverse_cdf(const float* __restrict__ l, const RowSoftmax& sm, int K, float u, int lane) {
    float carry = 0.0f;
    for (int j0 = 0; j0 < K; j0 += 32) {
        const int j = j0 + lane;
        float c = (j < K) ? sm.p(l[j]) : 0.0f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float t = __shfl_up_sync(0xffffffffu, c, o);
            if (lane >= o) c += t;
        }
        c += carry;
        const unsigned hit = __ballot_sync(0xffffffffu, j < K && u < c);
        if (hit != 0u) return j0 + __ffs(hit) - 1;
        carry = __shfl_sync(0xffffffffu, c, 31);
    }
    return K - 1;
}

// logits -> pd rows, one-hot actions, optional int64 indices; the window staging of this step and the fused slot
// assignment as in ppo_sample_kernel (rollout.cu).
__global__ void __launch_bounds__(LT) cat_sample_kernel(const float* __restrict__ logits, long long ldl, int N, int K,
                                                        int deterministic, unsigned long long seed,
                                                        const unsigned long long* step_ctr, float* __restrict__ action,
                                                        float* __restrict__ pd, long long* __restrict__ index,
                                                        const int* __restrict__ stage_pos, float* __restrict__ stage_act,
                                                        float* __restrict__ stage_pd, int n_step, FifoState* fifo,
                                                        int* __restrict__ dest, unsigned long long* step_ctr_mut) {
    const int lane = threadIdx.x & 31;
    const int i = blockIdx.x * WARPS + (threadIdx.x >> 5);
    if (i < N) {
        const float* l = logits + (long long)i * ldl;
        const RowSoftmax sm = row_softmax(l, K, lane);
        int a;
        if (deterministic) {
            a = row_argmax(l, K, lane);
        } else {
            const unsigned long long ctr = (step_ctr != nullptr) ? *step_ctr : 0ull;
            a = row_inverse_cdf(l, sm, K, cat_uniform(seed, ctr, (unsigned long long)i), lane);
        }
        const int p = (stage_pos != nullptr) ? stage_pos[i] : 0;
        float* pr = pd + (long long)i * 2 * K;
        float* ar = action + (long long)i * K;
        float* spr = (stage_pd != nullptr) ? stage_pd + ((long long)i * n_step + p) * 2 * K : nullptr;
        float* sar = (stage_act != nullptr) ? stage_act + ((long long)i * n_step + p) * K : nullptr;
        for (int j = lane; j < K; j += 32) {
            const float pj = sm.p(l[j]), lj = sm.logp(l[j]), oh = (j == a) ? 1.0f : 0.0f;
            pr[j] = pj;
            pr[K + j] = lj;
            ar[j] = oh;
            if (spr != nullptr) {
                spr[j] = pj;
                spr[K + j] = lj;
                sar[j] = oh;
            }
        }
        if (index != nullptr && lane == 0) index[i] = a;
    }
    if (fifo != nullptr) {
        // block 0 assigns the slots of the windows this step completes while the others sample; the LAST block to
        // finish advances the shared step counter, after every block has read it (as ppo_sample_kernel)
        if (blockIdx.x == 0) assign_window_slots(N, n_step, stage_pos, dest, fifo);
        if (last_block_ticket(fifo_ticket(fifo), gridDim.x) && threadIdx.x == 0 && step_ctr_mut != nullptr)
            *step_ctr_mut += 1ull;
    }
}

__global__ void __launch_bounds__(LT) cat_make_pd_kernel(const float* __restrict__ logits, long long ldl, int B, int K,
                                                         float* __restrict__ pd, long long ldp) {
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.x * WARPS + (threadIdx.x >> 5);
    if (b >= B) return;
    const float* l = logits + (long long)b * ldl;
    const RowSoftmax sm = row_softmax(l, K, lane);
    float* pr = pd + (long long)b * ldp;
    for (int j = lane; j < K; j += 32) {
        pr[j] = sm.p(l[j]);
        pr[K + j] = sm.logp(l[j]);
    }
}

// Rows [row0, row0 + 32) of warp `w` of this block: each row's per-row values are summed into `acc` (lane 0) in row
// order; the caller reduces the warps' sums in warp order.
__device__ __forceinline__ int warp_row0(int w) { return blockIdx.x * LT + w * ROWS_PER_WARP; }

// A warp's per-row sums are the same on every lane: lane 0 alone brings them into a block partial (put_partial).
__device__ __forceinline__ double lane0(double v) { return (threadIdx.x & 31) == 0 ? v : 0.0; }

// mode 0: clip (hyper[0] = clip_epsilon)   mode 1: adapt (hyper[1] = beta; ws->kl_mean from cat_kl_kernel(ref, learn))
__global__ void __launch_bounds__(LT) cat_policy_loss_kernel(int mode, const float* __restrict__ logits, long long ldl,
                                                             const float* __restrict__ actions, long long lda,
                                                             const float* __restrict__ adv,
                                                             const float* __restrict__ behave, long long ldb,
                                                             const float* __restrict__ ref, long long ldr, int B, int K,
                                                             const double* __restrict__ hyper, double eta,
                                                             double kl_target, float* __restrict__ dlogits,
                                                             long long ldd, float* __restrict__ stats, LossWs* ws,
                                                             const int* __restrict__ stop) {
    if (stop != nullptr && *stop) return;
    __shared__ double sh[32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const double invB = 1.0 / (double)B;
    const double kl_mean = ws->kl_mean;
    const float c_kl = (mode == 1) ? ppo_dev::adapt_ckl(kl_mean, invB, hyper, eta, kl_target) : 0.0f;
    double s_surr = 0.0, s_loss = 0.0, s_ent = 0.0;
    for (int r = 0; r < ROWS_PER_WARP; ++r) {
        const int b = warp_row0(w) + r;
        if (b >= B) break;
        const float* l = logits + (long long)b * ldl;
        const float* a = actions + (long long)b * lda;
        const float* bp = behave + (long long)b * ldb;
        const float* rp = ref + (long long)b * ldr;
        const RowSoftmax sm = row_softmax(l, K, lane);
        float pa = 0.0f, pb = 0.0f, ent = 0.0f;
        for (int j = lane; j < K; j += 32) {
            const float pj = sm.p(l[j]);
            pa += a[j] * pj;
            pb += a[j] * bp[j];
            if (pj > 0.0f) ent -= pj * sm.logp(l[j]);
        }
        pa = warp_sum(pa);
        pb = warp_sum(pb);
        ent = warp_sum(ent);
        const ppo_dev::Surrogate o = ppo_dev::surrogate(mode, pa, pb, adv[b], invB, hyper);
        // d/dl_j: g_ll * (a_j - p_j) through log p_a, c_kl * (p_j - r_j) through KL(ref || learn)
        float* dr = dlogits + (long long)b * ldd;
        for (int j = lane; j < K; j += 32) {
            const float pj = sm.p(l[j]);
            float d = o.g_ll * (a[j] - pj);
            if (mode == 1) d += c_kl * (pj - rp[j]);
            dr[j] = d;
        }
        for (int j = K + lane; j < ldd; j += 32) dr[j] = 0.0f;
        s_surr += (double)o.surr;
        s_loss += (double)o.rowloss;
        s_ent += (double)ent;
    }
    put_partial(ws, 3, 0, lane0(s_surr), sh);
    put_partial(ws, 3, 1, lane0(s_loss), sh);
    put_partial(ws, 3, 2, lane0(s_ent), sh);
    if (last_block_ticket(&ws->counter, gridDim.x) && threadIdx.x == 0) {
        double s[3];
        grid_sums(ws, 3, 0, s);
        for (int q = 0; q < 2; ++q) ppo_dev::loss_stats(mode, q, s[q], invB, hyper, eta, kl_target, kl_mean, stats);
        stats[SB200_STAT_ENTROPY] = (float)(s[2] * invB);
    }
}

// KL(p0 || q) = sum_j p0_j (log p0_j - log q_j) of a pd row p0 against a pd row (q_is_pd) or the softmax of logits
__device__ __forceinline__ float row_cat_kl(const float* __restrict__ p0, const float* __restrict__ q, bool q_is_pd, int K,
                                            int lane) {
    RowSoftmax sm = {0.0f, 1.0f, 0.0f};
    if (!q_is_pd) sm = row_softmax(q, K, lane);
    float kl = 0.0f;
    for (int j = lane; j < K; j += 32) {
        const float lq = q_is_pd ? q[K + j] : sm.logp(q[j]);
        if (p0[j] > 0.0f) kl += p0[j] * (p0[K + j] - lq);
    }
    return warp_sum(kl);
}

__global__ void __launch_bounds__(LT) cat_kl_kernel(const float* __restrict__ p0, long long ld0,
                                                    const float* __restrict__ logits, long long ldl, int B, int K,
                                                    float* __restrict__ stats, int slot, double stop_threshold,
                                                    int* __restrict__ stop, LossWs* ws) {
    if (stop != nullptr && *stop) return;
    __shared__ double sh[32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    double acc = 0.0;
    for (int r = 0; r < ROWS_PER_WARP; ++r) {
        const int b = warp_row0(w) + r;
        if (b >= B) break;
        acc += (double)row_cat_kl(p0 + (long long)b * ld0, logits + (long long)b * ldl, false, K, lane);
    }
    put_partial(ws, 1, 0, lane0(acc), sh);
    if (last_block_ticket(&ws->counter, gridDim.x) && threadIdx.x == 0) {
        double s[1];
        grid_sums(ws, 1, 0, s);
        ppo_dev::kl_publish((float)(s[0] / (double)B), ws, stats, slot, stop_threshold, stop, 0);
    }
}

// end-of-learn reporting (ppo.py:568-575) with the categorical likelihoods; _avg_log_sig has no counterpart
__global__ void __launch_bounds__(LT) cat_final_stats_kernel(const float* __restrict__ logits, long long ldl,
                                                             const float* __restrict__ actions, long long lda,
                                                             const float* __restrict__ behave, long long ldb,
                                                             const float* __restrict__ ref, long long ldr, int B, int K,
                                                             float* __restrict__ stats, LossWs* ws) {
    __shared__ double sh[32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    double lb = 0.0, isw = 0.0, kd = 0.0;
    for (int r = 0; r < ROWS_PER_WARP; ++r) {
        const int b = warp_row0(w) + r;
        if (b >= B) break;
        const float* l = logits + (long long)b * ldl;
        const float* a = actions + (long long)b * lda;
        const float* bp = behave + (long long)b * ldb;
        const RowSoftmax sm = row_softmax(l, K, lane);
        float pa = 0.0f, pb = 0.0f;
        for (int j = lane; j < K; j += 32) {
            pa += a[j] * sm.p(l[j]);
            pb += a[j] * bp[j];
        }
        pa = warp_sum(pa);
        pb = warp_sum(pb);
        const float Lb = fmaxf(pb, 1e-5f), Lc = fmaxf(pa, 1e-5f);
        lb += (double)Lb;
        isw += (double)(Lc / (Lb + 1e-4f));
        kd += (double)row_cat_kl(ref + (long long)b * ldr, bp, true, K, lane);
    }
    put_partial(ws, 3, 0, lane0(lb), sh);
    put_partial(ws, 3, 1, lane0(isw), sh);
    put_partial(ws, 3, 2, lane0(kd), sh);
    if (last_block_ticket(&ws->counter, gridDim.x) && threadIdx.x == 0) {
        double s[3];
        grid_sums(ws, 3, 0, s);
        ppo_dev::closing_stats(s, B, stats);
    }
}

inline unsigned row_blocks(int B) { return (unsigned)((B + LT - 1) / LT); }
inline unsigned warp_blocks(int N) { return (unsigned)((N + WARPS - 1) / WARPS); }
inline bool k_ok(int K) { return K >= 2 && K <= SB200_PPO_CAT_MAX_K; }

}  // namespace

extern "C" int sb200_ppo_cat_sample_f32(const float* logits, int64_t ldl, int N, int K, int deterministic, uint64_t seed,
                                        uint64_t* step_counter, float* action, float* pd, int64_t* index,
                                        const sb200_windows* stage, int assign_slots, void* stream) {
    SB200_REQUIRE(logits && action && pd && N >= 1 && k_ok(K) && ldl >= K);
    SB200_REQUIRE(stage == nullptr || (windows_ok(stage) && stage->N == N && stage->A == K));
    // the fused slot assignment advances the staging's step counter, which must be the one the draws are keyed by
    SB200_REQUIRE(!assign_slots || (stage != nullptr && step_counter != nullptr && step_counter == stage->step_counter));
    cat_sample_kernel<<<warp_blocks(N), LT, 0, (cudaStream_t)stream>>>(
        logits, ldl, N, K, deterministic, (unsigned long long)seed, (const unsigned long long*)step_counter, action, pd,
        (long long*)index, stage ? stage->stage_pos : nullptr, stage ? stage->stage_act : nullptr,
        stage ? stage->stage_pd : nullptr, stage ? stage->n_step : 1, assign_slots ? (FifoState*)stage->fifo_state : nullptr,
        assign_slots ? stage->dest : nullptr, assign_slots ? (unsigned long long*)step_counter : nullptr);
    return sb200_launch_status();
}

extern "C" int sb200_ppo_cat_make_pd_f32(const float* logits, int64_t ldl, int B, int K, float* pd, int64_t ldp,
                                         void* stream) {
    SB200_REQUIRE(logits && pd && B >= 1 && k_ok(K) && ldl >= K && ldp >= 2 * K);
    cat_make_pd_kernel<<<warp_blocks(B), LT, 0, (cudaStream_t)stream>>>(logits, ldl, B, K, pd, ldp);
    return sb200_launch_status();
}

extern "C" int sb200_ppo_cat_policy_loss_f32(int mode, const float* logits, int64_t ldl, const float* actions, int64_t lda,
                                             const float* adv, const float* behave_pd, int64_t ldb, const float* ref_pd,
                                             int64_t ldr, int B, int K, const double* hyper, double eta, double kl_target,
                                             float* dlogits, int64_t ldd, float* stats, void* workspace,
                                             const int* stop_flag, void* stream) {
    SB200_REQUIRE(mode == 0 || mode == 1);
    SB200_REQUIRE(logits && actions && adv && behave_pd && hyper && dlogits && stats && workspace);
    SB200_REQUIRE(mode == 0 || ref_pd != nullptr);
    SB200_REQUIRE(B >= 1 && k_ok(K) && ldl >= K && lda >= K && ldb >= 2 * K && ldd >= K);
    if (ref_pd == nullptr) { ref_pd = behave_pd; ldr = ldb; }
    SB200_REQUIRE(ldr >= 2 * K);
    cat_policy_loss_kernel<<<row_blocks(B), LT, 0, (cudaStream_t)stream>>>(
        mode, logits, ldl, actions, lda, adv, behave_pd, ldb, ref_pd, ldr, B, K, hyper, eta, kl_target, dlogits, ldd, stats,
        (LossWs*)workspace, stop_flag);
    return sb200_launch_status();
}

extern "C" int sb200_ppo_cat_kl_f32(const float* p0, int64_t ld0, const float* logits, int64_t ldl, int B, int K,
                                    float* stats, int stat_slot, double stop_threshold, int* stop_flag, void* workspace,
                                    void* stream) {
    SB200_REQUIRE(p0 && logits && workspace && B >= 1 && k_ok(K) && ld0 >= 2 * K && ldl >= K);
    SB200_REQUIRE(stat_slot < SB200_STAT_COUNT);
    cat_kl_kernel<<<row_blocks(B), LT, 0, (cudaStream_t)stream>>>(p0, ld0, logits, ldl, B, K, stats, stat_slot,
                                                                 stop_threshold, stop_flag, (LossWs*)workspace);
    return sb200_launch_status();
}

extern "C" int sb200_ppo_cat_final_stats_f32(const float* logits, int64_t ldl, const float* actions, int64_t lda,
                                             const float* behave_pd, int64_t ldb, const float* ref_pd, int64_t ldr, int B,
                                             int K, float* stats, void* workspace, void* stream) {
    SB200_REQUIRE(logits && actions && behave_pd && ref_pd && stats && workspace);
    SB200_REQUIRE(B >= 1 && k_ok(K) && ldl >= K && lda >= K && ldb >= 2 * K && ldr >= 2 * K);
    cat_final_stats_kernel<<<row_blocks(B), LT, 0, (cudaStream_t)stream>>>(logits, ldl, actions, lda, behave_pd, ldb,
                                                                          ref_pd, ldr, B, K, stats, (LossWs*)workspace);
    return sb200_launch_status();
}
