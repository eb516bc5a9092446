// DQN pieces around the shared MLP forward / backward / optimiser kernels (surreal/learner/dqn.py, agent/q_agent.py,
// model/q_net.py): the epsilon-greedy act over the dueling combine, the TD target / Huber loss / dueling backward of one
// update, and the hard target copy counted in samples.
#include "common.cuh"
#include <stddef.h>

namespace {

constexpr int QT = 256;
constexpr int QSTATS = 5;              // partial sums per block: loss, |td|, q, w, bad rows

struct DqnWs {
    unsigned int counter;
    int bad_action;                    // 1 when a batch action is not an integer in [0, n_actions)
    double partial[1];                 // [blocks][QSTATS]
};

// PiecewiseSchedule.value(t) (utils/schedule.py:34-73): sched = [t_0 .. t_{P-1} | v_0 .. v_{P-1} | outside].
// LinearSchedule(T, final, 1.0) is the two-point schedule [(0, 1), (T, final)] with outside value `final`: the same
// double arithmetic as its min(t / T, 1) form.
__device__ __forceinline__ double schedule_value(const double* __restrict__ sched, int P, long long t) {
    const double td = (double)t;
    for (int k = 0; k + 1 < P; ++k) {
        const double lt = sched[k], rt = sched[k + 1];
        if (lt <= td && td < rt) {
            const double l = sched[P + k], r = sched[P + k + 1];
            return l + (td - lt) / (rt - lt) * (r - l);
        }
    }
    return sched[2 * P];
}

// Q row j of the dueling head: (A_j - mean A) + V, or A_j without a value tower (q_net.py:44-59).
__device__ __forceinline__ float q_of(float a, float mean, const float* v) {
    return v != nullptr ? __fadd_rn(__fsub_rn(a, mean), *v) : a;
}

__device__ __forceinline__ float row_mean(const float* __restrict__ a, int n) {
    float s = 0.0f;
    for (int j = 0; j < n; ++j) s = __fadd_rn(s, a[j]);
    return __fdiv_rn(s, (float)n);
}

// argmax_j Q_j of one row, the first index among ties (torch.max(dim))
__device__ __forceinline__ int row_argmax(const float* __restrict__ a, const float* v, int n, float& best) {
    const float m = v != nullptr ? row_mean(a, n) : 0.0f;
    int bi = 0;
    best = q_of(a[0], m, v);
    for (int j = 1; j < n; ++j) {
        const float q = q_of(a[j], m, v);
        if (q > best) { best = q; bi = j; }
    }
    return bi;
}

// One warp per actor: dueling combine, argmax, epsilon-greedy (q_agent.py:35-53).  Philox keyed (seed, *act_counter,
// actor): word x decides (u = x / 2^32 < eps explores), word y draws the uniform action floor(y * n / 2^32).
__global__ void __launch_bounds__(QT) dqn_act_kernel(const float* __restrict__ adv, long long lda,
                                                     const float* __restrict__ value, long long ldv, int N, int n,
                                                     const double* __restrict__ sched, int P, double fixed_eps,
                                                     unsigned long long seed, const long long* __restrict__ act_counter,
                                                     float* __restrict__ action, float* __restrict__ one_hot,
                                                     long long ldo, long long* __restrict__ action_i64) {
    const int lane = threadIdx.x & 31;
    const int i = (int)(((long long)blockIdx.x * QT + threadIdx.x) >> 5);
    if (i >= N) return;
    const float* a = adv + (long long)i * lda;
    const float* v = value != nullptr ? value + (long long)i * ldv : nullptr;
    float m = 0.0f;
    if (v != nullptr) {                                   // lane-strided partial sums, then a fixed xor tree
        float s = 0.0f;
        for (int j = lane; j < n; j += 32) s = __fadd_rn(s, a[j]);
        s = warp_sum(s);
        m = __fdiv_rn(s, (float)n);
    }
    float best = -INFINITY;
    int bi = n;
    for (int j = lane; j < n; j += 32) {
        const float q = q_of(a[j], m, v);
        if (q > best || bi == n) { best = q; bi = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (oi < n && (bi == n || ob > best || (ob == best && oi < bi))) { best = ob; bi = oi; }
    }
    const long long t = act_counter != nullptr ? *act_counter : 0;
    const double eps = sched != nullptr ? schedule_value(sched, P, t) : fixed_eps;
    const Philox4 r = philox4x32_10(seed, (unsigned long long)t, (unsigned long long)i);
    const double u = (double)r.x * 2.3283064365386963e-10;
    const int act = (u < eps) ? (int)(((unsigned long long)r.y * (unsigned long long)n) >> 32) : bi;
    if (lane == 0) {
        action[i] = (float)act;
        if (action_i64 != nullptr) action_i64[i] = act;
    }
    if (one_hot != nullptr)
        for (int j = lane; j < (int)ldo; j += 32) one_hot[(long long)i * ldo + j] = (j == act) ? 1.0f : 0.0f;
}

// One update's TD part (dqn.py:44-69), one thread per batch row: q(s)[a], the target column at s' (double Q: the online
// argmax at s' picks it; else the target max), y = r + gamma (1 - done) q', td = q - y, Huber (delta 1) weighted by w,
// the gradient rows of both towers' outputs (dQ_a = w clamp(td, -1, 1) / B; dueling: dA_j = dQ_j - mean_k dQ_k,
// dV = sum_k dQ_k), the priorities |td| + eps, and the statistics as fixed-order sums of per-block partials.
__global__ void __launch_bounds__(QT) dqn_td_kernel(const float* __restrict__ qa, long long ldqa, const float* qv, long long ldqv,
                                                    const float* __restrict__ ta, long long ldta, const float* tv, long long ldtv,
                                                    const float* oa, long long ldoa, const float* ov, long long ldov,
                                                    const float* __restrict__ actions, const float* __restrict__ rewards,
                                                    const float* __restrict__ dones, const float* __restrict__ weights,
                                                    int B, int n, float gamma, double prio_eps,
                                                    float* __restrict__ da, long long ldda, float* dv, long long lddv,
                                                    float* __restrict__ prio, float* __restrict__ stats, DqnWs* ws) {
    __shared__ double sh[32];
    const int tid = threadIdx.x, b = blockIdx.x * QT + tid;
    double s_loss = 0.0, s_td = 0.0, s_q = 0.0, s_w = 0.0, s_bad = 0.0;
    if (b < B) {
        const float af = actions[b];
        const bool ok = af >= 0.0f && af < (float)n && af == floorf(af);
        const int ai = ok ? (int)af : 0;
        if (!ok) s_bad = 1.0;
        const float* ra = qa + (long long)b * ldqa;
        const float* rv = qv != nullptr ? qv + (long long)b * ldqv : nullptr;
        const float q = q_of(ra[ai], rv != nullptr ? row_mean(ra, n) : 0.0f, rv);
        const float* rta = ta + (long long)b * ldta;
        const float* rtv = tv != nullptr ? tv + (long long)b * ldtv : nullptr;
        float qn;
        if (oa != nullptr) {
            float ob;
            const int k = row_argmax(oa + (long long)b * ldoa, ov != nullptr ? ov + (long long)b * ldov : nullptr, n, ob);
            qn = q_of(rta[k], rtv != nullptr ? row_mean(rta, n) : 0.0f, rtv);
        } else {
            row_argmax(rta, rtv, n, qn);
        }
        const float y = __fadd_rn(rewards[b], __fmul_rn(gamma, __fmul_rn(__fsub_rn(1.0f, dones[b]), qn)));
        const float td = __fsub_rn(q, y);
        const float atd = fabsf(td);
        const float hub = atd < 1.0f ? __fmul_rn(0.5f, __fmul_rn(td, td)) : __fsub_rn(atd, 0.5f);
        const float w = weights != nullptr ? weights[b] : 1.0f;
        const float g = __fdiv_rn(__fmul_rn(w, fminf(fmaxf(td, -1.0f), 1.0f)), (float)B);
        float* rd = da + (long long)b * ldda;
        if (dv != nullptr) {
            const float gm = __fdiv_rn(g, (float)n);
            for (int j = 0; j < (int)ldda; ++j) rd[j] = j < n ? __fsub_rn(j == ai ? g : 0.0f, gm) : 0.0f;
            float* rdv = dv + (long long)b * lddv;
            rdv[0] = g;
            for (int j = 1; j < (int)lddv; ++j) rdv[j] = 0.0f;
        } else {
            for (int j = 0; j < (int)ldda; ++j) rd[j] = j == ai ? g : 0.0f;
        }
        if (prio != nullptr) prio[b] = (float)((double)atd + prio_eps);
        s_loss = (double)w * (double)hub;
        s_td = (double)atd;
        s_q = (double)q;
        s_w = (double)w;
    }
    double* part = ws->partial + (size_t)blockIdx.x * QSTATS;
    double t;
    t = block_sum(s_loss, sh); if (tid == 0) part[0] = t;
    t = block_sum(s_td, sh);   if (tid == 0) part[1] = t;
    t = block_sum(s_q, sh);    if (tid == 0) part[2] = t;
    t = block_sum(s_w, sh);    if (tid == 0) part[3] = t;
    t = block_sum(s_bad, sh);  if (tid == 0) part[4] = t;
    if (last_block_ticket(&ws->counter, gridDim.x)) {
        if (tid == 0) {
            double s[QSTATS] = {0, 0, 0, 0, 0};
            for (unsigned int k = 0; k < gridDim.x; ++k)
                for (int c = 0; c < QSTATS; ++c) s[c] += ws->partial[(size_t)k * QSTATS + c];
            stats[SB200_QSTAT_LOSS] = (float)(s[0] / B);
            stats[SB200_QSTAT_TD_ERROR] = (float)(s[1] / B);
            stats[SB200_QSTAT_Q] = (float)(s[2] / B);
            stats[SB200_QSTAT_IS_WEIGHT] = (float)(s[3] / B);
            stats[SB200_QSTAT_BAD_ROWS] = (float)s[4];
            ws->bad_action = s[4] > 0.0 ? 1 : 0;
        }
    }
}

// PeriodicTracker(period).track_increment(incr) on a device counter of samples (dqn.py:84-86): tick adds incr; the copy
// runs when the count crossed a multiple of the period, i.e. floor(c / period) > floor((c - incr) / period).
__global__ void hard_update_samples_tick_kernel(long long* counter, long long incr, const int* __restrict__ stop) {
    if (stop != nullptr && *stop) return;
    *counter += incr;
}

__global__ void __launch_bounds__(QT) hard_update_samples_kernel(float* __restrict__ target, const float* __restrict__ src,
                                                                 long long n, const long long* __restrict__ counter,
                                                                 long long period, long long incr,
                                                                 const int* __restrict__ stop) {
    if (stop != nullptr && *stop) return;
    const long long c = *counter;
    if (c / period <= (c - incr) / period) return;
    for (long long i = (long long)blockIdx.x * QT + threadIdx.x; i < n; i += (long long)gridDim.x * QT) target[i] = src[i];
}

inline int nb(int B) { return (B + QT - 1) / QT; }

int act_launch(const float* adv, int64_t lda, const float* value, int64_t ldv, int N, int n_actions, const double* sched,
               int n_points, double fixed_eps, uint64_t seed, const int64_t* act_counter, float* action, float* one_hot,
               int64_t ldo, int64_t* action_i64, cudaStream_t st) {
    const long long threads = (long long)N * 32;
    dqn_act_kernel<<<(unsigned)((threads + QT - 1) / QT), QT, 0, st>>>(
        adv, lda, value, ldv, N, n_actions, sched, n_points, fixed_eps, (unsigned long long)seed,
        (const long long*)act_counter, action, one_hot, ldo, (long long*)action_i64);
    return sb200_launch_status();
}

bool act_args_ok(const float* adv, int64_t lda, const float* value, int64_t ldv, int N, int n_actions,
                 const double* sched, int n_points, double fixed_eps, float* action, float* one_hot, int64_t ldo) {
    return adv && action && N >= 1 && n_actions >= 1 && n_actions <= SB200_DQN_MAX_ACTIONS && lda >= n_actions &&
           (value == nullptr || ldv >= 1) && (sched == nullptr ? (fixed_eps >= 0.0 && fixed_eps <= 1.0) : n_points >= 1) &&
           (one_hot == nullptr || ldo >= n_actions);
}

}  // namespace

extern "C" size_t sb200_dqn_workspace_bytes(int B) { return sizeof(DqnWs) + (size_t)nb(B) * QSTATS * sizeof(double); }

extern "C" size_t sb200_dqn_bad_action_offset(void) { return offsetof(DqnWs, bad_action); }

extern "C" int sb200_dqn_act_f32(const float* adv, int64_t lda, const float* value, int64_t ldv, int N, int n_actions,
                                 const double* schedule, int n_points, double fixed_eps, uint64_t seed,
                                 const int64_t* act_counter, float* action, float* one_hot, int64_t ldo,
                                 int64_t* action_i64, void* stream) {
    SB200_REQUIRE(act_args_ok(adv, lda, value, ldv, N, n_actions, schedule, n_points, fixed_eps, action, one_hot, ldo));
    return act_launch(adv, lda, value, ldv, N, n_actions, schedule, n_points, fixed_eps, seed, act_counter, action,
                      one_hot, ldo, action_i64, (cudaStream_t)stream);
}

extern "C" int sb200_dqn_act_host_f32(const sb200_mlp* adv_net, const sb200_mlp* value_net, const float* obs_host,
                                      float* obs_dev, int N, float* adv_dev, float* value_dev, const double* schedule,
                                      int n_points, double fixed_eps, uint64_t seed, const int64_t* act_counter,
                                      float* action_dev, int64_t* action_i64_dev, int64_t* action_host, void* stream) {
    SB200_REQUIRE(adv_net != nullptr && obs_dev != nullptr && action_i64_dev != nullptr && action_host != nullptr);
    SB200_REQUIRE((value_net == nullptr) == (value_dev == nullptr));
    const int D = adv_net->dims[0], n = adv_net->dims[adv_net->n_layers];
    SB200_REQUIRE(value_net == nullptr || (value_net->dims[0] == D && value_net->dims[value_net->n_layers] == 1));
    SB200_REQUIRE(act_args_ok(adv_dev, n, value_dev, 1, N, n, schedule, n_points, fixed_eps, action_dev, nullptr, 0));
    cudaStream_t st = (cudaStream_t)stream;
    if (obs_host != nullptr)
        SB200_CUDA(cudaMemcpyAsync(obs_dev, obs_host, (size_t)N * D * sizeof(float), cudaMemcpyHostToDevice, st));
    const sb200_zfilter nozf = {nullptr, 1e-5f};
    const sb200_rows in = {obs_dev, nullptr, D, N, 0, nullptr, 0, nullptr, 0};
    const sb200_mlp* nets[2] = {adv_net, value_net};
    float* outs[2] = {adv_dev, value_dev};
    for (int k = 0; k < 2; ++k) {
        if (nets[k] == nullptr) continue;
        float* save[SB200_MAX_LAYERS] = {nullptr, nullptr, nullptr, nullptr};
        int64_t lds[SB200_MAX_LAYERS] = {0, 0, 0, 0};
        save[nets[k]->n_layers - 1] = outs[k];
        lds[nets[k]->n_layers - 1] = k == 0 ? n : 1;
        const int rc = sb200_mlp_forward_f32(nets[k], &nozf, &in, save, lds, stream);
        if (rc != SB200_OK) return rc;
    }
    const int rc = act_launch(adv_dev, n, value_dev, 1, N, n, schedule, n_points, fixed_eps, seed, act_counter,
                              action_dev, nullptr, 0, action_i64_dev, st);
    if (rc != SB200_OK) return rc;
    SB200_CUDA(cudaMemcpyAsync(action_host, action_i64_dev, (size_t)N * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    SB200_CUDA(cudaStreamSynchronize(st));
    return SB200_OK;
}

extern "C" int sb200_dqn_td_f32(const float* q_a, int64_t ld_qa, const float* q_v, int64_t ld_qv, const float* t_a,
                                int64_t ld_ta, const float* t_v, int64_t ld_tv, const float* o_a, int64_t ld_oa,
                                const float* o_v, int64_t ld_ov, const float* actions, const float* rewards,
                                const float* dones, const float* weights, int B, int n_actions, double gamma,
                                double priority_eps, float* d_a, int64_t ld_da, float* d_v, int64_t ld_dv,
                                float* priorities, float* stats, void* workspace, void* stream) {
    SB200_REQUIRE(q_a && t_a && actions && rewards && dones && d_a && stats && workspace && B >= 1);
    SB200_REQUIRE(n_actions >= 1 && n_actions <= SB200_DQN_MAX_ACTIONS && ld_qa >= n_actions && ld_ta >= n_actions &&
                  ld_da >= n_actions);
    const bool dueling = q_v != nullptr;           // one head form for all three evaluations and the gradient
    SB200_REQUIRE((t_v != nullptr) == dueling && (d_v != nullptr) == dueling && (o_v != nullptr) == (dueling && o_a));
    SB200_REQUIRE(o_a == nullptr || ld_oa >= n_actions);
    SB200_REQUIRE(!dueling || (ld_qv >= 1 && ld_tv >= 1 && ld_dv >= 1 && (o_v == nullptr || ld_ov >= 1)));
    dqn_td_kernel<<<nb(B), QT, 0, (cudaStream_t)stream>>>(q_a, ld_qa, q_v, ld_qv, t_a, ld_ta, t_v, ld_tv, o_a, ld_oa, o_v,
                                                         ld_ov, actions, rewards, dones, weights, B, n_actions,
                                                         (float)gamma, priority_eps, d_a, ld_da, d_v, ld_dv, priorities,
                                                         stats, (DqnWs*)workspace);
    return sb200_launch_status();
}

extern "C" int sb200_hard_update_samples_f32(float* target, const float* src, int64_t n, int64_t* counter, int64_t period,
                                             int64_t incr, int tick, const int* stop_flag, void* stream) {
    SB200_REQUIRE(target && src && counter && n >= 1 && period >= 1 && incr >= 0);
    cudaStream_t st = (cudaStream_t)stream;
    if (tick) hard_update_samples_tick_kernel<<<1, 1, 0, st>>>((long long*)counter, incr, stop_flag);
    long long blocks = (n + 4 * QT - 1) / (4 * QT);
    if (blocks > 264) blocks = 264;
    hard_update_samples_kernel<<<(unsigned)blocks, QT, 0, st>>>(target, src, n, (const long long*)counter, period, incr,
                                                                 stop_flag);
    return sb200_launch_status(tick ? 2 : 1);
}
