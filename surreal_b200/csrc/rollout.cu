// Actor-side kernels of the batched rollout: policy sampling, exploration noise, the per-actor experience
// staging that replaces the Python deques of surreal/env/exp_sender_wrapper.py (windows for PPO, n-step SSAR
// records for DDPG), and the act entries.  The device-resident envs are in env.cu.
//
// All per-actor control state (deque length, episode step, RNG counter) lives in HBM so that a whole
// T-step rollout is a fixed launch sequence (CUDA-graph capturable) with no host round trip.
#include "common.cuh"
#include "rollout_dev.cuh"

namespace {

constexpr int RT = 256;


// ------------------------------------------------------------------------------------------------
// PPOAgent.act after the network (ppo_agent.py:138-149): pd = [mean | exp(log_var)*exp(noise_i)],
// action = clip(eps*std + mean, -1, 1) (or the mean when deterministic).  eps: injected N(0,1) draws
// [N,A] or NULL -> Philox4x32-10 keyed by (seed, step counter, actor).  Also writes the step's action
// and pd rows into the window staging area at the actor's current deque position.
__device__ __forceinline__ void sample_one(const float* __restrict__ mean, long long ldm,
                                           const float* __restrict__ log_var, const float* __restrict__ log_noise,
                                           const float* __restrict__ eps, int N, int A, int deterministic,
                                           unsigned long long seed, const unsigned long long* step_ctr,
                                           float* __restrict__ action, float* __restrict__ pd,
                                           const int* __restrict__ stage_pos, float* __restrict__ stage_act,
                                           float* __restrict__ stage_pd, int n_step, int t, int groups) {
    const int i = t / groups, j0 = (t - i * groups) * 4;
    const float sc = (log_noise != nullptr) ? expf(log_noise[i]) : 1.0f;
    const unsigned long long ctr = (step_ctr != nullptr) ? *step_ctr : 0ull;
    const int p = (stage_pos != nullptr) ? stage_pos[i] : 0;
    float z[4] = {0.f, 0.f, 0.f, 0.f};
    if (!deterministic && eps == nullptr) {
        const float4 n = action_noise4(seed, ctr, i, j0 >> 2);
        z[0] = n.x; z[1] = n.y; z[2] = n.z; z[3] = n.w;
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int j = j0 + c;
        if (j >= A) break;
        const float mu = mean[(long long)i * ldm + j];
        const float sd = ppo_std(log_var[j], sc);
        const float a = ppo_action(mu, sd, (eps != nullptr) ? eps[(long long)i * A + j] : z[c], deterministic);
        action[(long long)i * A + j] = a;
        pd[(long long)i * 2 * A + j] = mu;
        pd[(long long)i * 2 * A + A + j] = sd;
        if (stage_act != nullptr) {
            stage_act[((long long)i * n_step + p) * A + j] = a;
            stage_pd[((long long)i * n_step + p) * 2 * A + j] = mu;
            stage_pd[((long long)i * n_step + p) * 2 * A + A + j] = sd;
        }
    }
}

__global__ void __launch_bounds__(RT) ppo_sample_kernel(const float* __restrict__ mean, long long ldm,
                                                        const float* __restrict__ log_var,
                                                        const float* __restrict__ log_noise,
                                                        const float* __restrict__ eps, int N, int A,
                                                        int deterministic, unsigned long long seed,
                                                        const unsigned long long* step_ctr,
                                                        float* __restrict__ action, float* __restrict__ pd,
                                                        const int* __restrict__ stage_pos,
                                                        float* __restrict__ stage_act,
                                                        float* __restrict__ stage_pd, int n_step,
                                                        FifoState* fifo, int* __restrict__ dest,
                                                        unsigned long long* step_ctr_mut) {
    const int groups = (A + 3) >> 2;                      // one thread per (actor, 4 action dims)
    const int t = blockIdx.x * RT + threadIdx.x;
    if (t < N * groups) sample_one(mean, ldm, log_var, log_noise, eps, N, A, deterministic, seed, step_ctr, action, pd,
                                   stage_pos, stage_act, stage_pd, n_step, t, groups);
    if (fifo != nullptr) {
        // Fused slot assignment for the windows this step completes (it needs only the deque lengths): block 0,
        // while the other blocks sample.  The LAST block to finish advances the shared step counter, after
        // every block has read it.
        if (blockIdx.x == 0) assign_window_slots(N, n_step, stage_pos, dest, fifo);
        if (last_block_ticket(fifo_ticket(fifo), gridDim.x) && threadIdx.x == 0 && step_ctr_mut != nullptr)
            *step_ctr_mut += 1ull;
    }
}

// DDPGAgent.act after the network (ddpg_agent.py:176-183): clip -> + N(0, sigma_i) -> clip.
__global__ void __launch_bounds__(RT) ddpg_noise_kernel(const float* __restrict__ mean, long long ldm,
                                                        const float* __restrict__ sigma,
                                                        const float* __restrict__ unit_noise, int N, int A,
                                                        int deterministic, unsigned long long seed,
                                                        const unsigned long long* __restrict__ step_ctr,
                                                        float* __restrict__ action) {
    const int i = blockIdx.x * RT + threadIdx.x;
    if (i >= N) return;
    const unsigned long long ctr = (step_ctr != nullptr) ? *step_ctr : 0ull;
    const float sg = sigma[i];
    for (int j0 = 0; j0 < A; j0 += 4) {
        float z[4] = {0.f, 0.f, 0.f, 0.f};
        if (!deterministic && unit_noise == nullptr) {
            const float4 n = action_noise4(seed, ctr, i, j0 >> 2);
            z[0] = n.x; z[1] = n.y; z[2] = n.z; z[3] = n.w;
        }
        for (int c = 0; c < 4 && j0 + c < A; ++c) {
            const int j = j0 + c;
            float a = fminf(fmaxf(mean[(long long)i * ldm + j], -1.0f), 1.0f);
            if (!deterministic) {
                const float e = (unit_noise != nullptr) ? unit_noise[(long long)i * A + j] : z[c];
                a = (float)((double)a + (double)sg * (double)e);      // float32 array += float64 noise
            }
            action[(long long)i * A + j] = fminf(fmaxf(a, -1.0f), 1.0f);
        }
    }
}

// DDPGAgent.act with Ornstein-Uhlenbeck exploration (action_noise.py:22-39): per-actor float64 state
//   x <- x + theta*(mu - x)*dt + sigma_i*sqrt(dt)*N(0,1)   (mu = 0; numpy evaluates it left to right in float64),
// action = clip(clip(pi(s)) + x).  One thread per (actor, action dim); no FMA contraction, to match numpy.
__global__ void __launch_bounds__(RT) ddpg_ou_noise_kernel(const float* __restrict__ mean, long long ldm,
                                                           const double* __restrict__ sigma,
                                                           const float* __restrict__ unit_noise, int N, int A,
                                                           int deterministic, unsigned long long seed,
                                                           const unsigned long long* __restrict__ step_ctr, double theta,
                                                           double dt, double* __restrict__ ou_state,
                                                           float* __restrict__ action) {
    const int idx = blockIdx.x * RT + threadIdx.x;
    if (idx >= N * A) return;
    const int i = idx / A, j = idx - i * A;
    float a = fminf(fmaxf(mean[(long long)i * ldm + j], -1.0f), 1.0f);
    if (!deterministic) {
        double e;
        if (unit_noise != nullptr) {
            e = (double)unit_noise[idx];
        } else {
            const unsigned long long ctr = (step_ctr != nullptr) ? *step_ctr : 0ull;
            e = (double)action_noise1(seed, ctr, i, j);
        }
        const double xp = ou_state[idx];
        const double drift = __dmul_rn(__dmul_rn(theta, 0.0 - xp), dt);
        const double diff = __dmul_rn(__dmul_rn(sigma[i], sqrt(dt)), e);
        const double x = __dadd_rn(__dadd_rn(xp, drift), diff);
        ou_state[idx] = x;
        a = (float)((double)a + x);                          // float32 array += float64 noise
    }
    action[(long long)i * A + j] = fminf(fmaxf(a, -1.0f), 1.0f);
}

__global__ void __launch_bounds__(1024) ppo_window_slots_kernel(int N, int n_step, const int* __restrict__ stage_pos,
                                                                int* __restrict__ dest, FifoState* fifo,
                                                                unsigned long long* step_ctr) {
    assign_window_slots(N, n_step, stage_pos, dest, fifo);
    if (threadIdx.x == 0 && step_ctr != nullptr) *step_ctr += 1ull;
}

__global__ void __launch_bounds__(128) ppo_window_commit_kernel(const float* __restrict__ obs_next,
                                                                const float* __restrict__ obs_reset,
                                                                const float* __restrict__ reward,
                                                                const float* __restrict__ done, int N, int n_step,
                                                                int stride, int D, int A,
                                                                int* __restrict__ stage_pos,
                                                                float* __restrict__ stage_obs,
                                                                float* __restrict__ stage_act,
                                                                float* __restrict__ stage_pd,
                                                                float* __restrict__ stage_rew,
                                                                float* __restrict__ stage_done,
                                                                const int* __restrict__ dest,
                                                                float* __restrict__ r_obs, float* __restrict__ r_act,
                                                                float* __restrict__ r_pd, float* __restrict__ r_rew,
                                                                float* __restrict__ r_done) {
    const int i = blockIdx.x;
    commit_actor(true, i, threadIdx.x, blockDim.x, obs_next + (long long)i * D, obs_reset + (long long)i * D, reward[i],
                 done[i], n_step, stride, D, A, stage_pos + i, dest[i], stage_obs, stage_act, stage_pd, stage_rew,
                 stage_done, r_obs, r_act, r_pd, r_rew, r_done);
}

// Window commit of an RNN policy: the record row [obs (Do) | h_0 .. h_{L-1} | c_0 .. c_{L-1}] (utils.rnn_cell_layout) is
// assembled in shared memory from the env's row and the agent's [L][N][H] cells, for the successor and the reset row alike,
// then committed as any other row.
__global__ void __launch_bounds__(128) ppo_window_commit_rnn_kernel(const float* __restrict__ obs_next,
                                                                    const float* __restrict__ obs_reset,
                                                                    const float* __restrict__ reward,
                                                                    const float* __restrict__ done, int N, int n_step,
                                                                    int stride, int Do, int L, int H,
                                                                    const float* __restrict__ h,
                                                                    const float* __restrict__ c, int A,
                                                                    int* __restrict__ stage_pos,
                                                                    float* __restrict__ stage_obs,
                                                                    float* __restrict__ stage_act,
                                                                    float* __restrict__ stage_pd,
                                                                    float* __restrict__ stage_rew,
                                                                    float* __restrict__ stage_done,
                                                                    const int* __restrict__ dest,
                                                                    float* __restrict__ r_obs, float* __restrict__ r_act,
                                                                    float* __restrict__ r_pd, float* __restrict__ r_rew,
                                                                    float* __restrict__ r_done) {
    extern __shared__ float rows[];                // [2][D]: successor row, reset row
    const int i = blockIdx.x;
    const int LH = L * H, D = Do + 2 * LH;
    float* s_next = rows;
    float* s_reset = rows + D;
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
        if (d < Do) {
            s_next[d] = obs_next[(long long)i * Do + d];
            s_reset[d] = obs_reset[(long long)i * Do + d];
        } else {
            const int e = d - Do, which = e / LH, r = e - which * LH, k = r / H, j = r - k * H;
            const float v = (which == 0 ? h : c)[((long long)k * N + i) * H + j];
            s_next[d] = v;
            s_reset[d] = v;
        }
    }
    __syncthreads();
    commit_actor(true, i, threadIdx.x, blockDim.x, s_next, s_reset, reward[i], done[i], n_step, stride, D, A, stage_pos + i,
                 dest[i], stage_obs, stage_act, stage_pd, stage_rew, stage_done, r_obs, r_act, r_pd, r_rew, r_done);
}

// Record row [obs (Do) | h_0 .. h_{L-1} | c_0 .. c_{L-1}] of actor i read straight from the env's row and the agent's
// [L][N][H] cells: the commit of rows too wide to stage in shared memory (a pixel frame plus the cells).
struct CellRow {
    const float* __restrict__ obs;      // the actor's Do observation words
    const float* __restrict__ h;
    const float* __restrict__ c;
    int Do, LH, H, N, i;
    __device__ __forceinline__ float operator[](int d) const {
        if (d < Do) return obs[d];
        int e = d - Do;
        const float* cells = h;
        if (e >= LH) {
            e -= LH;
            cells = c;
        }
        const int k = e / H;
        return cells[((long long)k * N + i) * H + (e - k * H)];
    }
};

__global__ void __launch_bounds__(128, 4) ppo_window_commit_rnn_wide_kernel(const float* __restrict__ obs_next,
                                                                         const float* __restrict__ obs_reset,
                                                                         const float* __restrict__ reward,
                                                                         const float* __restrict__ done, int N, int n_step,
                                                                         int stride, int Do, int L, int H,
                                                                         const float* __restrict__ h,
                                                                         const float* __restrict__ c, int A,
                                                                         int* __restrict__ stage_pos,
                                                                         float* __restrict__ stage_obs,
                                                                         float* __restrict__ stage_act,
                                                                         float* __restrict__ stage_pd,
                                                                         float* __restrict__ stage_rew,
                                                                         float* __restrict__ stage_done,
                                                                         const int* __restrict__ dest,
                                                                         float* __restrict__ r_obs, float* __restrict__ r_act,
                                                                         float* __restrict__ r_pd, float* __restrict__ r_rew,
                                                                         float* __restrict__ r_done) {
    const int i = blockIdx.x;
    const CellRow next = {obs_next + (long long)i * Do, h, c, Do, L * H, H, N, i};
    const CellRow reset = {obs_reset + (long long)i * Do, h, c, Do, L * H, H, N, i};
    commit_actor<BlockBarrier, CellRow>(true, i, threadIdx.x, blockDim.x, next, reset, reward[i], done[i], n_step, stride,
                                        Do + 2 * L * H, A, stage_pos + i, dest[i], stage_obs, stage_act, stage_pd, stage_rew,
                                        stage_done, r_obs, r_act, r_pd, r_rew, r_done);
}

}  // namespace

static bool sample_args_ok(const float* mean, int64_t ldm, const float* log_var, int N, int A,
                           const uint64_t* step_counter, const float* action, const float* pd, const sb200_windows* stage,
                           int assign_slots) {
    return mean && log_var && action && pd && N >= 1 && A >= 1 && ldm >= A &&
           (stage == nullptr || (windows_ok(stage) && stage->N == N && stage->A == A)) &&
           // the fused slot assignment advances the staging's step counter, which must be the one the draws are keyed by
           (!assign_slots || (stage != nullptr && step_counter != nullptr && step_counter == stage->step_counter));
}

extern "C" int sb200_ppo_sample_f32(const float* mean, int64_t ldm, const float* log_var, const float* log_noise,
                                    const float* eps, int N, int A, int deterministic, uint64_t seed, uint64_t* step_counter,
                                    float* action, float* pd, const sb200_windows* stage, int assign_slots, void* stream) {
    SB200_REQUIRE(sample_args_ok(mean, ldm, log_var, N, A, step_counter, action, pd, stage, assign_slots));
    ppo_sample_kernel<<<(N * ((A + 3) / 4) + RT - 1) / RT, RT, 0, (cudaStream_t)stream>>>(
        mean, ldm, log_var, log_noise, eps, N, A, deterministic, (unsigned long long)seed,
        (const unsigned long long*)step_counter, action, pd, stage ? stage->stage_pos : nullptr,
        stage ? stage->stage_act : nullptr, stage ? stage->stage_pd : nullptr, stage ? stage->n_step : 1,
        assign_slots ? (FifoState*)stage->fifo_state : nullptr, assign_slots ? stage->dest : nullptr,
        assign_slots ? (unsigned long long*)step_counter : nullptr);
    return sb200_launch_status();
}

extern "C" int sb200_ddpg_noise_f32(const float* mean, int64_t ldm, const float* sigma, const float* unit_noise, int N,
                                    int A, int deterministic, uint64_t seed, const uint64_t* step_counter,
                                    float* action, void* stream) {
    SB200_REQUIRE(mean && sigma && action && N >= 1 && A >= 1 && ldm >= A);
    ddpg_noise_kernel<<<(N + RT - 1) / RT, RT, 0, (cudaStream_t)stream>>>(
        mean, ldm, sigma, unit_noise, N, A, deterministic, (unsigned long long)seed,
        (const unsigned long long*)step_counter, action);
    return sb200_launch_status();
}

extern "C" int sb200_ddpg_ou_noise_f32(const float* mean, int64_t ldm, const double* sigma, const float* unit_noise,
                                       int N, int A, int deterministic, uint64_t seed, const uint64_t* step_counter,
                                       double theta, double dt, double* ou_state, float* action, void* stream) {
    SB200_REQUIRE(mean && sigma && ou_state && action && N >= 1 && A >= 1 && ldm >= A);
    ddpg_ou_noise_kernel<<<(N * A + RT - 1) / RT, RT, 0, (cudaStream_t)stream>>>(
        mean, ldm, sigma, unit_noise, N, A, deterministic, (unsigned long long)seed,
        (const unsigned long long*)step_counter, theta, dt, ou_state, action);
    return sb200_launch_status();
}

extern "C" size_t sb200_fifo_state_bytes(void) { return sizeof(FifoState); }

extern "C" int sb200_ppo_window_step_f32(const sb200_windows* w, const sb200_window_rows* r, void* stream) {
    SB200_REQUIRE(windows_ok(w) && r != nullptr && r->obs_next && r->obs_reset && r->reward && r->done);
    SB200_REQUIRE(r->obs_dim >= 1 && r->layers >= 0 && (r->layers == 0 || (r->H >= 1 && r->h && r->c)));
    SB200_REQUIRE(w->D == r->obs_dim + 2 * r->layers * r->H);
    const bool host = r->obs_reset_host != nullptr;
    SB200_REQUIRE(host ? (r->obs_next_host && r->reward_host && r->done_host)
                       : (!r->obs_next_host && !r->reward_host && !r->done_host));
    const int N = w->N, n = w->n_step, L = r->layers, H = r->H, Do = r->obs_dim;
    cudaStream_t st = (cudaStream_t)stream;
    const float* next = r->obs_next;
    if (host) {
        const size_t row_bytes = (size_t)N * Do * sizeof(float);
        SB200_CUDA(cudaMemcpyAsync(r->obs_reset, r->obs_reset_host, row_bytes, cudaMemcpyHostToDevice, st));
        if (r->obs_next_host != r->obs_reset_host)
            SB200_CUDA(cudaMemcpyAsync(r->obs_next, r->obs_next_host, row_bytes, cudaMemcpyHostToDevice, st));
        else
            next = r->obs_reset;
        SB200_CUDA(cudaMemcpyAsync(r->reward, r->reward_host, (size_t)N * sizeof(float), cudaMemcpyHostToDevice, st));
        SB200_CUDA(cudaMemcpyAsync(r->done, r->done_host, (size_t)N * sizeof(float), cudaMemcpyHostToDevice, st));
    }
    if (!r->slots_assigned)
        ppo_window_slots_kernel<<<1, 1024, 0, st>>>(N, n, w->stage_pos, w->dest, (FifoState*)w->fifo_state,
                                                    (unsigned long long*)w->step_counter);
    const size_t smem = (size_t)2 * w->D * sizeof(float);
    if (L == 0)
        ppo_window_commit_kernel<<<N, 128, 0, st>>>(next, r->obs_reset, r->reward, r->done, N, n, w->stride, w->D, w->A,
                                                    w->stage_pos, w->stage_obs, w->stage_act, w->stage_pd, w->stage_rew,
                                                    w->stage_done, w->dest, w->r_obs, w->r_act, w->r_pd, w->r_rew, w->r_done);
    else if (smem > 48 * 1024 || r->force_wide)             // rows too wide to stage in shared memory
        ppo_window_commit_rnn_wide_kernel<<<N, 128, 0, st>>>(next, r->obs_reset, r->reward, r->done, N, n, w->stride, Do, L,
                                                             H, r->h, r->c, w->A, w->stage_pos, w->stage_obs, w->stage_act,
                                                             w->stage_pd, w->stage_rew, w->stage_done, w->dest, w->r_obs,
                                                             w->r_act, w->r_pd, w->r_rew, w->r_done);
    else
        ppo_window_commit_rnn_kernel<<<N, 128, smem, st>>>(next, r->obs_reset, r->reward, r->done, N, n, w->stride, Do, L, H,
                                                           r->h, r->c, w->A, w->stage_pos, w->stage_obs, w->stage_act,
                                                           w->stage_pd, w->stage_rew, w->stage_done, w->dest, w->r_obs,
                                                           w->r_act, w->r_pd, w->r_rew, w->r_done);
    return sb200_launch_status(r->slots_assigned ? 1 : 2);
}

// ------------------------------------------------------------------------------------------------
// Act entries: one C call per agent.act() for host and device observations alike.  The per-step work is tens of
// microseconds of GPU time, so separate Python-level copy / launch calls would cost more than the kernels; here the PCIe
// copies, launches and the single stream synchronisation are issued back to back from C, after every argument has been
// checked.  Host pointers must be pinned (cudaHostAlloc / torch pin_memory) for the copies to be asynchronous.
extern "C" int sb200_ppo_act_f32(const sb200_ppo_act* a, void* stream) {
    SB200_REQUIRE(a != nullptr && a->head != nullptr && a->head->n_layers >= 1 && a->head->n_layers <= SB200_MAX_LAYERS);
    SB200_REQUIRE(a->layers >= 0 && a->layers <= SB200_MAX_RNN_LAYERS && a->N >= 1 && a->D >= 1);
    const bool stem = a->frames != nullptr, rnn = a->layers > 0;
    const int N = a->N, D = a->D, H = a->H, L = a->layers, A = a->head->dims[a->head->n_layers];
    // stem geometry (k8 s4 then k4 s2)
    const int H1 = (a->frame_h - 8) / 4 + 1, W1 = (a->frame_w - 8) / 4 + 1;
    const int H2 = (H1 - 4) / 2 + 1, W2 = (W1 - 4) / 2 + 1;
    SB200_REQUIRE(stem ? (a->fc && a->conv_w1 && a->conv_b1 && a->conv_w2 && a->conv_b2 && a->a1 && a->a2 &&
                          a->obs_host == nullptr && a->frame_c >= 1 && a->frame_h >= 8 && a->frame_w >= 8 && H1 >= 4 &&
                          W1 >= 4 && a->fc->n_layers == 1 && a->fc->dims[0] == 32 * H2 * W2 && a->fc->dims[1] == D)
                       : (a->obs && a->ld_obs >= D && a->frames_host == nullptr));
    SB200_REQUIRE(a->obs_host == nullptr || a->ld_obs == D);
    SB200_REQUIRE(!(stem || rnn) || (a->xf && a->ld_xf >= D));
    SB200_REQUIRE(a->head_packed == nullptr || !(stem || rnn));
    SB200_REQUIRE(a->head->dims[0] == (rnn ? H : D));
    if (rnn) {
        SB200_REQUIRE(H >= 1 && a->ldh >= H && a->pre_x && a->h_out[0] && (L == 1 || a->h_out[1]));
        SB200_REQUIRE(a->h && a->c && a->h_before && a->c_before);
        for (int k = 0; k < L; ++k)
            SB200_REQUIRE(a->ih[k] && a->whh[k] && a->bhh[k] && a->ih[k]->n_layers == 1 && a->ih[k]->dims[1] == 4 * H);
    }
    SB200_REQUIRE(a->action_host == nullptr || a->pd_host != nullptr);
    SB200_REQUIRE((a->h_before_host == nullptr) == (a->c_before_host == nullptr) && (a->h_before_host == nullptr || rnn));
    SB200_REQUIRE(a->pd_type == SB200_PD_GAUSSIAN || a->pd_type == SB200_PD_CATEGORICAL);
    const bool cat = a->pd_type == SB200_PD_CATEGORICAL;
    // the categorical sampler checks its own arguments when it is called, after the forward
    SB200_REQUIRE(cat || sample_args_ok(a->mean, A, a->log_var, N, A, a->step_counter, a->action, a->pd, a->stage,
                                        a->assign_slots));
    SB200_REQUIRE(!cat || (A >= 2 && A <= SB200_PPO_CAT_MAX_K && a->mean && a->action && a->pd));
    // no LayerNorm in the recurrent policy's head, input projections or CNN stem
    if ((rnn && sb200_mlp_has_ln(a->head)) || (stem && sb200_mlp_has_ln(a->fc))) return SB200_ERR_UNSUPPORTED;
    for (int k = 0; k < L; ++k)
        if (sb200_mlp_has_ln(a->ih[k])) return SB200_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t cells = (size_t)L * N * H * sizeof(float);
    const sb200_zfilter nozf = {nullptr, 1e-5f};
    if (a->obs_host != nullptr)
        SB200_CUDA(cudaMemcpyAsync(a->obs, a->obs_host, (size_t)N * D * sizeof(float), cudaMemcpyHostToDevice, st));
    if (a->frames_host != nullptr)
        SB200_CUDA(cudaMemcpyAsync(a->frames, a->frames_host, (size_t)N * a->frame_c * a->frame_h * a->frame_w,
                                   cudaMemcpyHostToDevice, st));
    if (rnn) {
        SB200_CUDA(cudaMemcpyAsync(a->h_before, a->h, cells, cudaMemcpyDeviceToDevice, st));
        SB200_CUDA(cudaMemcpyAsync(a->c_before, a->c, cells, cudaMemcpyDeviceToDevice, st));
    }
    int rc = SB200_OK;
    if (stem) {
        rc = sb200_conv_forward_f32(1, a->frames, 1, N, a->frame_c, a->frame_h, a->frame_w, a->conv_w1, a->conv_b1,
                                    1.0 / 255.0, a->a1, stream);
        if (rc != SB200_OK) return rc;
        rc = sb200_conv_forward_f32(2, a->a1, 0, N, 16, H1, W1, a->conv_w2, a->conv_b2, 1.0, a->a2, stream);
        if (rc != SB200_OK) return rc;
        rc = sb200_forward_out(a->fc, &nozf, a->a2, a->fc->dims[0], N, a->xf, a->ld_xf, stream);
    } else if (rnn) {
        rc = sb200_rows_zfilter_f32(a->obs, D, a->ld_obs, N, 1, D, a->zf.stats, (double)a->zf.eps, a->xf, a->ld_xf, stream);
    }
    if (rc != SB200_OK) return rc;
    // the MLP policy's head reads the observation rows and applies the z-filter itself
    const float* x = (stem || rnn) ? a->xf : a->obs;
    int64_t ldx = (stem || rnn) ? a->ld_xf : a->ld_obs;
    for (int k = 0; k < L; ++k) {
        rc = sb200_forward_out(a->ih[k], &nozf, x, ldx, N, a->pre_x, 4 * H, stream);
        if (rc != SB200_OK) return rc;
        float* ho = a->h_out[(L - 1 - k) & 1];
        float* hk = a->h + (size_t)k * N * H;
        float* ck = a->c + (size_t)k * N * H;
        rc = sb200_lstm_forward_f32(a->pre_x, a->whh[k], a->bhh[k], hk, ck, H, N, 1, H, a->ldh, ho, nullptr, nullptr, nullptr,
                                    hk, ck, stream);
        if (rc != SB200_OK) return rc;
        x = ho;
        ldx = a->ldh;
    }
    const sb200_zfilter* zf = (stem || rnn) ? &nozf : &a->zf;
    if (a->head_packed != nullptr) {
        const sb200_rows in = {x, nullptr, ldx, N, 0, nullptr, 0, nullptr, 0};
        rc = sb200_mlp_forward_packed_f32(a->head, a->head_packed, zf, &in, a->mean, A, stream);
    } else {
        rc = sb200_forward_out(a->head, zf, x, ldx, N, a->mean, A, stream);
    }
    if (rc != SB200_OK) return rc;
    if (cat)
        rc = sb200_ppo_cat_sample_f32(a->mean, A, N, A, a->deterministic, a->seed, a->step_counter, a->action, a->pd, nullptr,
                                      a->stage, a->assign_slots, stream);
    else
        rc = sb200_ppo_sample_f32(a->mean, A, a->log_var, a->log_noise, a->eps, N, A, a->deterministic, a->seed,
                                  a->step_counter, a->action, a->pd, a->stage, a->assign_slots, stream);
    if (rc != SB200_OK || a->action_host == nullptr) return rc;
    SB200_CUDA(cudaMemcpyAsync(a->action_host, a->action, (size_t)N * A * sizeof(float), cudaMemcpyDeviceToHost, st));
    SB200_CUDA(cudaMemcpyAsync(a->pd_host, a->pd, (size_t)N * 2 * A * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (a->h_before_host != nullptr) {
        SB200_CUDA(cudaMemcpyAsync(a->h_before_host, a->h_before, cells, cudaMemcpyDeviceToHost, st));
        SB200_CUDA(cudaMemcpyAsync(a->c_before_host, a->c_before, cells, cudaMemcpyDeviceToHost, st));
    }
    SB200_CUDA(cudaStreamSynchronize(st));
    return SB200_OK;
}

extern "C" int sb200_ddpg_act_f32(const sb200_ddpg_act* a, void* stream) {
    SB200_REQUIRE(a != nullptr && a->net != nullptr && a->net->n_layers >= 1 && a->net->n_layers <= SB200_MAX_LAYERS);
    const int N = a->N, D = a->net->dims[0], A = a->net->dims[a->net->n_layers];
    SB200_REQUIRE(N >= 1 && A >= 1 && a->obs && a->ld_obs >= D && (a->obs_host == nullptr || a->ld_obs == D));
    SB200_REQUIRE(a->mean && a->action && (a->ou_state != nullptr ? a->sigma64 != nullptr : a->sigma != nullptr));
    SB200_REQUIRE(a->forward == SB200_DDPG_FWD_FUSED || (a->forward == SB200_DDPG_FWD_PACKED && a->packed) ||
                  (a->forward == SB200_DDPG_FWD_PER_ACTOR && a->actor_stride >= 0 && a->actor_stride % 4 == 0 &&
                   (a->shared == nullptr || (a->dist && a->pn_state && a->dist_interval >= 1))));
    cudaStream_t st = (cudaStream_t)stream;
    if (a->obs_host != nullptr)
        SB200_CUDA(cudaMemcpyAsync(a->obs, a->obs_host, (size_t)N * D * sizeof(float), cudaMemcpyHostToDevice, st));
    const sb200_zfilter nozf = {nullptr, 1e-5f};
    int rc;
    if (a->forward == SB200_DDPG_FWD_PER_ACTOR) {
        rc = sb200_mlp_forward_per_actor_f32(a->net, a->actor_stride, a->obs, a->ld_obs, N, a->mean, A, a->shared, a->dist,
                                             a->dist_interval, a->pn_state, stream);
    } else if (a->forward == SB200_DDPG_FWD_PACKED) {
        const sb200_rows in = {a->obs, nullptr, a->ld_obs, N, 0, nullptr, 0, nullptr, 0};
        rc = sb200_mlp_forward_packed_f32(a->net, a->packed, &nozf, &in, a->mean, A, stream);
    } else {
        rc = sb200_forward_out(a->net, &nozf, a->obs, a->ld_obs, N, a->mean, A, stream);
    }
    if (rc != SB200_OK) return rc;
    if (a->ou_state != nullptr)
        rc = sb200_ddpg_ou_noise_f32(a->mean, A, a->sigma64, a->unit_noise, N, A, a->deterministic, a->seed, a->step_counter,
                                     a->theta, a->dt, a->ou_state, a->action, stream);
    else
        rc = sb200_ddpg_noise_f32(a->mean, A, a->sigma, a->unit_noise, N, A, a->deterministic, a->seed, a->step_counter,
                                  a->action, stream);
    if (rc != SB200_OK || a->action_host == nullptr) return rc;
    SB200_CUDA(cudaMemcpyAsync(a->action_host, a->action, (size_t)N * A * sizeof(float), cudaMemcpyDeviceToHost, st));
    SB200_CUDA(cudaStreamSynchronize(st));
    return SB200_OK;
}
