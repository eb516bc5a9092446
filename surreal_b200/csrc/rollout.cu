// Actor-side kernels of the batched rollout: policy sampling, exploration noise, the synthetic
// device-resident environment, and the per-actor experience staging that replaces the Python deques of
// surreal/env/exp_sender_wrapper.py (windows for PPO, n-step SSAR records for DDPG).
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
        const Philox4 r = philox4x32_10(seed, ctr, ((unsigned long long)i << 16) | (unsigned long long)(j0 >> 2));
        const float2 a = box_muller(r.x, r.y), b = box_muller(r.z, r.w);
        z[0] = a.x; z[1] = a.y; z[2] = b.x; z[3] = b.y;
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int j = j0 + c;
        if (j >= A) break;
        const float mu = mean[(long long)i * ldm + j];
        const float sd = __fmul_rn(expf(log_var[j]), sc);
        float a = mu;
        if (!deterministic) {
            const float e = (eps != nullptr) ? eps[(long long)i * A + j] : z[c];
            a = __fadd_rn(__fmul_rn(e, sd), mu);
        }
        a = fminf(fmaxf(a, -1.0f), 1.0f);
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
            const Philox4 r = philox4x32_10(seed, ctr, ((unsigned long long)i << 16) | (unsigned long long)(j0 >> 2));
            const float2 a = box_muller(r.x, r.y), b = box_muller(r.z, r.w);
            z[0] = a.x; z[1] = a.y; z[2] = b.x; z[3] = b.y;
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
            const Philox4 r = philox4x32_10(seed, ctr, ((unsigned long long)i << 16) | (unsigned long long)(j >> 2));
            const float2 z01 = box_muller(r.x, r.y), z23 = box_muller(r.z, r.w);
            const int c = j & 3;
            e = (double)((c == 0) ? z01.x : (c == 1) ? z01.y : (c == 2) ? z23.x : z23.y);
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

// ------------------------------------------------------------------------------------------------
// Synthetic environment of SURVEY §8(d) cfg 2/3/5, batched and device-resident:
//   s' = tanh(Ws s + Wa a) + 0.01*xi,   r = -|s|^2 / D + 0.1*xi',   done when the episode reaches
//   `max_steps` (MaxStepWrapper, env/wrapper.py:142-163); on done the state is re-drawn ~ N(0,1).
// One block per 4 actors; the weights are passed TRANSPOSED (WsT [D][D], WaT [A][D]: k-major) so that the
// threads of a warp read consecutive addresses; they stay L1/L2-resident (18 KB).  obs_next = the true successor (terminal
// when done), state = what the agent observes next (reset when done).
// Block-level body (RT threads, 4 actors).  s_n / s_z (optional) receive the successor and the next observed
// state of the block's actors, s_rew / s_dn their reward and done flag.
__device__ void synth_env_block(float* __restrict__ state, const float* __restrict__ action,
                                const float* __restrict__ Ws, const float* __restrict__ Wa, int N, int D, int A,
                                int max_steps, int* __restrict__ ep_step, unsigned long long seed,
                                const unsigned long long* __restrict__ step_ctr, float* __restrict__ obs_next,
                                float* __restrict__ reward, float* __restrict__ done, float* s_s, float* s_a,
                                float* s_q, float* s_n, float* s_z, float* s_rew, float* s_dn,
                                unsigned long long ctr_bias) {
    const int per = 4;
    const int a0 = blockIdx.x * per;
    const int tid = threadIdx.x;
    for (int idx = tid; idx < per * D; idx += RT) {
        const int q = idx / D, d = idx - q * D;
        s_s[idx] = (a0 + q < N) ? state[(long long)(a0 + q) * D + d] : 0.0f;
    }
    for (int idx = tid; idx < per * A; idx += RT) {
        const int q = idx / A, j = idx - q * A;
        s_a[idx] = (a0 + q < N) ? action[(long long)(a0 + q) * A + j] : 0.0f;
    }
    __syncthreads();
    // ctr_bias = -1 in the fused rollout, where the sampling kernel has already advanced the counter: both launch
    // sequences then draw the same noise for the same step
    const unsigned long long ctr = ((step_ctr != nullptr) ? *step_ctr : 0ull) + ctr_bias;
    // reward: -|s|^2/D (+ noise), one warp per actor (warps 0..3)
    const int warp = tid >> 5, lane = tid & 31;
    if (warp < per) {
        float q = 0.0f;
        for (int d = lane; d < D; d += 32) q += s_s[warp * D + d] * s_s[warp * D + d];
        q = warp_sum(q);
        if (lane == 0) s_q[warp] = q;
    }
    __syncthreads();
    for (int idx = tid; idx < per * D; idx += RT) {
        const int q = idx / D, d = idx - q * D;
        const int i = a0 + q;
        if (i >= N) continue;
        float acc = 0.0f;                                   // WsT / WaT are [k][d]: coalesced across d
#pragma unroll 8
        for (int k = 0; k < D; ++k) acc = fmaf(__ldg(Ws + (long long)k * D + d), s_s[q * D + k], acc);
#pragma unroll 4
        for (int k = 0; k < A; ++k) acc = fmaf(__ldg(Wa + (long long)k * D + d), s_a[q * A + k], acc);
        const Philox4 r = philox4x32_10(seed ^ 0x5851F42D4C957F2Dull, ctr, ((unsigned long long)i << 20) | (unsigned long long)d);
        const float2 g = box_muller(r.x, r.y);
        const float nxt = tanhf(acc) + 0.01f * g.x;
        const int t = ep_step[i] + 1;
        const bool dn = (max_steps > 0) && (t >= max_steps);
        const float st = dn ? box_muller(r.z, r.w).x : nxt;
        obs_next[(long long)i * D + d] = nxt;
        state[(long long)i * D + d] = st;
        if (s_n != nullptr) {
            s_n[idx] = nxt;
            s_z[idx] = st;
        }
        if (d == 0) {
            const float rw = -s_q[q] / (float)D + 0.1f * g.y;
            reward[i] = rw;
            done[i] = dn ? 1.0f : 0.0f;
            if (s_rew != nullptr) {
                s_rew[q] = rw;
                s_dn[q] = dn ? 1.0f : 0.0f;
            }
        }
    }
    __syncthreads();
    for (int q = tid; q < per; q += RT) {
        const int i = a0 + q;
        if (i < N) {
            const int t = ep_step[i] + 1;
            ep_step[i] = ((max_steps > 0) && (t >= max_steps)) ? 0 : t;
        }
    }
}

__global__ void __launch_bounds__(RT) synth_env_step_kernel(float* __restrict__ state, const float* __restrict__ action,
                                                            const float* __restrict__ Ws, const float* __restrict__ Wa,
                                                            int N, int D, int A, int max_steps,
                                                            int* __restrict__ ep_step, unsigned long long seed,
                                                            const unsigned long long* __restrict__ step_ctr,
                                                            float* __restrict__ obs_next, float* __restrict__ reward,
                                                            float* __restrict__ done) {
    extern __shared__ float sm[];                  // [4][D] states, [4][A] actions
    __shared__ float s_q[4];
    synth_env_block(state, action, Ws, Wa, N, D, A, max_steps, ep_step, seed, step_ctr, obs_next, reward, done, sm,
                    sm + 4 * D, s_q, nullptr, nullptr, nullptr, nullptr, 0ull);
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

// Fused environment step + window commit for the device-resident synthetic env: the successor state never
// leaves shared memory before it is staged.  One block per 4 actors, 64 threads per actor in the commit.
__global__ void __launch_bounds__(RT) synth_env_window_step_kernel(
    float* __restrict__ state, const float* __restrict__ action, const float* __restrict__ Ws,
    const float* __restrict__ Wa, int N, int D, int A, int max_steps, int* __restrict__ ep_step,
    unsigned long long seed, const unsigned long long* __restrict__ step_ctr, float* __restrict__ obs_next,
    float* __restrict__ reward, float* __restrict__ done, int n_step, int stride, int* __restrict__ stage_pos,
    float* __restrict__ stage_obs, float* __restrict__ stage_act, float* __restrict__ stage_pd,
    float* __restrict__ stage_rew, float* __restrict__ stage_done, const int* __restrict__ dest,
    float* __restrict__ r_obs, float* __restrict__ r_act, float* __restrict__ r_pd, float* __restrict__ r_rew,
    float* __restrict__ r_done) {
    extern __shared__ float sm[];                  // [4][D] states, [4][A] actions, [4][D] successor, [4][D] reset
    const int per = 4;
    const int a0 = blockIdx.x * per;
    float* s_s = sm;
    float* s_a = sm + per * D;
    float* s_n = s_a + per * A;
    float* s_z = s_n + per * D;
    __shared__ float s_q[4], s_rew[4], s_dn[4];
    const int tid = threadIdx.x;
    synth_env_block(state, action, Ws, Wa, N, D, A, max_steps, ep_step, seed, step_ctr, obs_next, reward, done, s_s, s_a,
                    s_q, s_n, s_z, s_rew, s_dn, ~0ull);
    __syncthreads();
    const int q = tid >> 6, g = tid & 63;
    const int i = a0 + q;
    commit_actor(i < N, i, g, 64, s_n + q * D, s_z + q * D, s_rew[q], s_dn[q], n_step, stride, D, A, stage_pos + min(i, N - 1),
                 (i < N) ? dest[i] : SLOT_NONE, stage_obs, stage_act, stage_pd, stage_rew, stage_done, r_obs, r_act, r_pd,
                 r_rew, r_done);
}

}  // namespace

extern "C" int sb200_ppo_sample_f32(const float* mean, int64_t ldm, const float* log_var, const float* log_noise,
                                    const float* eps, int N, int A, int deterministic, uint64_t seed,
                                    const uint64_t* step_counter, float* action, float* pd, const int* stage_pos,
                                    float* stage_act, float* stage_pd, int n_step, void* stream) {
    SB200_REQUIRE(mean && log_var && action && pd && N >= 1 && A >= 1 && ldm >= A);
    SB200_REQUIRE(stage_act == nullptr || (stage_pos != nullptr && stage_pd != nullptr && n_step >= 1));
    ppo_sample_kernel<<<(N * ((A + 3) / 4) + RT - 1) / RT, RT, 0, (cudaStream_t)stream>>>(
        mean, ldm, log_var, log_noise, eps, N, A, deterministic, (unsigned long long)seed,
        (const unsigned long long*)step_counter, action, pd, stage_pos, stage_act, stage_pd, n_step, nullptr, nullptr,
        nullptr);
    return sb200_launch_status();
}

extern "C" int sb200_ppo_sample_assign_f32(const float* mean, int64_t ldm, const float* log_var,
                                           const float* log_noise, const float* eps, int N, int A, int deterministic,
                                           uint64_t seed, uint64_t* step_counter, float* action, float* pd,
                                           const int* stage_pos, float* stage_act, float* stage_pd, int n_step,
                                           void* fifo_state, int* dest, void* stream) {
    SB200_REQUIRE(mean && log_var && action && pd && N >= 1 && A >= 1 && ldm >= A);
    SB200_REQUIRE(stage_pos && stage_act && stage_pd && n_step >= 1 && fifo_state && dest && step_counter);
    ppo_sample_kernel<<<(N * ((A + 3) / 4) + RT - 1) / RT, RT, 0, (cudaStream_t)stream>>>(
        mean, ldm, log_var, log_noise, eps, N, A, deterministic, (unsigned long long)seed,
        (const unsigned long long*)step_counter, action, pd, stage_pos, stage_act, stage_pd, n_step,
        (FifoState*)fifo_state, dest, (unsigned long long*)step_counter);
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

extern "C" int sb200_synth_env_step_f32(float* state, const float* action, const float* Ws, const float* Wa, int N,
                                        int D, int A, int max_steps, int* ep_step, uint64_t seed,
                                        const uint64_t* step_counter, float* obs_next, float* reward, float* done,
                                        void* stream) {
    SB200_REQUIRE(state && action && Ws && Wa && ep_step && obs_next && reward && done);
    SB200_REQUIRE(N >= 1 && D >= 1 && A >= 1 && (size_t)(4 * (D + A)) * 4 <= 40 * 1024);
    const size_t smem = (size_t)(4 * (D + A)) * sizeof(float);
    synth_env_step_kernel<<<(N + 3) / 4, RT, smem, (cudaStream_t)stream>>>(
        state, action, Ws, Wa, N, D, A, max_steps, ep_step, (unsigned long long)seed,
        (const unsigned long long*)step_counter, obs_next, reward, done);
    return sb200_launch_status();
}

static bool env_smem_ok(int D, int A, bool fused) {
    return (size_t)(4 * (D + A) + (fused ? 8 * D : 0)) * sizeof(float) <= 40 * 1024;
}

extern "C" int sb200_synth_env_window_step_f32(float* state, const float* action, const float* Ws, const float* Wa,
                                               int N, int D, int A, int max_steps, int* ep_step, uint64_t seed,
                                               const uint64_t* step_counter, float* obs_next, float* reward,
                                               float* done, int n_step, int stride, int* stage_pos, float* stage_obs,
                                               float* stage_act, float* stage_pd, float* stage_rew, float* stage_done,
                                               const int* dest, float* r_obs, float* r_act, float* r_pd, float* r_rew,
                                               float* r_done, void* stream) {
    SB200_REQUIRE(state && action && Ws && Wa && ep_step && obs_next && reward && done);
    SB200_REQUIRE(stage_pos && stage_obs && stage_act && stage_pd && stage_rew && stage_done && dest);
    SB200_REQUIRE(r_obs && r_act && r_pd && r_rew && r_done);
    SB200_REQUIRE(N >= 1 && D >= 1 && A >= 1 && n_step >= 1 && stride >= 1 && env_smem_ok(D, A, true));
    const size_t smem = (size_t)(4 * (D + A) + 8 * D) * sizeof(float);
    synth_env_window_step_kernel<<<(N + 3) / 4, RT, smem, (cudaStream_t)stream>>>(
        state, action, Ws, Wa, N, D, A, max_steps, ep_step, (unsigned long long)seed,
        (const unsigned long long*)step_counter, obs_next, reward, done, n_step, stride, stage_pos, stage_obs, stage_act,
        stage_pd, stage_rew, stage_done, dest, r_obs, r_act, r_pd, r_rew, r_done);
    return sb200_launch_status();
}

extern "C" size_t sb200_fifo_state_bytes(void) { return sizeof(FifoState); }

extern "C" int sb200_ppo_window_step_f32(const float* obs_next, const float* obs_reset, const float* reward,
                                         const float* done, int N, int n_step, int stride, int D, int A,
                                         int* stage_pos, float* stage_obs, float* stage_act, float* stage_pd,
                                         float* stage_rew, float* stage_done, int* dest_scratch, void* fifo_state,
                                         float* r_obs, float* r_act, float* r_pd, float* r_rew, float* r_done,
                                         uint64_t* step_counter, int slots_assigned, void* stream) {
    SB200_REQUIRE(obs_next && obs_reset && reward && done && stage_pos && stage_obs && stage_act && stage_pd);
    SB200_REQUIRE(stage_rew && stage_done && dest_scratch && fifo_state && r_obs && r_act && r_pd && r_rew && r_done);
    SB200_REQUIRE(N >= 1 && n_step >= 1 && stride >= 1 && D >= 1 && A >= 1);
    cudaStream_t st = (cudaStream_t)stream;
    if (!slots_assigned)
        ppo_window_slots_kernel<<<1, 1024, 0, st>>>(N, n_step, stage_pos, dest_scratch, (FifoState*)fifo_state,
                                                    (unsigned long long*)step_counter);
    ppo_window_commit_kernel<<<N, 128, 0, st>>>(obs_next, obs_reset, reward, done, N, n_step, stride, D, A, stage_pos,
                                                stage_obs, stage_act, stage_pd, stage_rew, stage_done, dest_scratch,
                                                r_obs, r_act, r_pd, r_rew, r_done);
    return sb200_launch_status(slots_assigned ? 1 : 2);
}

// ------------------------------------------------------------------------------------------------
// Host-env fast path: one C call per agent.act() / wrapper.step() with a HOST environment.  The per-step work is
// tens of microseconds of GPU time, so the ~10 separate Python-level copy / launch calls of the generic path cost
// more than the kernels; here the PCIe copies, launches and the single stream synchronisation are issued back to
// back from C.  Host pointers must be pinned (cudaHostAlloc / torch pin_memory) for the copies to be asynchronous.
extern "C" int sb200_ppo_act_host_f32(const sb200_mlp* net, const sb200_zfilter* zf, const float* obs_host,
                                      float* obs_dev, int N, float* mean_dev, const float* log_var,
                                      const float* log_noise, int deterministic, uint64_t seed,
                                      uint64_t* step_counter, float* action_dev, float* pd_dev, const int* stage_pos,
                                      float* stage_act, float* stage_pd, int n_step, void* fifo_state, int* dest,
                                      float* action_host, float* pd_host, void* stream) {
    SB200_REQUIRE(net != nullptr && obs_dev != nullptr && mean_dev != nullptr && N >= 1);
    SB200_REQUIRE(action_dev && pd_dev && action_host && pd_host && step_counter);
    cudaStream_t st = (cudaStream_t)stream;
    const int D = net->dims[0], A = net->dims[net->n_layers];
    if (obs_host != nullptr)
        SB200_CUDA(cudaMemcpyAsync(obs_dev, obs_host, (size_t)N * D * sizeof(float), cudaMemcpyHostToDevice, st));
    sb200_rows in = {};
    in.x = obs_dev;
    in.x_next = nullptr;
    in.ldx = D;
    in.rows = N;
    in.win_n = 0;
    in.aux = nullptr;
    in.aux_ld = 0;
    in.save_x = nullptr;
    in.ld_save_x = 0;
    float* save[SB200_MAX_LAYERS] = {nullptr, nullptr, nullptr, nullptr};
    int64_t lds[SB200_MAX_LAYERS] = {0, 0, 0, 0};
    save[net->n_layers - 1] = mean_dev;
    lds[net->n_layers - 1] = A;
    int rc = sb200_mlp_forward_f32(net, zf, &in, save, lds, stream);
    if (rc != SB200_OK) return rc;
    if (fifo_state != nullptr)
        rc = sb200_ppo_sample_assign_f32(mean_dev, A, log_var, log_noise, nullptr, N, A, deterministic, seed, step_counter,
                                         action_dev, pd_dev, stage_pos, stage_act, stage_pd, n_step, fifo_state, dest,
                                         stream);
    else
        rc = sb200_ppo_sample_f32(mean_dev, A, log_var, log_noise, nullptr, N, A, deterministic, seed, step_counter,
                                  action_dev, pd_dev, stage_pos, stage_act, stage_pd, n_step, stream);
    if (rc != SB200_OK) return rc;
    SB200_CUDA(cudaMemcpyAsync(action_host, action_dev, (size_t)N * A * sizeof(float), cudaMemcpyDeviceToHost, st));
    SB200_CUDA(cudaMemcpyAsync(pd_host, pd_dev, (size_t)N * 2 * A * sizeof(float), cudaMemcpyDeviceToHost, st));
    SB200_CUDA(cudaStreamSynchronize(st));
    return SB200_OK;
}

extern "C" int sb200_ppo_window_step_host_f32(const float* obs_next_host, const float* obs_reset_host,
                                              const float* reward_host, const float* done_host, float* obs_next_dev,
                                              float* obs_reset_dev, float* reward_dev, float* done_dev, int N,
                                              int n_step, int stride, int D, int A, int* stage_pos, float* stage_obs,
                                              float* stage_act, float* stage_pd, float* stage_rew, float* stage_done,
                                              int* dest_scratch, void* fifo_state, float* r_obs, float* r_act,
                                              float* r_pd, float* r_rew, float* r_done, uint64_t* step_counter,
                                              int slots_assigned, void* stream) {
    SB200_REQUIRE(obs_next_host && obs_reset_host && reward_host && done_host);
    SB200_REQUIRE(obs_next_dev && obs_reset_dev && reward_dev && done_dev && N >= 1 && D >= 1);
    cudaStream_t st = (cudaStream_t)stream;
    SB200_CUDA(cudaMemcpyAsync(obs_reset_dev, obs_reset_host, (size_t)N * D * sizeof(float), cudaMemcpyHostToDevice, st));
    if (obs_next_host != obs_reset_host)
        SB200_CUDA(cudaMemcpyAsync(obs_next_dev, obs_next_host, (size_t)N * D * sizeof(float), cudaMemcpyHostToDevice, st));
    SB200_CUDA(cudaMemcpyAsync(reward_dev, reward_host, (size_t)N * sizeof(float), cudaMemcpyHostToDevice, st));
    SB200_CUDA(cudaMemcpyAsync(done_dev, done_host, (size_t)N * sizeof(float), cudaMemcpyHostToDevice, st));
    return sb200_ppo_window_step_f32((obs_next_host != obs_reset_host) ? obs_next_dev : obs_reset_dev, obs_reset_dev,
                                     reward_dev, done_dev, N, n_step, stride, D, A, stage_pos, stage_obs, stage_act,
                                     stage_pd, stage_rew, stage_done, dest_scratch, fifo_state, r_obs, r_act, r_pd, r_rew,
                                     r_done, step_counter, slots_assigned, stream);
}

extern "C" int sb200_ddpg_act_host_f32(const sb200_mlp* net, const float* obs_host, float* obs_dev, int N, float* mean_dev,
                                       const float* sigma, const double* sigma64, const float* unit_noise, int deterministic,
                                       uint64_t seed, const uint64_t* step_counter, double theta, double dt,
                                       double* ou_state, float* action_dev, float* action_host, void* stream) {
    SB200_REQUIRE(net != nullptr && obs_dev != nullptr && mean_dev != nullptr && action_dev && action_host && N >= 1);
    SB200_REQUIRE(ou_state != nullptr ? sigma64 != nullptr : sigma != nullptr);
    cudaStream_t st = (cudaStream_t)stream;
    const int D = net->dims[0], A = net->dims[net->n_layers];
    if (obs_host != nullptr)
        SB200_CUDA(cudaMemcpyAsync(obs_dev, obs_host, (size_t)N * D * sizeof(float), cudaMemcpyHostToDevice, st));
    const sb200_zfilter nozf = {nullptr, 1e-5f};
    const sb200_rows in = {obs_dev, nullptr, D, N, 0, nullptr, 0, nullptr, 0};
    float* save[SB200_MAX_LAYERS] = {nullptr, nullptr, nullptr, nullptr};
    int64_t lds[SB200_MAX_LAYERS] = {0, 0, 0, 0};
    save[net->n_layers - 1] = mean_dev;
    lds[net->n_layers - 1] = A;
    int rc = sb200_mlp_forward_f32(net, &nozf, &in, save, lds, stream);
    if (rc != SB200_OK) return rc;
    if (ou_state != nullptr)
        rc = sb200_ddpg_ou_noise_f32(mean_dev, A, sigma64, unit_noise, N, A, deterministic, seed, step_counter, theta, dt,
                                     ou_state, action_dev, stream);
    else
        rc = sb200_ddpg_noise_f32(mean_dev, A, sigma, unit_noise, N, A, deterministic, seed, step_counter, action_dev, stream);
    if (rc != SB200_OK) return rc;
    SB200_CUDA(cudaMemcpyAsync(action_host, action_dev, (size_t)N * A * sizeof(float), cudaMemcpyDeviceToHost, st));
    SB200_CUDA(cudaStreamSynchronize(st));
    return SB200_OK;
}

extern "C" int sb200_ppo_act_rnn_f32(const sb200_ppo_act_rnn* a, void* stream) {
    SB200_REQUIRE(a != nullptr && a->head != nullptr && a->layers >= 1 && a->layers <= SB200_MAX_RNN_LAYERS);
    const bool stem = a->frames != nullptr;
    SB200_REQUIRE(a->N >= 1 && a->D >= 1 && a->H >= 1 && a->ldh >= a->H && a->ld_xf >= a->D);
    // stem geometry (k8 s4 then k4 s2), checked before anything is issued
    const int H1 = (a->frame_h - 8) / 4 + 1, W1 = (a->frame_w - 8) / 4 + 1;
    const int H2 = (H1 - 4) / 2 + 1, W2 = (W1 - 4) / 2 + 1;
    SB200_REQUIRE(stem ? (a->fc && a->conv_w1 && a->conv_b1 && a->conv_w2 && a->conv_b2 && a->a1 && a->a2 &&
                          a->obs_host == nullptr && a->frame_c >= 1 && a->frame_h >= 8 && a->frame_w >= 8 && H1 >= 4 &&
                          W1 >= 4 && a->fc->n_layers == 1 && a->fc->dims[0] == 32 * H2 * W2 && a->fc->dims[1] == a->D)
                       : (a->obs && a->ld_obs >= a->D && a->frames_host == nullptr));
    SB200_REQUIRE(a->xf && a->pre_x && a->h_out[0] && (a->layers == 1 || a->h_out[1]));
    SB200_REQUIRE(a->h && a->c && a->h_before && a->c_before && a->mean && a->log_var && a->action && a->pd);
    SB200_REQUIRE(a->obs_host == nullptr || a->ld_obs == a->D);
    SB200_REQUIRE(a->action_host == nullptr || a->pd_host != nullptr);
    SB200_REQUIRE((a->h_before_host == nullptr) == (a->c_before_host == nullptr));
    for (int k = 0; k < a->layers; ++k) SB200_REQUIRE(a->ih[k] && a->whh[k] && a->bhh[k] && a->ih[k]->dims[1] == 4 * a->H);
    // no LayerNorm in the recurrent policy's head, input projections or CNN stem
    if (sb200_mlp_has_ln(a->head) || (stem && sb200_mlp_has_ln(a->fc))) return SB200_ERR_UNSUPPORTED;
    for (int k = 0; k < a->layers; ++k)
        if (sb200_mlp_has_ln(a->ih[k])) return SB200_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    const int N = a->N, D = a->D, H = a->H, L = a->layers, A = a->head->dims[a->head->n_layers];
    const size_t cells = (size_t)L * N * H * sizeof(float);
    const sb200_zfilter nozf = {nullptr, 1e-5f};
    float* save[SB200_MAX_LAYERS] = {nullptr, nullptr, nullptr, nullptr};
    int64_t lds[SB200_MAX_LAYERS] = {0, 0, 0, 0};
    int rc = SB200_OK;
    if (stem) {
        const size_t frame_bytes = (size_t)a->frame_c * a->frame_h * a->frame_w;
        if (a->frames_host != nullptr)
            SB200_CUDA(cudaMemcpyAsync(a->frames, a->frames_host, (size_t)N * frame_bytes, cudaMemcpyHostToDevice, st));
        SB200_CUDA(cudaMemcpyAsync(a->h_before, a->h, cells, cudaMemcpyDeviceToDevice, st));
        SB200_CUDA(cudaMemcpyAsync(a->c_before, a->c, cells, cudaMemcpyDeviceToDevice, st));
        rc = sb200_conv_forward_f32(1, a->frames, 1, N, a->frame_c, a->frame_h, a->frame_w, a->conv_w1, a->conv_b1,
                                    1.0 / 255.0, a->a1, stream);
        if (rc != SB200_OK) return rc;
        rc = sb200_conv_forward_f32(2, a->a1, 0, N, 16, H1, W1, a->conv_w2, a->conv_b2, 1.0, a->a2, stream);
        if (rc != SB200_OK) return rc;
        const sb200_rows fin = {a->a2, nullptr, a->fc->dims[0], N, 0, nullptr, 0, nullptr, 0};
        save[0] = a->xf;
        lds[0] = a->ld_xf;
        rc = sb200_mlp_forward_f32(a->fc, &nozf, &fin, save, lds, stream);
    } else {
        if (a->obs_host != nullptr)
            SB200_CUDA(cudaMemcpyAsync(a->obs, a->obs_host, (size_t)N * D * sizeof(float), cudaMemcpyHostToDevice, st));
        SB200_CUDA(cudaMemcpyAsync(a->h_before, a->h, cells, cudaMemcpyDeviceToDevice, st));
        SB200_CUDA(cudaMemcpyAsync(a->c_before, a->c, cells, cudaMemcpyDeviceToDevice, st));
        rc = sb200_rows_zfilter_f32(a->obs, D, a->ld_obs, N, 1, D, a->zf.stats, (double)a->zf.eps, a->xf, a->ld_xf, stream);
    }
    if (rc != SB200_OK) return rc;
    sb200_rows in = {a->xf, nullptr, a->ld_xf, N, 0, nullptr, 0, nullptr, 0};
    for (int k = 0; k < L; ++k) {
        save[0] = a->pre_x;
        lds[0] = 4 * H;
        rc = sb200_mlp_forward_f32(a->ih[k], &nozf, &in, save, lds, stream);
        if (rc != SB200_OK) return rc;
        float* ho = a->h_out[(L - 1 - k) & 1];
        float* hk = a->h + (size_t)k * N * H;
        float* ck = a->c + (size_t)k * N * H;
        rc = sb200_lstm_forward_f32(a->pre_x, a->whh[k], a->bhh[k], hk, ck, H, N, 1, H, a->ldh, ho, nullptr, nullptr, nullptr,
                                    hk, ck, stream);
        if (rc != SB200_OK) return rc;
        in.x = ho;
        in.ldx = a->ldh;
    }
    save[0] = nullptr;
    lds[0] = 0;
    save[a->head->n_layers - 1] = a->mean;
    lds[a->head->n_layers - 1] = A;
    rc = sb200_mlp_forward_f32(a->head, &nozf, &in, save, lds, stream);
    if (rc != SB200_OK) return rc;
    if (a->fifo_state != nullptr)
        rc = sb200_ppo_sample_assign_f32(a->mean, A, a->log_var, a->log_noise, a->eps, N, A, a->deterministic, a->seed,
                                         a->step_counter, a->action, a->pd, a->stage_pos, a->stage_act, a->stage_pd,
                                         a->n_step, a->fifo_state, a->dest, stream);
    else
        rc = sb200_ppo_sample_f32(a->mean, A, a->log_var, a->log_noise, a->eps, N, A, a->deterministic, a->seed,
                                  a->step_counter, a->action, a->pd, a->stage_pos, a->stage_act, a->stage_pd, a->n_step,
                                  stream);
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

extern "C" int sb200_ppo_window_step_rnn_f32(const float* obs_next_host, const float* obs_reset_host,
                                             const float* reward_host, const float* done_host, float* obs_next,
                                             float* obs_reset, float* reward, float* done, int N, int n_step, int stride,
                                             int obs_dim, int layers, int H, const float* h, const float* c, int A,
                                             int* stage_pos, float* stage_obs, float* stage_act, float* stage_pd,
                                             float* stage_rew, float* stage_done, int* dest_scratch, void* fifo_state,
                                             float* r_obs, float* r_act, float* r_pd, float* r_rew, float* r_done,
                                             uint64_t* step_counter, int slots_assigned, int force_wide, void* stream) {
    SB200_REQUIRE(obs_next && obs_reset && reward && done && h && c && stage_pos && stage_obs && stage_act && stage_pd);
    SB200_REQUIRE(stage_rew && stage_done && dest_scratch && fifo_state && r_obs && r_act && r_pd && r_rew && r_done);
    SB200_REQUIRE(N >= 1 && n_step >= 1 && stride >= 1 && obs_dim >= 1 && layers >= 1 && H >= 1 && A >= 1);
    const bool host = obs_reset_host != nullptr;
    SB200_REQUIRE(host ? (obs_next_host && reward_host && done_host) : (!obs_next_host && !reward_host && !done_host));
    const int D = obs_dim + 2 * layers * H;
    const size_t smem = (size_t)2 * D * sizeof(float);
    const bool wide = smem > 48 * 1024 || force_wide;            // rows too wide to stage in shared memory
    cudaStream_t st = (cudaStream_t)stream;
    const float* next = obs_next;
    if (host) {
        const size_t row_bytes = (size_t)N * obs_dim * sizeof(float);
        SB200_CUDA(cudaMemcpyAsync(obs_reset, obs_reset_host, row_bytes, cudaMemcpyHostToDevice, st));
        if (obs_next_host != obs_reset_host)
            SB200_CUDA(cudaMemcpyAsync(obs_next, obs_next_host, row_bytes, cudaMemcpyHostToDevice, st));
        else
            next = obs_reset;
        SB200_CUDA(cudaMemcpyAsync(reward, reward_host, (size_t)N * sizeof(float), cudaMemcpyHostToDevice, st));
        SB200_CUDA(cudaMemcpyAsync(done, done_host, (size_t)N * sizeof(float), cudaMemcpyHostToDevice, st));
    }
    if (!slots_assigned)
        ppo_window_slots_kernel<<<1, 1024, 0, st>>>(N, n_step, stage_pos, dest_scratch, (FifoState*)fifo_state,
                                                    (unsigned long long*)step_counter);
    if (wide)
        ppo_window_commit_rnn_wide_kernel<<<N, 128, 0, st>>>(next, obs_reset, reward, done, N, n_step, stride, obs_dim, layers,
                                                             H, h, c, A, stage_pos, stage_obs, stage_act, stage_pd, stage_rew,
                                                             stage_done, dest_scratch, r_obs, r_act, r_pd, r_rew, r_done);
    else
        ppo_window_commit_rnn_kernel<<<N, 128, smem, st>>>(next, obs_reset, reward, done, N, n_step, stride, obs_dim, layers,
                                                           H, h, c, A, stage_pos, stage_obs, stage_act, stage_pd, stage_rew,
                                                           stage_done, dest_scratch, r_obs, r_act, r_pd, r_rew, r_done);
    return sb200_launch_status(slots_assigned ? 1 : 2);
}
