// Device-resident envs behind one descriptor (sb200_env) and one step entry: the synthetic env of the benchmark configs,
// its pixel form, and the classic-control tasks CartPole-v1 and Pendulum-v1.  Every buffer lives in HBM at a fixed address,
// so a step is a fixed launch sequence (CUDA-graph capturable), and done actors auto-reset inside it.
#include "common.cuh"
#include "rollout_dev.cuh"

namespace {

constexpr int RT = 256;        // threads per block of the synthetic env

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
        const Philox4 r = env_noise(seed, ctr, i, d);
        const float2 g = box_muller(r.x, r.y);
        const float nxt = env_successor(acc, g.x);
        const bool dn = env_done(ep_step[i] + 1, max_steps);
        const float st = dn ? env_reset_draw(r) : nxt;
        obs_next[(long long)i * D + d] = nxt;
        state[(long long)i * D + d] = st;
        if (s_n != nullptr) {
            s_n[idx] = nxt;
            s_z[idx] = st;
        }
        if (d == 0) {
            const float rw = env_reward(s_q[q], D, g.y);
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
            ep_step[i] = env_done(t, max_steps) ? 0 : t;
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

// ------------------------------------------------------------------------------------------------
// Synthetic PIXEL environment of BASELINE configs[3] (SURVEY §8d cfg 4): every step each actor observes a fresh frame of
// uniform random bytes (Philox keyed by (seed, step, actor, word)), reward = -mean(a^2) + 0.1 xi, done at the episode cap.
// Frames are written as 32-bit words (4 pixels each); `state` = what the actor observes next (a reset frame where done),
// `obs_next` = the true successor.
__global__ void __launch_bounds__(256) synth_pixel_env_kernel(unsigned int* __restrict__ state, const float* __restrict__ action, int N,
                                                              int words, int A, int max_steps, int* __restrict__ ep_step,
                                                              unsigned long long seed, const unsigned long long* __restrict__ step_ctr,
                                                              unsigned int* __restrict__ obs_next, float* __restrict__ reward,
                                                              float* __restrict__ done) {
    const int i = blockIdx.y;
    const unsigned long long ctr = (step_ctr != nullptr) ? *step_ctr : 0ull;
    const int t = ep_step[i] + 1;
    const bool dn = (max_steps > 0) && (t >= max_steps);
    const int w4 = words / 4;
    for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < w4; g += gridDim.x * blockDim.x) {
        const Philox4 r = philox4x32_10(seed ^ 0x2545F4914F6CDD1Dull, ctr, ((unsigned long long)i << 24) | (unsigned long long)g);
        uint4 nx = make_uint4(r.x, r.y, r.z, r.w);
        reinterpret_cast<uint4*>(obs_next + (long long)i * words)[g] = nx;
        if (dn) {
            const Philox4 z = philox4x32_10(seed ^ 0x9E3779B97F4A7C15ull, ctr, ((unsigned long long)i << 24) | (unsigned long long)g);
            nx = make_uint4(z.x, z.y, z.z, z.w);
        }
        reinterpret_cast<uint4*>(state + (long long)i * words)[g] = nx;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        float s = 0.0f;
        for (int j = 0; j < A; ++j) s += action[(long long)i * A + j] * action[(long long)i * A + j];
        const Philox4 r = philox4x32_10(seed ^ 0x5851F42D4C957F2Dull, ctr, ((unsigned long long)i << 24) | 0xFFFFFFull);
        reward[i] = -s / (float)A + 0.1f * box_muller(r.x, r.y).x;
        done[i] = dn ? 1.0f : 0.0f;
    }
}
// ep_step update must happen after every block has read it: separate tiny kernel
__global__ void synth_pixel_env_tick_kernel(int N, int max_steps, int* __restrict__ ep_step) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int t = ep_step[i] + 1;
    ep_step[i] = ((max_steps > 0) && (t >= max_steps)) ? 0 : t;
}

// ------------------------------------------------------------------------------------------------
// Classic-control tasks as batched, device-resident environments: CartPole-v1 and Pendulum-v1 (gym's classic_control
// dynamics; the float64 statement every kernel here follows is tests/classic_ref.py).  One thread per actor steps the
// physics; state, episode step, episode index, observations, reward and done all live in HBM, so a step is one launch
// at fixed addresses (CUDA-graph capturable).  Done actors auto-reset inside the same launch.
//
// Reset states are Philox4x32-10 words keyed by (env seed ^ CLASSIC_KEY, episode index, actor): word k gives the uniform
// u_k = (word >> 8) * 2^-24 and the component lo_k + width_k * u_k, rounded after the product and after the sum.  The
// seed therefore fixes every episode's start for a given action stream.
constexpr int CT = 128;        // actors per block, one thread each
constexpr int CG = 8;          // threads per actor in the fused window commit
// The synthetic envs, the action noise and the parameter noise key on other constants: no two streams share a key.
constexpr unsigned long long CLASSIC_KEY = 0xD6E8FEB86659FD93ull;

__device__ __forceinline__ Philox4 reset_words(unsigned long long seed, int episode, int actor) {
    return philox4x32_10(seed ^ CLASSIC_KEY, (unsigned long long)(unsigned int)episode, (unsigned long long)actor);
}

__device__ __forceinline__ float reset_value(unsigned int word, float lo, float width) {
    const float u = (float)(word >> 8) * 5.9604644775390625e-08f;          // exact: 24 bits times 2^-24
    return __fadd_rn(__fmul_rn(width, u), lo);
}

// CartPole-v1.  State = observation = (x, x_dot, theta, theta_dot); action index 1 (a[1] > a[0] of a one-hot row) pushes
// right.  Explicit Euler in gym's order; terminal outside |x| <= 2.4 or |theta| <= 12 deg (strict comparisons against
// the fp32 values of the thresholds, since the state is fp32).  Reward 1 on every step.
struct CartPole {
    static constexpr int S = 4, D = 4, A = 2;
    __device__ static void reset(const Philox4& r, float* s) {
        s[0] = reset_value(r.x, -0.05f, 0.1f);
        s[1] = reset_value(r.y, -0.05f, 0.1f);
        s[2] = reset_value(r.z, -0.05f, 0.1f);
        s[3] = reset_value(r.w, -0.05f, 0.1f);
    }
    __device__ static void observe(const float* s, float* o) {
#pragma unroll
        for (int k = 0; k < 4; ++k) o[k] = s[k];
    }
    __device__ static void step(float* s, const float* a, float& rew, bool& term) {
        const float force = (a[1] > a[0]) ? 10.0f : -10.0f;
        float sn, cs;
        sincosf(s[2], &sn, &cs);
        const float temp = (force + 0.05f * s[3] * s[3] * sn) / 1.1f;
        const float thacc = (9.8f * sn - cs * temp) / (0.5f * (4.0f / 3.0f - 0.1f * cs * cs / 1.1f));
        const float xacc = temp - 0.05f * thacc * cs / 1.1f;
        s[0] = s[0] + 0.02f * s[1];
        s[1] = s[1] + 0.02f * xacc;
        s[2] = s[2] + 0.02f * s[3];
        s[3] = s[3] + 0.02f * thacc;
        const float thr = 0.20943951023931953f;                            // 12 * 2 pi / 360
        term = s[0] < -2.4f || s[0] > 2.4f || s[2] < -thr || s[2] > thr;
        rew = 1.0f;
    }
};

// Pendulum-v1.  State (theta, theta_dot), observation (cos theta, sin theta, theta_dot); torque u = 2 clip(a, -1, 1).
// reward = -(norm(theta)^2 + 0.1 theta_dot^2 + 0.001 u^2) on the state before the update, norm(x) = ((x + pi) mod 2 pi)
// - pi; theta_dot' = clip(theta_dot + (15 sin theta + 3 u) 0.05, -8, 8), then theta' = theta + theta_dot' 0.05.  Never
// terminal: only the episode cap ends an episode.
struct Pendulum {
    static constexpr int S = 2, D = 3, A = 1;
    __device__ static void reset(const Philox4& r, float* s) {
        s[0] = reset_value(r.x, -3.14159265358979f, 6.28318530717959f);
        s[1] = reset_value(r.y, -1.0f, 2.0f);
    }
    __device__ static void observe(const float* s, float* o) {
        sincosf(s[0], &o[1], &o[0]);
        o[2] = s[1];
    }
    __device__ static float norm(float x) {
        float m = fmodf(x + 3.14159265358979f, 6.28318530717959f);
        if (m < 0.0f) m += 6.28318530717959f;                               // Python's mod: the sign of the divisor
        return m - 3.14159265358979f;
    }
    __device__ static void step(float* s, const float* a, float& rew, bool& term) {
        const float u = 2.0f * fminf(fmaxf(a[0], -1.0f), 1.0f);
        const float th = s[0], thd = s[1];
        const float n = norm(th);
        rew = -(n * n + 0.1f * thd * thd + 0.001f * u * u);
        const float nthd = fminf(fmaxf(thd + (15.0f * sinf(th) + 3.0f * u) * 0.05f, -8.0f), 8.0f);
        s[0] = th + nthd * 0.05f;
        s[1] = nthd;
        term = false;
    }
};

// One actor's step: physics, the episode cap (env_done, MaxStepWrapper), auto-reset of done actors with the next
// episode index.  Writes the true successor to obs_next and what the actor observes next to obs; n_row / z_row / rew_out
// / dn_out (fused commit, optional) receive the same rows and scalars.
template <class T>
__device__ __forceinline__ void classic_actor(int i, const float* __restrict__ action, int max_steps,
                                              unsigned long long seed, float* __restrict__ state,
                                              float* __restrict__ obs, int* __restrict__ ep_step,
                                              int* __restrict__ episode, float* __restrict__ obs_next,
                                              float* __restrict__ reward, float* __restrict__ done, float* n_row,
                                              float* z_row, float* rew_out, float* dn_out) {
    float s[T::S], a[T::A], o[T::D];
#pragma unroll
    for (int k = 0; k < T::S; ++k) s[k] = state[(long long)i * T::S + k];
#pragma unroll
    for (int k = 0; k < T::A; ++k) a[k] = action[(long long)i * T::A + k];
    float rew;
    bool term;
    T::step(s, a, rew, term);
    T::observe(s, o);
#pragma unroll
    for (int k = 0; k < T::D; ++k) obs_next[(long long)i * T::D + k] = o[k];
    if (n_row != nullptr) {
#pragma unroll
        for (int k = 0; k < T::D; ++k) n_row[k] = o[k];
    }
    const int t = ep_step[i] + 1;
    const bool dn = term || env_done(t, max_steps);
    if (dn) {
        const int e = episode[i] + 1;
        episode[i] = e;
        T::reset(reset_words(seed, e, i), s);
        T::observe(s, o);
    }
    ep_step[i] = dn ? 0 : t;
#pragma unroll
    for (int k = 0; k < T::S; ++k) state[(long long)i * T::S + k] = s[k];
#pragma unroll
    for (int k = 0; k < T::D; ++k) obs[(long long)i * T::D + k] = o[k];
    reward[i] = rew;
    done[i] = dn ? 1.0f : 0.0f;
    if (z_row != nullptr) {
#pragma unroll
        for (int k = 0; k < T::D; ++k) z_row[k] = o[k];
        *rew_out = rew;
        *dn_out = dn ? 1.0f : 0.0f;
    }
}

template <class T>
__global__ void __launch_bounds__(CT) classic_reset_kernel(int N, unsigned long long seed, float* __restrict__ state,
                                                           float* __restrict__ obs, int* __restrict__ ep_step,
                                                           int* __restrict__ episode) {
    const int i = blockIdx.x * CT + threadIdx.x;
    if (i >= N) return;
    float s[T::S], o[T::D];
    T::reset(reset_words(seed, 0, i), s);
    T::observe(s, o);
#pragma unroll
    for (int k = 0; k < T::S; ++k) state[(long long)i * T::S + k] = s[k];
#pragma unroll
    for (int k = 0; k < T::D; ++k) obs[(long long)i * T::D + k] = o[k];
    ep_step[i] = 0;
    episode[i] = 0;
}

template <class T>
__global__ void __launch_bounds__(CT) classic_step_kernel(const float* __restrict__ action, int N, int max_steps,
                                                          unsigned long long seed, float* __restrict__ state,
                                                          float* __restrict__ obs, int* __restrict__ ep_step,
                                                          int* __restrict__ episode, float* __restrict__ obs_next,
                                                          float* __restrict__ reward, float* __restrict__ done) {
    const int i = blockIdx.x * CT + threadIdx.x;
    if (i < N)
        classic_actor<T>(i, action, max_steps, seed, state, obs, ep_step, episode, obs_next, reward, done, nullptr,
                         nullptr, nullptr, nullptr);
}

// Step fused with the commit half of ppo_window_step: the block's successor and reset rows stay in shared memory, then
// groups of CG threads commit the block's actors through commit_actor, as ppo_window_commit_kernel does.  The groups of a
// warp run the same barrier sequence (it depends only on n_step, stride, D, A and CG), so a warp barrier suffices.
template <class T>
__global__ void __launch_bounds__(CT) classic_window_step_kernel(
    const float* __restrict__ action, int N, int max_steps, unsigned long long seed, float* __restrict__ state,
    float* __restrict__ obs, int* __restrict__ ep_step, int* __restrict__ episode, float* __restrict__ obs_next,
    float* __restrict__ reward, float* __restrict__ done, int n_step, int stride, int* __restrict__ stage_pos,
    float* __restrict__ stage_obs, float* __restrict__ stage_act, float* __restrict__ stage_pd,
    float* __restrict__ stage_rew, float* __restrict__ stage_done, const int* __restrict__ dest,
    float* __restrict__ r_obs, float* __restrict__ r_act, float* __restrict__ r_pd, float* __restrict__ r_rew,
    float* __restrict__ r_done) {
    __shared__ float s_n[CT][T::D], s_z[CT][T::D], s_rew[CT], s_dn[CT];
    const int a0 = blockIdx.x * CT;
    const int i = a0 + threadIdx.x;
    if (i < N)
        classic_actor<T>(i, action, max_steps, seed, state, obs, ep_step, episode, obs_next, reward, done,
                         s_n[threadIdx.x], s_z[threadIdx.x], &s_rew[threadIdx.x], &s_dn[threadIdx.x]);
    __syncthreads();
    const int g = threadIdx.x % CG;
    for (int q = threadIdx.x / CG; q < CT; q += CT / CG) {
        const int j = a0 + q;
        const bool valid = j < N;
        commit_actor<WarpBarrier>(valid, j, g, CG, s_n[q], s_z[q], valid ? s_rew[q] : 0.0f, valid ? s_dn[q] : 0.0f,
                                  n_step, stride, T::D, T::A, stage_pos + min(j, N - 1), valid ? dest[j] : SLOT_NONE,
                                  stage_obs, stage_act, stage_pd, stage_rew, stage_done, r_obs, r_act, r_pd, r_rew,
                                  r_done);
    }
}

// ------------------------------------------------------------------------------------------------
// Host side: one launcher per env family, each checking the descriptor fields its kind reads before it launches.
bool env_smem_ok(int D, int A, bool fused) {
    return (size_t)(4 * (D + A) + (fused ? 8 * D : 0)) * sizeof(float) <= 40 * 1024;
}

int synth_step(const sb200_env* e, const float* action, const sb200_windows* w, cudaStream_t st) {
    SB200_REQUIRE(e->WsT && e->WaT && e->D >= 1 && e->A >= 1 && env_smem_ok(e->D, e->A, w != nullptr));
    const int N = e->N, D = e->D, A = e->A;
    float* state = (float*)e->state;
    float* obs_next = (float*)e->obs_next;
    const unsigned long long* ctr = (const unsigned long long*)e->step_counter;
    if (w == nullptr) {
        const size_t smem = (size_t)(4 * (D + A)) * sizeof(float);
        synth_env_step_kernel<<<(N + 3) / 4, RT, smem, st>>>(state, action, e->WsT, e->WaT, N, D, A, e->max_steps,
                                                             e->ep_step, (unsigned long long)e->seed, ctr, obs_next,
                                                             e->reward, e->done);
    } else {
        const size_t smem = (size_t)(4 * (D + A) + 8 * D) * sizeof(float);
        synth_env_window_step_kernel<<<(N + 3) / 4, RT, smem, st>>>(
            state, action, e->WsT, e->WaT, N, D, A, e->max_steps, e->ep_step, (unsigned long long)e->seed, ctr, obs_next,
            e->reward, e->done, w->n_step, w->stride, w->stage_pos, w->stage_obs, w->stage_act, w->stage_pd, w->stage_rew,
            w->stage_done, w->dest, w->r_obs, w->r_act, w->r_pd, w->r_rew, w->r_done);
    }
    return sb200_launch_status();
}

// D = the frame's 32-bit words; the Philox counter of a word packs (actor << 24 | word / 4)
int pixel_step(const sb200_env* e, const float* action, cudaStream_t st) {
    const int N = e->N, words = e->D;
    SB200_REQUIRE(e->A >= 1 && words >= 4 && words % 4 == 0 && words / 4 < (1 << 24) && N < (1 << 24));
    dim3 grid((unsigned)((words / 4 + 255) / 256 < 8 ? (words / 4 + 255) / 256 : 8), (unsigned)N);
    synth_pixel_env_kernel<<<grid, 256, 0, st>>>((unsigned int*)e->state, action, N, words, e->A, e->max_steps, e->ep_step,
                                                 (unsigned long long)e->seed, (const unsigned long long*)e->step_counter,
                                                 (unsigned int*)e->obs_next, e->reward, e->done);
    synth_pixel_env_tick_kernel<<<(N + 255) / 256, 256, 0, st>>>(N, e->max_steps, e->ep_step);
    return sb200_launch_status(2);
}

template <class T>
bool classic_ok(const sb200_env* e) {
    return e->D == T::D && e->A == T::A && e->obs && e->episode;
}

template <class T>
int classic_reset(const sb200_env* e, cudaStream_t st) {
    SB200_REQUIRE(classic_ok<T>(e));
    classic_reset_kernel<T><<<(e->N + CT - 1) / CT, CT, 0, st>>>(e->N, (unsigned long long)e->seed, (float*)e->state,
                                                                 e->obs, e->ep_step, e->episode);
    return sb200_launch_status();
}

template <class T>
int classic_step(const sb200_env* e, const float* action, const sb200_windows* w, cudaStream_t st) {
    SB200_REQUIRE(classic_ok<T>(e));
    const int N = e->N, grid = (N + CT - 1) / CT;
    const unsigned long long seed = e->seed;
    float* state = (float*)e->state;
    float* obs_next = (float*)e->obs_next;
    if (w == nullptr) {
        classic_step_kernel<T><<<grid, CT, 0, st>>>(action, N, e->max_steps, seed, state, e->obs, e->ep_step, e->episode,
                                                    obs_next, e->reward, e->done);
    } else {
        classic_window_step_kernel<T><<<grid, CT, 0, st>>>(
            action, N, e->max_steps, seed, state, e->obs, e->ep_step, e->episode, obs_next, e->reward, e->done, w->n_step,
            w->stride, w->stage_pos, w->stage_obs, w->stage_act, w->stage_pd, w->stage_rew, w->stage_done, w->dest, w->r_obs,
            w->r_act, w->r_pd, w->r_rew, w->r_done);
    }
    return sb200_launch_status();
}

}  // namespace

extern "C" int sb200_env_step_f32(const sb200_env* e, const float* action, const sb200_windows* windows, void* stream) {
    SB200_REQUIRE(e != nullptr && action != nullptr && e->N >= 1);
    SB200_REQUIRE(e->state && e->ep_step && e->obs_next && e->reward && e->done);
    SB200_REQUIRE(windows == nullptr ||
                  (windows_ok(windows) && windows->N == e->N && windows->D == e->D && windows->A == e->A));
    cudaStream_t st = (cudaStream_t)stream;
    switch (e->kind) {
        case SB200_ENV_SYNTH: return synth_step(e, action, windows, st);
        case SB200_ENV_SYNTH_PIXEL: return windows != nullptr ? SB200_ERR_UNSUPPORTED : pixel_step(e, action, st);
        case SB200_ENV_CARTPOLE: return classic_step<CartPole>(e, action, windows, st);
        case SB200_ENV_PENDULUM: return classic_step<Pendulum>(e, action, windows, st);
        default: return SB200_ERR_ARG;
    }
}

extern "C" int sb200_env_reset_f32(const sb200_env* e, void* stream) {
    SB200_REQUIRE(e != nullptr && e->N >= 1 && e->state && e->ep_step);
    cudaStream_t st = (cudaStream_t)stream;
    switch (e->kind) {
        case SB200_ENV_CARTPOLE: return classic_reset<CartPole>(e, st);
        case SB200_ENV_PENDULUM: return classic_reset<Pendulum>(e, st);
        default: return SB200_ERR_ARG;
    }
}
