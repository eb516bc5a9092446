// Classic-control tasks as batched, device-resident environments: CartPole-v1 and Pendulum-v1 (gym's classic_control
// dynamics; the float64 statement every kernel here follows is tests/classic_ref.py).  One thread per actor steps the
// physics; state, episode step, episode index, observations, reward and done all live in HBM, so a step is one launch
// at fixed addresses (CUDA-graph capturable).  Done actors auto-reset inside the same launch.
//
// Reset states are Philox4x32-10 words keyed by (env seed ^ CLASSIC_KEY, episode index, actor): word k gives the uniform
// u_k = (word >> 8) * 2^-24 and the component lo_k + width_k * u_k, rounded after the product and after the sum.  The
// seed therefore fixes every episode's start for a given action stream.
#include "common.cuh"
#include "rollout_dev.cuh"

namespace {

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

template <class T>
int classic_reset(int N, uint64_t seed, float* state, float* obs, int* ep_step, int* episode, cudaStream_t st) {
    classic_reset_kernel<T><<<(N + CT - 1) / CT, CT, 0, st>>>(N, (unsigned long long)seed, state, obs, ep_step, episode);
    return sb200_launch_status();
}

template <class T>
int classic_step(const float* action, int N, int max_steps, uint64_t seed, float* state, float* obs, int* ep_step,
                 int* episode, float* obs_next, float* reward, float* done, const sb200_windows* w, cudaStream_t st) {
    const int grid = (N + CT - 1) / CT;
    if (w == nullptr) {
        classic_step_kernel<T><<<grid, CT, 0, st>>>(action, N, max_steps, (unsigned long long)seed, state, obs, ep_step,
                                                    episode, obs_next, reward, done);
    } else {
        SB200_REQUIRE(w->N == N && w->D == T::D && w->A == T::A);
        classic_window_step_kernel<T><<<grid, CT, 0, st>>>(
            action, N, max_steps, (unsigned long long)seed, state, obs, ep_step, episode, obs_next, reward, done,
            w->n_step, w->stride, w->stage_pos, w->stage_obs, w->stage_act, w->stage_pd, w->stage_rew, w->stage_done,
            w->dest, w->r_obs, w->r_act, w->r_pd, w->r_rew, w->r_done);
    }
    return sb200_launch_status();
}

}  // namespace

extern "C" int sb200_classic_env_reset_f32(int task, int N, uint64_t seed, float* state, float* obs, int* ep_step,
                                           int* episode, void* stream) {
    SB200_REQUIRE(N >= 1 && state && obs && ep_step && episode);
    cudaStream_t st = (cudaStream_t)stream;
    switch (task) {
        case SB200_CLASSIC_CARTPOLE: return classic_reset<CartPole>(N, seed, state, obs, ep_step, episode, st);
        case SB200_CLASSIC_PENDULUM: return classic_reset<Pendulum>(N, seed, state, obs, ep_step, episode, st);
        default: return SB200_ERR_ARG;
    }
}

static int classic_step_any(int task, const float* action, int N, int max_steps, uint64_t seed, float* state,
                            float* obs, int* ep_step, int* episode, float* obs_next, float* reward, float* done,
                            const sb200_windows* w, void* stream) {
    SB200_REQUIRE(N >= 1 && action && state && obs && ep_step && episode && obs_next && reward && done);
    cudaStream_t st = (cudaStream_t)stream;
    switch (task) {
        case SB200_CLASSIC_CARTPOLE:
            return classic_step<CartPole>(action, N, max_steps, seed, state, obs, ep_step, episode, obs_next, reward, done,
                                          w, st);
        case SB200_CLASSIC_PENDULUM:
            return classic_step<Pendulum>(action, N, max_steps, seed, state, obs, ep_step, episode, obs_next, reward, done,
                                          w, st);
        default: return SB200_ERR_ARG;
    }
}

extern "C" int sb200_classic_env_step_f32(int task, const float* action, int N, int max_steps, uint64_t seed,
                                          float* state, float* obs, int* ep_step, int* episode, float* obs_next,
                                          float* reward, float* done, void* stream) {
    return classic_step_any(task, action, N, max_steps, seed, state, obs, ep_step, episode, obs_next, reward, done,
                            nullptr, stream);
}

extern "C" int sb200_classic_env_window_step_f32(int task, const float* action, int N, int max_steps, uint64_t seed,
                                                 float* state, float* obs, int* ep_step, int* episode, float* obs_next,
                                                 float* reward, float* done, const sb200_windows* windows,
                                                 void* stream) {
    SB200_REQUIRE(windows_ok(windows));
    return classic_step_any(task, action, N, max_steps, seed, state, obs, ep_step, episode, obs_next, reward, done,
                            windows, stream);
}
