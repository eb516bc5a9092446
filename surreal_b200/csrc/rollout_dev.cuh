// Device-side building blocks shared by the per-step rollout kernels (rollout.cu), the device envs (env.cu) and the
// persistent rollout kernels (rollout_fused.cu, rollout_rnn.cu): FIFO control block, replay-slot assignment, the
// sampling and env formulas, per-actor window commit.
#pragma once
#include "common.cuh"

namespace {

// ------------------------------------------------------------------------------------------------
// ExpSenderWrapperMultiStepMovingWindowWithInfo._step (exp_sender_wrapper.py:209-228), batched.
// Slot assignment (one block, ordered): detect the deques that reach n_step with this step's append and give
// them FIFO slots in (step, actor) order with drop-oldest at `capacity` (fifo_replay.py:27).  It depends only
// on the deque lengths, so it can run before the environment has stepped (fused into the sampling kernel).
struct FifoState {
    int head;        // physical index of the oldest window
    int count;       // windows currently queued
    int capacity;    // memory_size + 3
    int dropped;     // windows silently dropped so far (diagnostic)
    long long total_in;
    long long total_out;
    unsigned int ticket;   // last-block ticket of the fused sampling kernel (self-resetting)
    int pad_;
};

// Host check of a staging descriptor: every buffer present and the shape sane (step_counter may be NULL).
inline bool windows_ok(const sb200_windows* w) {
    return w != nullptr && w->N >= 1 && w->n_step >= 1 && w->stride >= 1 && w->D >= 1 && w->A >= 1 && w->stage_pos &&
           w->stage_obs && w->stage_act && w->stage_pd && w->stage_rew && w->stage_done && w->dest && w->fifo_state &&
           w->r_obs && w->r_act && w->r_pd && w->r_rew && w->r_done;
}

// Host check of a persistent rollout's env: the synthetic env, stepping the rollout's N actors with its D / A.
inline bool rollout_env_ok(const sb200_ppo_rollout* a) {
    const sb200_env* e = a->env;
    return e != nullptr && e->kind == SB200_ENV_SYNTH && e->N == a->N && e->D == a->D && e->A == a->A;
}

constexpr int SLOT_NONE = -1;      // deque not full after this step
constexpr int SLOT_DROPPED = -2;   // window completes but falls straight out of the deque(maxlen)

// dest[i] <- physical slot | SLOT_NONE | SLOT_DROPPED; advances the queue.  Called by all threads of ONE block.
__device__ void assign_window_slots(int N, int n_step, const int* __restrict__ stage_pos, int* __restrict__ dest,
                                    FifoState* fifo) {
    __shared__ int warp_tot[32];
    __shared__ int warp_excl[32];
    __shared__ int chunk_total;
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    int base = 0;                                  // windows completed by actors before this chunk
    for (int i0 = 0; i0 < N; i0 += nt) {
        const int i = i0 + tid;
        const int flag = (i < N && stage_pos[i] + 1 == n_step) ? 1 : 0;
        int incl = flag;                           // inclusive scan inside the warp (actor order)
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const int w = (lane < nw) ? warp_tot[lane] : 0;
            int wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += t;
            }
            warp_excl[lane] = wi - w;
            if (lane == 31) chunk_total = wi;
        }
        __syncthreads();
        if (i < N) dest[i] = flag ? (base + warp_excl[warp] + incl - flag) : SLOT_NONE;
        base += chunk_total;
        __syncthreads();
    }
    // translate ranks into physical slots; advance the queue
    const int K = base;
    const int cap = fifo->capacity;
    const int head = fifo->head, count = fifo->count;
    __syncthreads();
    for (int i = tid; i < N; i += nt) {
        const int r = dest[i];
        if (r >= 0) {
            // more arrivals than the deque holds: the earliest of THIS step fall out immediately
            dest[i] = (K > cap && r < K - cap) ? SLOT_DROPPED : (int)(((long long)head + count + r) % cap);
        }
    }
    if (tid == 0) {
        int nc = count + K, nh = head, dr = 0;
        if (nc > cap) {                       // deque(maxlen): the oldest entries fall out
            dr = nc - cap;
            nh = (int)(((long long)head + dr) % cap);
            nc = cap;
        }
        fifo->head = nh;
        fifo->count = nc;
        fifo->dropped += dr;
        fifo->total_in += K;
    }
}

__device__ unsigned int* fifo_ticket(FifoState* fifo) { return &fifo->ticket; }

// ------------------------------------------------------------------------------------------------
// Per-element formulas of PPO sampling and of the synthetic env, used by the per-step kernels (rollout.cu, env.cu) and
// by the persistent rollout (rollout_fused.cu), whose results must agree bit for bit.  Each formula is one expression, so
// every caller gets the same FMA contraction.

// PPOAgent.act (ppo_agent.py:138-149): std = exp(log_var) * scale, scale = exp(noise_i) (1 without per-actor noise)
__device__ __forceinline__ float ppo_std(float log_var, float scale) { return __fmul_rn(expf(log_var), scale); }

// action = clip(z * std + mean, -1, 1) with z ~ N(0, 1), or clip(mean) when deterministic
__device__ __forceinline__ float ppo_action(float mu, float sd, float z, int deterministic) {
    float a = mu;
    if (!deterministic) a = __fadd_rn(__fmul_rn(z, sd), mu);
    return fminf(fmaxf(a, -1.0f), 1.0f);
}

// The episode ends when its step count `ep` (this step included) reaches max_steps (MaxStepWrapper, env/wrapper.py:142-163)
__device__ __forceinline__ bool env_done(int ep, int max_steps) { return (max_steps > 0) && (ep >= max_steps); }

// successor s' = tanh(Ws s + Wa a) + 0.01 xi, acc = Ws s + Wa a, xi = box_muller(r.x, r.y).x of env_noise
__device__ __forceinline__ float env_successor(float acc, float xi) { return tanhf(acc) + 0.01f * xi; }

// reward -|s|^2 / D + 0.1 xi', sq = |s|^2, xi' = box_muller(r.x, r.y).y of env_noise at d = 0
__device__ __forceinline__ float env_reward(float sq, int D, float xi) { return -sq / (float)D + 0.1f * xi; }

// state component d of the next episode, drawn ~ N(0, 1) when the step ends the episode
__device__ __forceinline__ float env_reset_draw(const Philox4& r) { return box_muller(r.z, r.w).x; }

__device__ __forceinline__ void copy_floats(float* __restrict__ dst, const float* __restrict__ src, int count, int g,
                                            int G) {
    if (((count & 3) == 0) && ((((uintptr_t)dst) | ((uintptr_t)src)) & 15) == 0) {
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* d4 = reinterpret_cast<float4*>(dst);
        for (int k = g; k < (count >> 2); k += G) d4[k] = s4[k];
    } else {
        for (int k = g; k < count; k += G) dst[k] = src[k];
    }
}

// Commit of one actor's step by a group of G threads (g = index inside the group).  `pos` points at the actor's
// deque length (global or shared memory), `slot` is the record slot its window ships to when it completes with this
// step (SLOT_NONE: not complete, SLOT_DROPPED: complete but not stored).  Appends (reward, done) at
// deque position p and obs_next at p+1; if the window completed, copies it into its replay slot and pops
// `stride` items; if the episode ended, clears the deque (exp_sender_wrapper.py:204-207) and seeds position 0
// with the reset observation.  `barrier` is executed by EVERY thread of the barrier's group (valid or not): block-wide by
// default; a caller whose commit group is one warp and whose other warps are busy elsewhere passes WarpBarrier.
struct BlockBarrier {
    __device__ __forceinline__ void operator()() const { __syncthreads(); }
};
struct WarpBarrier {
    __device__ __forceinline__ void operator()() const { __syncwarp(); }
};
// `next_row` / `reset_row` are read as next_row[d], d < D: float pointers by default, or -- given explicitly as Row -- a
// type that assembles the row on the fly (rollout.cu's CellRow).
template <class T>
struct NoDeduce {
    using type = T;
};
template <class Barrier = BlockBarrier, class Row = const float* __restrict__>
__device__ void commit_actor(bool valid, int i, int g, int G, typename NoDeduce<Row>::type next_row,
                             typename NoDeduce<Row>::type reset_row, float rew, float dn, int n_step, int stride, int D,
                             int A, int* __restrict__ pos, int slot, float* __restrict__ stage_obs,
                             float* __restrict__ stage_act, float* __restrict__ stage_pd,
                             float* __restrict__ stage_rew, float* __restrict__ stage_done,
                             float* __restrict__ r_obs, float* __restrict__ r_act,
                             float* __restrict__ r_pd, float* __restrict__ r_rew, float* __restrict__ r_done,
                             Barrier barrier = Barrier()) {
    const long long ii = valid ? i : 0;
    const int p = valid ? *pos : 0;
    float* so = stage_obs + ii * (n_step + 1) * D;
    float* sa = stage_act + ii * n_step * A;
    float* sp = stage_pd + ii * n_step * 2 * A;
    float* sr = stage_rew + ii * n_step;
    float* sd = stage_done + ii * n_step;
    if (valid) {
        for (int d = g; d < D; d += G) so[(long long)(p + 1) * D + d] = next_row[d];
        if (g == 0) {
            sr[p] = rew;
            sd[p] = dn;
        }
    }
    barrier();
    int len = p + 1;
    if (!valid) slot = SLOT_NONE;
    const bool complete = (slot != SLOT_NONE);               // len == n_step
    if (slot >= 0) {                                         // ship the window
        copy_floats(r_obs + (long long)slot * (n_step + 1) * D, so, (n_step + 1) * D, g, G);
        copy_floats(r_act + (long long)slot * n_step * A, sa, n_step * A, g, G);
        copy_floats(r_pd + (long long)slot * n_step * 2 * A, sp, n_step * 2 * A, g, G);
        copy_floats(r_rew + (long long)slot * n_step, sr, n_step, g, G);
        copy_floats(r_done + (long long)slot * n_step, sd, n_step, g, G);
    }
    barrier();
    const int pop = min(stride, n_step);                     // uniform: every completing deque holds n_step items
    const int keep = n_step - pop;
    if (keep > 0) {                                          // overlapping windows: slide the deque down
        for (int k0 = 0; k0 < (keep + 1) * D; k0 += G) {
            const int k = k0 + g;
            const bool on = complete && k < (keep + 1) * D;
            float v = 0.f;
            if (on) v = so[(long long)pop * D + k];
            barrier();
            if (on) so[k] = v;
            barrier();
        }
        for (int k0 = 0; k0 < keep * 2 * A; k0 += G) {
            const int k = k0 + g;
            float va = 0.f, vp = 0.f;
            if (complete && k < keep * A) va = sa[(long long)pop * A + k];
            if (complete && k < keep * 2 * A) vp = sp[(long long)pop * 2 * A + k];
            barrier();
            if (complete && k < keep * A) sa[k] = va;
            if (complete && k < keep * 2 * A) sp[k] = vp;
            barrier();
        }
        for (int k0 = 0; k0 < keep; k0 += G) {
            const int k = k0 + g;
            float vr = 0.f, vd = 0.f;
            if (complete && k < keep) { vr = sr[pop + k]; vd = sd[pop + k]; }
            barrier();
            if (complete && k < keep) { sr[k] = vr; sd[k] = vd; }
            barrier();
        }
    } else if (complete) {
        for (int d = g; d < D; d += G) so[d] = next_row[d];                 // obs_next -> next window's first obs
    }
    if (complete) len = keep;
    barrier();
    if (valid && dn > 0.5f) {                                // episode over: deque cleared, new episode's first obs
        for (int d = g; d < D; d += G) so[d] = reset_row[d];
        len = 0;
    }
    if (valid && g == 0) *pos = len;
}

}  // namespace
