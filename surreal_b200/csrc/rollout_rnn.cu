// Persistent rollout of the recurrent (LSTM) PPO policy: T env steps of ALL co-located actors in ONE launch.
//
// The per-step chain of the LSTM policy (sb200_ppo_act_f32 + the synthetic env step + sb200_ppo_window_step_f32)
// is about 9 launches per step, and every step moves each actor's [L][H] cells through HBM (copied to h_before /
// c_before, read and rewritten by every layer, read again by the window commit) while each launch re-fetches its
// weights from L2.  Actors are independent, so the loop over time moves inside the kernel:
//   * a CTA owns R = 8 actors for the whole chunk; their env state, observations and LSTM cells stay in shared memory
//     from the first step to the last;
//   * per step: z-filter -> per layer one GEMM over the gate columns (thread = gate column, all R actors in registers)
//     and the cell update (lstm_dev.cuh, shared with the learner's lstm_fwd_kernel) -> actor head (thread = output
//     column; narrow layers split k and sum the slices in fixed order) -> sampling -> synthetic env step -> window
//     staging by one warp per actor (commit_actor of rollout_dev.cuh) into the per-actor outbox that
//     sb200_ppo_rollout_commit_f32 turns into FIFO records in (step, actor) order;
//   * weights are streamed through L1/L2 (read-only loads): the chain's largest launch, the LSTM cell kernel, reads
//     W_hh once per ACTOR and step, this kernel once per R actors and step.
// Sampling, env arithmetic and Philox keys are those of the chain (rollout_dev.cuh, common.cuh): the action noise is
// keyed by the step counter of the step, the env noise by that counter + 1, as the chain's sampling launch advances the
// shared counter before the env step reads it.
#include <algorithm>

#include "common.cuh"
#include "lstm_dev.cuh"
#include "rollout_dev.cuh"

namespace {

constexpr int RR_THREADS = 512;           // 16 warps
constexpr int RR_MAX_H = RR_THREADS / 4;  // one thread per gate column
constexpr int RR_MAX_D = 256;             // env observation width
constexpr int RR_MAX_WIDTH = 512;         // head layer widths
constexpr int RR_MAX_A = 32;              // one warp lane per action dim
constexpr int RR_R = 8;                   // actors per CTA (16 spills registers in the gate GEMM)

struct RrParams {
    // LSTM
    int L, H;
    const float* Wih[SB200_MAX_RNN_LAYERS];   // [in][ldih] (W_ih^T)
    const float* bih[SB200_MAX_RNN_LAYERS];
    int ldih[SB200_MAX_RNN_LAYERS];
    const float* Whh[SB200_MAX_RNN_LAYERS];   // [H][4H] (W_hh^T)
    const float* bhh[SB200_MAX_RNN_LAYERS];
    float* h;                                 // [L][N][H]
    float* c;
    float* h_before;
    float* c_before;
    // head
    int nh;
    int hdims[SB200_MAX_LAYERS + 1];
    const float* hW[SB200_MAX_LAYERS];
    const float* hb[SB200_MAX_LAYERS];
    int hldw[SB200_MAX_LAYERS];
    int hact[SB200_MAX_LAYERS];
    // sampling / env
    int Do, A, Drec;
    const float* zf;
    float zf_eps;
    const float* log_var;
    const float* log_noise;
    unsigned long long agent_seed;
    int deterministic;
    float* state;
    const float* WsT;
    const float* WaT;
    int* ep_step;
    int max_steps;
    unsigned long long env_seed;
    float* action;
    float* pd;
    float* obs_next;
    float* reward;
    float* done;
    // staging / outbox
    int* stage_pos;
    float* stage_obs;
    float* stage_act;
    float* stage_pd;
    float* stage_rew;
    float* stage_done;
    float* o_obs;
    float* o_act;
    float* o_pd;
    float* o_rew;
    float* o_done;
    int* ev_step;
    int* ev_count;
    int Wout;
    int N, n_step, stride, T;
    const unsigned long long* step_ctr;
    // shared-memory plan (float offsets)
    int ldx, ldh, ldact;
    int oS0, oS1, oNx, oX, oHc, oCc, oG, oAct0, oAct1, oPart, oZf, oSd, oAc, oQ;
};

// A staged record row [obs (Do) | h_0 .. h_{L-1} | c_0 .. c_{L-1}] (utils.rnn_cell_layout) of the CTA's actor r, read
// from its observation row and the cells in shared memory ([L][R][ldh]).
struct SmemCellRow {
    const float* obs;
    const float* h;
    const float* c;
    int Do, LH, H, Rld;                     // Rld = R * ldh: floats between two layers' cells
    __device__ __forceinline__ float operator[](int d) const {
        if (d < Do) return obs[d];
        int e = d - Do;
        const float* cells = h;
        if (e >= LH) {
            e -= LH;
            cells = c;
        }
        const int k = e / H;
        return cells[k * Rld + (e - k * H)];
    }
};

// acc[r] += sum_{k0 <= k < k1} in[r][k] * W[k][n] in k order, for the CTA's R rows
template <int R>
__device__ __forceinline__ void rr_dot(const float* __restrict__ in, int ldin, int k0, int k1, const float* __restrict__ W,
                                       int ldw, int n, float (&acc)[R]) {
    const float* wp = W + n;
    int k = k0;
    for (; k + 4 <= k1 && (k & 3) == 0; k += 4) {
        const float w0 = __ldg(wp + (long long)(k + 0) * ldw), w1 = __ldg(wp + (long long)(k + 1) * ldw);
        const float w2 = __ldg(wp + (long long)(k + 2) * ldw), w3 = __ldg(wp + (long long)(k + 3) * ldw);
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const float4 x = *reinterpret_cast<const float4*>(in + r * ldin + k);
            acc[r] = fmaf(x.x, w0, acc[r]);
            acc[r] = fmaf(x.y, w1, acc[r]);
            acc[r] = fmaf(x.z, w2, acc[r]);
            acc[r] = fmaf(x.w, w3, acc[r]);
        }
    }
    for (; k < k1; ++k) {
        const float w = __ldg(wp + (long long)k * ldw);
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r] = fmaf(in[r * ldin + k], w, acc[r]);
    }
}

// out[r][n] = act(in[r] . W[:, n] + b[n]) for the R rows.  Wide layers: one output column per thread.  Narrow layers
// (< RR_THREADS / 2 columns): S = RR_THREADS / ncols_pad threads per column, each over one k slice; the slice sums meet
// in `part` and are added in slice order.  Ends with a block barrier.
template <int R>
__device__ void rr_dense(const float* __restrict__ in, int ldin, int K, const float* __restrict__ W, int ldw,
                         const float* __restrict__ b, int act, int ncols, float* __restrict__ out, int ldout,
                         float* __restrict__ part) {
    const int tid = threadIdx.x;
    const int npad = (ncols + 31) & ~31;
    if (2 * npad > RR_THREADS) {
        for (int n = tid; n < ncols; n += RR_THREADS) {
            float acc[R];
#pragma unroll
            for (int r = 0; r < R; ++r) acc[r] = 0.0f;
            rr_dot<R>(in, ldin, 0, K, W, ldw, n, acc);
            const float bn = __ldg(b + n);
#pragma unroll
            for (int r = 0; r < R; ++r) out[r * ldout + n] = apply_act(acc[r] + bn, act);
        }
        __syncthreads();
        return;
    }
    const int S = RR_THREADS / npad;
    const int kc = (((K + S - 1) / S) + 3) & ~3;          // k slice, a multiple of 4
    const int s = tid / npad, n = tid - s * npad;
    if (s < S && n < ncols) {
        float acc[R];
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r] = 0.0f;
        rr_dot<R>(in, ldin, min(K, s * kc), min(K, (s + 1) * kc), W, ldw, n, acc);
#pragma unroll
        for (int r = 0; r < R; ++r) part[(s * R + r) * npad + n] = acc[r];
    }
    __syncthreads();
    for (int e = tid; e < R * ncols; e += RR_THREADS) {
        const int r = e / ncols, nn = e - r * ncols;
        float v = 0.0f;
        for (int q = 0; q < S; ++q) v += part[(q * R + r) * npad + nn];
        out[r * ldout + nn] = apply_act(v + __ldg(b + nn), act);
    }
    __syncthreads();
}

__global__ void __launch_bounds__(RR_THREADS, 1) ppo_rollout_rnn_kernel(const __grid_constant__ RrParams p) {
    constexpr int R = RR_R;
    extern __shared__ __align__(16) float smem[];
    __shared__ int s_pos[R], s_ep[R], s_cnt[R];
    __shared__ float s_rew[R], s_dn[R];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int Do = p.Do, A = p.A, H = p.H, L = p.L, G4 = 4 * H;
    const long long i0 = (long long)blockIdx.x * R;
    float* Hc = smem + p.oHc;                            // [L][R][ldh] cells
    float* Cc = smem + p.oCc;
    float* Zm = smem + p.oZf;
    float* Zs = Zm + Do;
    float* Sd = smem + p.oSd;                            // [R][A] std rows
    float* Ac = smem + p.oAc;                            // [R][A] actions
    float* Qs = smem + p.oQ;                             // [R] |s|^2
    float* X = smem + p.oX;
    float* Gt = smem + p.oG;                             // [R][4H] gate pre-activations
    float* Nx = smem + p.oNx;                            // [R][Do] successor
    float* Part = smem + p.oPart;

    // ---- one-time loads
    for (int e = tid; e < R * Do; e += RR_THREADS) {
        const int r = e / Do, d = e - r * Do;
        const long long i = i0 + r;
        smem[p.oS0 + e] = (i < p.N) ? p.state[i * Do + d] : 0.0f;
    }
    for (int e = tid; e < L * R * H; e += RR_THREADS) {
        const int k = e / (R * H), rem = e - k * R * H, r = rem / H, j = rem - r * H;
        const long long i = i0 + r;
        const bool v = i < p.N;
        Hc[(k * R + r) * p.ldh + j] = v ? p.h[((long long)k * p.N + i) * H + j] : 0.0f;
        Cc[(k * R + r) * p.ldh + j] = v ? p.c[((long long)k * p.N + i) * H + j] : 0.0f;
    }
    if (p.zf != nullptr) {
        const float cnt = p.zf[2 * Do];
        for (int d = tid; d < Do; d += RR_THREADS) {
            const float mean = p.zf[d] / cnt;
            const float var = p.zf[Do + d] / cnt - mean * mean;
            Zm[d] = mean;
            Zs[d] = fmaxf(sqrtf(var), p.zf_eps);
        }
    }
    for (int e = tid; e < R * A; e += RR_THREADS) {
        const int r = e / A, j = e - r * A;
        const long long i = i0 + r;
        const float sc = (i < p.N && p.log_noise != nullptr) ? expf(p.log_noise[i]) : 1.0f;
        Sd[e] = ppo_std(p.log_var[j], sc);
    }
    if (tid < R) {
        const long long i = i0 + tid;
        s_pos[tid] = (i < p.N) ? p.stage_pos[i] : 0;
        s_ep[tid] = (i < p.N) ? p.ep_step[i] : 0;
        s_cnt[tid] = 0;
    }
    const unsigned long long ctr0 = (p.step_ctr != nullptr) ? *p.step_ctr : 0ull;
    __syncthreads();

    for (int t = 0; t < p.T; ++t) {
        const bool final_step = (t == p.T - 1);
        const unsigned long long ctr = ctr0 + (unsigned long long)t;
        float* Scur = smem + ((t & 1) ? p.oS1 : p.oS0);
        float* Snext = smem + ((t & 1) ? p.oS0 : p.oS1);
        // ---- input rows (z-filter), |s|^2 of each actor, and on the last step the cells before it
        for (int e = tid; e < R * Do; e += RR_THREADS) {
            const int r = e / Do, d = e - r * Do;
            float v = Scur[e];
            if (p.zf != nullptr) v = fminf(fmaxf((v - Zm[d]) / Zs[d], -5.0f), 5.0f);
            X[r * p.ldx + d] = (i0 + r < p.N) ? v : 0.0f;
        }
        for (int r = warp; r < R; r += RR_THREADS / 32) {
            float q = 0.0f;
            for (int d = lane; d < Do; d += 32) q += Scur[r * Do + d] * Scur[r * Do + d];
            q = warp_sum(q);
            if (lane == 0) Qs[r] = q;
        }
        if (final_step) {
            for (int e = tid; e < L * R * H; e += RR_THREADS) {
                const int k = e / (R * H), rem = e - k * R * H, r = rem / H, j = rem - r * H;
                const long long i = i0 + r;
                if (i < p.N) {
                    p.h_before[((long long)k * p.N + i) * H + j] = Hc[(k * R + r) * p.ldh + j];
                    p.c_before[((long long)k * p.N + i) * H + j] = Cc[(k * R + r) * p.ldh + j];
                }
            }
        }
        __syncthreads();
        // ---- LSTM layers: gate column j of all R actors per thread, then the cell update
        for (int k = 0; k < L; ++k) {
            const float* in = (k == 0) ? X : Hc + (k - 1) * R * p.ldh;
            const int ldin = (k == 0) ? p.ldx : p.ldh, Kin = (k == 0) ? Do : H;
            const float* hk = Hc + k * R * p.ldh;
            for (int j = tid; j < G4; j += RR_THREADS) {
                float acc[R];
#pragma unroll
                for (int r = 0; r < R; ++r) acc[r] = 0.0f;
                rr_dot<R>(in, ldin, 0, Kin, p.Wih[k], p.ldih[k], j, acc);
                const float bi = __ldg(p.bih[k] + j);
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    Gt[r * G4 + j] = acc[r] + bi;                 // pre_x = x . W_ih^T + b_ih
                    acc[r] = 0.0f;
                }
                rr_dot<R>(hk, p.ldh, 0, H, p.Whh[k], G4, j, acc);
                const float bh = __ldg(p.bhh[k] + j);
#pragma unroll
                for (int r = 0; r < R; ++r) Gt[r * G4 + j] = lstm_gate_pre(Gt[r * G4 + j], acc[r], bh);
            }
            __syncthreads();
            for (int e = tid; e < R * H; e += RR_THREADS) {
                const int r = e / H, j = e - r * H;
                const float* g = Gt + r * G4;
                LstmGates q;
                float c = Cc[(k * R + r) * p.ldh + j];
                const float h = lstm_cell(g[j], g[H + j], g[2 * H + j], g[3 * H + j], c, q);
                Cc[(k * R + r) * p.ldh + j] = c;
                Hc[(k * R + r) * p.ldh + j] = h;
            }
            __syncthreads();
        }
        // ---- actor head
        const float* in = Hc + (L - 1) * R * p.ldh;
        int ldin = p.ldh;
        float* outb = smem + p.oAct0;
        for (int l = 0; l < p.nh; ++l) {
            rr_dense<R>(in, ldin, p.hdims[l], p.hW[l], p.hldw[l], p.hb[l], p.hact[l], p.hdims[l + 1], outb, p.ldact, Part);
            in = outb;
            ldin = p.ldact;
            outb = (outb == smem + p.oAct0) ? smem + p.oAct1 : smem + p.oAct0;
        }
        const float* Mu = in;                                  // [R][ldact] policy mean
        // ---- sampling (sample_one of rollout.cu)
        for (int e = tid; e < R * A; e += RR_THREADS) {
            const int r = e / A, j = e - r * A;
            const long long i = i0 + r;
            const float mu = Mu[r * p.ldact + j], sd = Sd[e];
            const float z = p.deterministic ? 0.0f : action_noise1(p.agent_seed, ctr, (unsigned long long)i, j);
            const float a = ppo_action(mu, sd, z, p.deterministic);
            Ac[e] = a;
            if (i < p.N) {
                const int pos = s_pos[r];
                p.stage_act[(i * p.n_step + pos) * A + j] = a;
                p.stage_pd[(i * p.n_step + pos) * 2 * A + j] = mu;
                p.stage_pd[(i * p.n_step + pos) * 2 * A + A + j] = sd;
                if (final_step) {
                    p.action[i * A + j] = a;
                    p.pd[i * 2 * A + j] = mu;
                    p.pd[i * 2 * A + A + j] = sd;
                }
            }
        }
        __syncthreads();
        // ---- env step (synth_env_block of rollout.cu); its noise is keyed by the counter the sampling advanced
        for (int e = tid; e < R * Do; e += RR_THREADS) {
            const int r = e / Do, d = e - r * Do;
            const long long i = i0 + r;
            const float* s = Scur + r * Do;
            float acc = 0.0f;
#pragma unroll 8
            for (int k = 0; k < Do; ++k) acc = fmaf(__ldg(p.WsT + (long long)k * Do + d), s[k], acc);
#pragma unroll 4
            for (int k = 0; k < A; ++k) acc = fmaf(__ldg(p.WaT + (long long)k * Do + d), Ac[r * A + k], acc);
            const Philox4 rn = env_noise(p.env_seed, ctr + 1ull, (unsigned long long)i, d);
            const float2 g = box_muller(rn.x, rn.y);
            const float nxt = env_successor(acc, g.x);
            const bool dn = env_done(s_ep[r] + 1, p.max_steps);
            Nx[e] = nxt;
            Snext[e] = dn ? env_reset_draw(rn) : nxt;
            if (d == 0) {
                s_rew[r] = env_reward(Qs[r], Do, g.y);
                s_dn[r] = dn ? 1.0f : 0.0f;
            }
            if (final_step && i < p.N) {
                p.obs_next[i * Do + d] = nxt;
                if (d == 0) {
                    p.reward[i] = env_reward(Qs[r], Do, g.y);
                    p.done[i] = dn ? 1.0f : 0.0f;
                }
            }
        }
        __syncthreads();
        // ---- window staging: one warp per actor
        for (int r = warp; r < R; r += RR_THREADS / 32) {
            const long long i = i0 + r;
            const bool valid = i < p.N;
            const int pos = s_pos[r];
            int slot = SLOT_NONE;
            if (lane == 0) {
                const int ep = s_ep[r] + 1;
                s_ep[r] = env_done(ep, p.max_steps) ? 0 : ep;
                if (valid && pos + 1 == p.n_step) {
                    const int w = s_cnt[r];
                    if (w < p.Wout) {
                        slot = (int)(i * p.Wout + w);
                        p.ev_step[slot] = t;
                        s_cnt[r] = w + 1;
                    } else {
                        slot = SLOT_DROPPED;
                    }
                }
            }
            slot = __shfl_sync(0xffffffffu, slot, 0);
            const SmemCellRow next = {Nx + r * Do, Hc + r * p.ldh, Cc + r * p.ldh, Do, L * H, H, R * p.ldh};
            const SmemCellRow reset = {Snext + r * Do, Hc + r * p.ldh, Cc + r * p.ldh, Do, L * H, H, R * p.ldh};
            commit_actor<WarpBarrier, SmemCellRow>(valid, (int)(valid ? i : 0), lane, 32, next, reset, s_rew[r], s_dn[r],
                                                   p.n_step, p.stride, p.Drec, A, &s_pos[r], slot, p.stage_obs,
                                                   p.stage_act, p.stage_pd, p.stage_rew, p.stage_done, p.o_obs, p.o_act,
                                                   p.o_pd, p.o_rew, p.o_done, WarpBarrier());
        }
        __syncthreads();
    }

    // ---- write-back
    const float* Sfin = smem + ((p.T & 1) ? p.oS1 : p.oS0);
    for (int e = tid; e < R * Do; e += RR_THREADS) {
        const int r = e / Do, d = e - r * Do;
        if (i0 + r < p.N) p.state[(i0 + r) * Do + d] = Sfin[e];
    }
    for (int e = tid; e < L * R * H; e += RR_THREADS) {
        const int k = e / (R * H), rem = e - k * R * H, r = rem / H, j = rem - r * H;
        const long long i = i0 + r;
        if (i < p.N) {
            p.h[((long long)k * p.N + i) * H + j] = Hc[(k * R + r) * p.ldh + j];
            p.c[((long long)k * p.N + i) * H + j] = Cc[(k * R + r) * p.ldh + j];
        }
    }
    if (tid < R && i0 + tid < p.N) {
        p.stage_pos[i0 + tid] = s_pos[tid];
        p.ep_step[i0 + tid] = s_ep[tid];
        p.ev_count[i0 + tid] = s_cnt[tid];
    }
}

// Shapes the kernel takes: low-dim LSTM stem (1..SB200_MAX_RNN_LAYERS layers, H <= 128 so that each gate column has a
// thread), env observation width D <= 256, a head H -> ... -> A of 1..SB200_MAX_LAYERS layers no wider than 512, A <= 32,
// no LayerNorm and no aux input anywhere.
bool rr_shape_ok(const sb200_ppo_rollout_rnn* a) {
    if (a == nullptr || a->base == nullptr || a->base->net == nullptr) return false;
    const sb200_mlp* head = a->base->net;
    const int L = a->layers, H = a->H, D = a->base->D, A = a->base->A;
    if (L < 1 || L > SB200_MAX_RNN_LAYERS || H < 1 || H > RR_MAX_H || D < 1 || D > RR_MAX_D || A < 1 || A > RR_MAX_A)
        return false;
    if (head->n_layers < 1 || head->n_layers > SB200_MAX_LAYERS || head->aux_layer >= 0 || sb200_mlp_has_ln(head))
        return false;
    if (head->dims[0] != H || head->dims[head->n_layers] != A) return false;
    for (int l = 0; l < head->n_layers; ++l)
        if (head->dims[l + 1] > RR_MAX_WIDTH || head->ldw[l] < head->dims[l + 1]) return false;
    for (int k = 0; k < L; ++k) {
        const sb200_mlp* ih = a->ih[k];
        if (ih == nullptr || ih->n_layers != 1 || ih->aux_layer >= 0 || sb200_mlp_has_ln(ih)) return false;
        if (ih->dims[0] != (k == 0 ? D : H) || ih->dims[1] != 4 * H || ih->ldw[0] < 4 * H || ih->act[0] != SB200_ACT_NONE)
            return false;
    }
    return true;
}

int rr_round4(int v) { return (v + 3) & ~3; }

// Shared-memory plan -> byte count (p may be NULL).
size_t rr_plan(const sb200_ppo_rollout_rnn* a, RrParams* p) {
    constexpr int R = RR_R;
    const sb200_mlp* head = a->base->net;
    const int L = a->layers, H = a->H, D = a->base->D, A = a->base->A;
    int wmax = 4;
    for (int l = 0; l < head->n_layers; ++l) wmax = std::max(wmax, head->dims[l + 1]);
    const int ldx = rr_round4(D), ldh = rr_round4(H), ldact = rr_round4(wmax);
    long long off = 0;
    auto take = [&](long long n) { const long long o = off; off += (n + 3) / 4 * 4; return (int)o; };
    const int oS0 = take((long long)R * D), oS1 = take((long long)R * D), oNx = take((long long)R * D);
    const int oX = take((long long)R * ldx), oHc = take((long long)L * R * ldh), oCc = take((long long)L * R * ldh);
    const int oG = take((long long)R * 4 * H), oAct0 = take((long long)R * ldact), oAct1 = take((long long)R * ldact);
    const int oPart = take((long long)R * RR_THREADS), oZf = take(2LL * D), oSd = take((long long)R * A);
    const int oAc = take((long long)R * A), oQ = take(R);
    if (p != nullptr) {
        p->ldx = ldx; p->ldh = ldh; p->ldact = ldact;
        p->oS0 = oS0; p->oS1 = oS1; p->oNx = oNx; p->oX = oX; p->oHc = oHc; p->oCc = oCc; p->oG = oG;
        p->oAct0 = oAct0; p->oAct1 = oAct1; p->oPart = oPart; p->oZf = oZf; p->oSd = oSd; p->oAc = oAc; p->oQ = oQ;
    }
    return (size_t)off * sizeof(float);
}

constexpr size_t RR_SMEM_MAX = 200 * 1024;

cudaError_t rr_set_smem() {
    return cudaFuncSetAttribute(ppo_rollout_rnn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RR_SMEM_MAX);
}

int rr_sm_count(int* sms) {
    int dev = 0;
    SB200_CUDA(cudaGetDevice(&dev));
    SB200_CUDA(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
    return SB200_OK;
}

bool rr_windows_ok(const sb200_ppo_rollout_rnn* a) {
    const sb200_windows* w = a->base->windows;
    return windows_ok(w) && w->N == a->base->N && w->A == a->base->A && w->D == a->base->D + 2 * a->layers * a->H;
}

}  // namespace

extern "C" int sb200_ppo_rollout_rnn_supported(const sb200_ppo_rollout_rnn* a) {
    return (rr_shape_ok(a) && rr_plan(a, nullptr) <= RR_SMEM_MAX) ? 1 : 0;
}

extern "C" int sb200_ppo_rollout_rnn_f32(const sb200_ppo_rollout_rnn* a, void* stream) {
    SB200_REQUIRE(a != nullptr && a->base != nullptr);
    if (sb200_ppo_rollout_rnn_supported(a) != 1) return SB200_ERR_UNSUPPORTED;
    const sb200_ppo_rollout* b = a->base;
    SB200_REQUIRE(b->N >= 1 && b->T >= 1 && b->W >= 1 && rr_windows_ok(a) && rollout_env_ok(b));
    const sb200_env* e = b->env;
    SB200_REQUIRE(e->state && e->WsT && e->WaT && e->ep_step && b->action && b->pd && e->obs_next && e->reward && e->done);
    SB200_REQUIRE(b->log_var && b->o_obs && b->o_act && b->o_pd && b->o_rew && b->o_done && b->ev_step && b->ev_count);
    SB200_REQUIRE(a->h && a->c && a->h_before && a->c_before);
    RrParams p = {};
    p.L = a->layers;
    p.H = a->H;
    for (int k = 0; k < a->layers; ++k) {
        SB200_REQUIRE(a->ih[k]->W[0] && a->ih[k]->b[0] && a->whh[k] && a->bhh[k]);
        p.Wih[k] = a->ih[k]->W[0];
        p.bih[k] = a->ih[k]->b[0];
        p.ldih[k] = a->ih[k]->ldw[0];
        p.Whh[k] = a->whh[k];
        p.bhh[k] = a->bhh[k];
    }
    p.h = a->h;
    p.c = a->c;
    p.h_before = a->h_before;
    p.c_before = a->c_before;
    const sb200_mlp* head = b->net;
    p.nh = head->n_layers;
    for (int l = 0; l <= head->n_layers; ++l) p.hdims[l] = head->dims[l];
    for (int l = 0; l < head->n_layers; ++l) {
        SB200_REQUIRE(head->W[l] && head->b[l]);
        p.hW[l] = head->W[l];
        p.hb[l] = head->b[l];
        p.hldw[l] = head->ldw[l];
        p.hact[l] = head->act[l];
    }
    p.Do = b->D;
    p.A = b->A;
    p.Drec = b->D + 2 * a->layers * a->H;
    p.zf = b->zf_stats;
    p.zf_eps = b->zf_eps;
    p.log_var = b->log_var;
    p.log_noise = b->log_noise;
    p.agent_seed = b->agent_seed;
    p.deterministic = b->deterministic;
    p.state = (float*)e->state;
    p.WsT = e->WsT;
    p.WaT = e->WaT;
    p.ep_step = e->ep_step;
    p.max_steps = e->max_steps;
    p.env_seed = e->seed;
    p.action = b->action;
    p.pd = b->pd;
    p.obs_next = (float*)e->obs_next;
    p.reward = e->reward;
    p.done = e->done;
    const sb200_windows* w = b->windows;
    p.stage_pos = w->stage_pos;
    p.stage_obs = w->stage_obs;
    p.stage_act = w->stage_act;
    p.stage_pd = w->stage_pd;
    p.stage_rew = w->stage_rew;
    p.stage_done = w->stage_done;
    p.o_obs = b->o_obs;
    p.o_act = b->o_act;
    p.o_pd = b->o_pd;
    p.o_rew = b->o_rew;
    p.o_done = b->o_done;
    p.ev_step = b->ev_step;
    p.ev_count = b->ev_count;
    p.Wout = b->W;
    p.N = b->N;
    p.n_step = w->n_step;
    p.stride = w->stride;
    p.T = b->T;
    p.step_ctr = (const unsigned long long*)w->step_counter;
    const size_t smem = rr_plan(a, &p);
    const unsigned ctas = (unsigned)(((long long)b->N + RR_R - 1) / RR_R);
    SB200_CUDA(rr_set_smem());
    ppo_rollout_rnn_kernel<<<ctas, RR_THREADS, smem, (cudaStream_t)stream>>>(p);
    return sb200_launch_status();
}

extern "C" int sb200_ppo_rollout_rnn_footprint(const sb200_ppo_rollout_rnn* a, int* sms_out) {
    SB200_REQUIRE(a != nullptr && a->base != nullptr && sms_out != nullptr && a->base->N >= 1 && rollout_env_ok(a->base));
    *sms_out = 0;
    if (sb200_ppo_rollout_rnn_supported(a) != 1) return SB200_ERR_UNSUPPORTED;
    int sms = 0;
    int rc = rr_sm_count(&sms);
    if (rc != SB200_OK) return rc;
    const size_t smem = rr_plan(a, nullptr);
    int per_sm = 0;
    SB200_CUDA(rr_set_smem());
    SB200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ppo_rollout_rnn_kernel, RR_THREADS, smem));
    const long long ctas = ((long long)a->base->N + RR_R - 1) / RR_R;
    // one CTA per SM (launch bounds and the register budget), spread over the SMs: a grid of at most one CTA per SM holds
    // exactly `ctas` SMs for the whole chunk
    if (per_sm >= 1 && ctas <= sms) *sms_out = (int)ctas;
    return SB200_OK;
}
