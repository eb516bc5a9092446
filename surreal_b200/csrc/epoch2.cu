// Persistent learner kernel, second generation: BOTH optimisers of PPOLearner._optimize (policy epochs on the actor,
// value epochs on the critic; surreal/learner/ppo.py:194-353 losses and updates, 541-557 epoch loops and KL early stop)
// in ONE launch of one CTA per SM.
//
// What the first generation (one launch per optimiser, 64x64 tiles, a grid barrier after every layer; removed) taught:
// at 1024-row minibatches a layer is 64 tiles for 148 SMs and an epoch is 8-9 grid barriers, so the kernel spent its time
// waiting (114 us per epoch for 0.5 GFLOP).  Two observations restructure it:
//   * rows are independent through forward AND input-gradient: a CTA that owns a block of 16 rows runs
//     x -> h1 -> h2 -> head -> loss -> d2 -> d1 without talking to anybody, activations in shared memory.  With both
//     networks in one launch there are 2 x M/16 = 128 such items for 148 SMs -- one wave, no barrier inside.
//   * a thread that owns 16 rows x 4 columns of such a block reads every weight it needs exactly once, so the weight
//     matrix streams L2 -> registers (coalesced ld.global.cg.v4, software prefetch) and only the 16 activation rows
//     come from shared memory, as warp-wide broadcasts: 16 LDS.128 + 4 LDG.128 per 256 FMA.  The same micro-kernel does
//     the weight gradients (rows = 16 input features, reduction over the minibatch rows) and d1 (through a transposed
//     copy of W2 that the Adam phase keeps up to date).
// An epoch is now 4 grid barriers (5 in adapt mode, whose loss needs the batch-mean KL first):
//   P1  per (net, 16-row block): forward, head, KL partial, loss rows, d2, d1          -> barrier
//       gate: mean KL(ref || current) = post-step KL of the previous epoch, early stop (ppo.py:553-556)
//   P2  weight-gradient items (net, layer, 16 input features, row split z) -> slab z    -> barrier
//   P3  grad = sum of slabs in fixed order, squared-norm partials [+ peer all-reduce]   -> barrier
//   P4  clip by global norm + Adam (torch's arithmetic, optim_dev.cuh), W2^T refresh    -> barrier
// Everything is deterministic (static work assignment, fixed-order sums).  Buffers rewritten by other CTAs between
// barriers are read with ld.global.cg only.  Data-parallel exchanges (KL scalar, flat gradients) happen inside the
// kernel over NVLink peer memory with the protocol of peer_allreduce.cu (peer_dev.cuh).
#include <math.h>
#include <stddef.h>

#include <algorithm>

#include "common.cuh"
#include "gemm_tiles.cuh"
#include "optim_dev.cuh"
#include "peer_dev.cuh"
#include "ppo_loss_dev.cuh"

namespace {

using namespace peer_dev;
using optim_dev::OptWs;

constexpr int E2T = 512;              // threads per CTA (16 warps: the phases are latency-bound, 8 warps hid too little)
constexpr int E2W = E2T / 32;
constexpr int RB = 16;                // rows per block
constexpr int E2_MAX_OUT = 32;
constexpr int E2_SLOTS = 4 + E2_MAX_OUT;
constexpr int E2_MAX_G = 192;

struct Job {                          // one optimiser
    float* params;
    long long n_params;
    int w_off[3], b_off[3], ldw[3];
    int D, H1, H2, NO, act_out, extra_off;
    const float* x;
    long long ldx;
    int M;
    const float* zf;
    float zf_eps;
    float *x_in, *h1, *h2, *out, *d1, *d2, *dpre;
    int ld_x, ld_h1, ld_h2, ld_out;
    float *slabs, *grad, *m, *v;
    float* w2t;                       // [H2][ld_h1]: w2t[n][k] = W2[k][n]
    float* w3part;                    // [n_rb][(H2 + 1) * ldw3]: per-row-block dW3 | db3
    const double* lr;
    double weight_decay, clip_value;
    int clip_mode;
    OptWs* opt;
    float* norm_out;
    int mode;                         // 0 clip, 1 adapt, 2 value
    const float* actions; long long lda;
    const float* adv;
    const float* behave; long long ldb;
    const float* ref; long long ldr;
    const float* returns;
    const double* hyper;
    double eta, kl_target, stop_threshold;
    float* stats;
    int* stop;
    int epochs;
    double* kl_part;                  // [n_rb]
    double* loss_part;                // [n_rb][E2_SLOTS]
    double* sq_part;                  // [n_sq]
    double* kl_global;
    int n_rb;                         // row blocks
    int s;                            // row splits of the weight-gradient phase (slabs used)
    int rps;                          // rows per split
    sb200_par par;                    // world 1 (and no peers) when the job does not exchange
};

struct E2Params {
    Job job[2];
    int n_jobs;
    int n_sq;                         // chunks of the squared-norm sum (fixed per device: the sum does not depend on the grid)
    unsigned int* bar;
    unsigned long long* prof;         // [2][16] clock64 cycles per phase, accumulated by CTA 0 and the last CTA
    unsigned long long* cta_prof;     // [G][8] per-CTA cycles: 0 P1, 1 P2, 2 forward, 3 GEMMs of forward, 4 loss rows + d2, 5 d1 GEMM
    // shared-memory plan (float offsets)
    int o_xs, o_h1, o_h2, o_d2, o_out, o_dp, o_part, o_w3, o_rows;
    int ld_xs, ld_h1s, ld_h2s, ldp;
};

// Mean over the ranks of grad[lo, hi) (quads), read from every rank's slot in rank order (bit-identical on all ranks);
// returns this thread's share of the squared norm.  Peer loads are NVLink round trips (~3 us): a thread issues the loads of
// CH quads from EVERY rank before it touches the first result (the scalar loop this replaces paid one round trip per
// element: +0.9 ms per learn() at N = 2).  W = compile-time bound on the world size (slots past it re-read the last rank).
template <int W, int CH>
__device__ __forceinline__ double peer_sum_slice(const Job& p, long long lo, long long hi, unsigned int parity, float scale) {
    double sq = 0.0;
    const float* slot[W];
#pragma unroll
    for (int q = 0; q < W; ++q) slot[q] = slot_of(p.par, min(q, p.par.world - 1), parity);
    for (long long base = lo + (long long)threadIdx.x * 4; base < hi; base += (long long)E2T * 4 * CH) {
        float4 v[CH][W];
#pragma unroll
        for (int u = 0; u < CH; ++u) {
            const long long i = min(base + (long long)u * E2T * 4, hi - 4);
#pragma unroll
            for (int q = 0; q < W; ++q) v[u][q] = ld_sys4(slot[q] + i);
        }
#pragma unroll
        for (int u = 0; u < CH; ++u) {
            const long long i = base + (long long)u * E2T * 4;
            if (i < hi) {
                float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int q = 0; q < W; ++q)
                    if (q < p.par.world) {
                        a.x += v[u][q].x; a.y += v[u][q].y; a.z += v[u][q].z; a.w += v[u][q].w;
                    }
                a.x = __fmul_rn(a.x, scale); a.y = __fmul_rn(a.y, scale);
                a.z = __fmul_rn(a.z, scale); a.w = __fmul_rn(a.w, scale);
                *reinterpret_cast<float4*>(p.grad + i) = a;
                sq += (double)a.x * (double)a.x;
                sq += (double)a.y * (double)a.y;
                sq += (double)a.z * (double)a.z;
                sq += (double)a.w * (double)a.w;
            }
        }
    }
    return sq;
}

__device__ __forceinline__ void grid_bar(unsigned int* ctr, unsigned int& target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        target += gridDim.x;
        __threadfence();
        atomicAdd(ctr, 1u);
        for (;;) {
            unsigned int v;
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
            if ((int)(v - target) >= 0) break;
        }
        __threadfence();
    }
    __syncthreads();
}

__device__ __forceinline__ float4 zero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }

// ---- the micro-kernel: C[16][N] (+ optional column sums of W) = A[16][K] . W[K][N]
// A in shared memory ([RB][lda], zero padded to a multiple of 4 columns), W in global memory ([K][ldw], ldw % 4 == 0,
// padding columns zero).  512 threads = (column quad cq = tid & 63, row half rg = bit 6, k quarter kh = tid >> 7): an 8 x 4
// register tile per thread (32 accumulators, so that 16 warps fit the register file -- the 8-warp version with 8 x 8 tiles
// issued 17 % of the time: every phase here is bound by L2 / shared-memory latency, not by the FMA pipe).  W streams
// L2 -> L1 -> registers two k quads ahead (the two row halves of a column quad are different warps and share the line
// through L1, which the grid barrier's fence invalidates, so cached loads are coherent here); the k loop is unrolled by 3
// so that the rotation of the three operand sets is renaming, not copies.  The partial tiles of the four k quarters go to
// Part [4][RB + 1][ldp] (row RB: column sums); the caller sums them after a barrier.  One call covers 64 column quads
// (pass c40); wider layers take several passes.
__device__ __forceinline__ float4 ldw4(const float* p) {                 // L1-allocating load (see above)
    float4 r;
    asm volatile("ld.global.ca.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
// rb_gemm is a called function, not inlined: inlined at its six call sites it shared the 128 registers with the epoch
// loop's live state, so the kernel spilled (1300 B) and reloaded operands from local memory inside the k loop, and its
// code was several times larger.  Called, it spills 4 B and the kernel 612 B (-Xptxas -v); the epoch kernel at the
// bench shape runs 12 % faster on 68 SMs and 16 % faster on all 132 (H100 SXM, tools/prof_epoch2.py).
template <bool COLSUM>
__device__ __noinline__ void rb_gemm(const float* __restrict__ As, int lda, int K, const float* __restrict__ W, int ldw,
                                     float* __restrict__ Part, int ldp, int c40) {
    const int tid = threadIdx.x, cq = tid & 63, rg = (tid >> 6) & 1, kh = tid >> 7;
    const int Kp = (K + 3) & ~3;
    const int kq = (((Kp >> 2) + 3) >> 2) << 2;
    const int k_lo = kh * kq, k_hi = min(Kp, k_lo + kq);
    const int nq = ldw >> 2;
    const int c4 = c40 + cq;
    const bool on = c4 < nq;
    const float* Wc = W + (on ? c4 : 0) * 4;                   // a column quad past the layer reads quad 0 (never stored)
    const float* Ar = As + rg * 8 * lda;
    float2 acc[8][2];
#pragma unroll
    for (int r = 0; r < 8; ++r) acc[r][0] = acc[r][1] = make_float2(0.0f, 0.0f);
    float4 cs = zero4();
    float4 w[4], w1[4], w2[4];
    // no range predicates on the loads: a row index past K is clamped to K - 1 (A is zero there, so the product vanishes)
    auto loadq = [&](int k, float4 (&d)[4]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) d[i] = ldw4(Wc + (long long)max(min(k + i, K - 1), 0) * ldw);
    };
    loadq(k_lo, w);
    loadq(k_lo + 4, w1);
#pragma unroll 3
    for (int k = k_lo; k < k_hi; k += 4) {
        loadq(k + 8, w2);
        if (COLSUM) {
#pragma unroll
            for (int i = 0; i < 4; ++i)
                if (k + i < K) {
                    cs.x += w[i].x; cs.y += w[i].y; cs.z += w[i].z; cs.w += w[i].w;
                }
        }
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            const float4 a = *reinterpret_cast<const float4*>(Ar + r * lda + k);
            const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 aa = make_float2(av[i], av[i]);
                acc[r][0] = fma2(aa, make_float2(w[i].x, w[i].y), acc[r][0]);
                acc[r][1] = fma2(aa, make_float2(w[i].z, w[i].w), acc[r][1]);
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            w[i] = w1[i];
            w1[i] = w2[i];
        }
    }
    if (on) {
        float* pp = Part + (size_t)kh * (RB + 1) * ldp + c4 * 4;
#pragma unroll
        for (int r = 0; r < 8; ++r)
            *reinterpret_cast<float4*>(pp + (rg * 8 + r) * ldp) = make_float4(acc[r][0].x, acc[r][0].y, acc[r][1].x, acc[r][1].y);
        if (COLSUM && rg == 0) *reinterpret_cast<float4*>(pp + RB * ldp) = cs;
    }
}

__device__ __forceinline__ float4 part_sum(const float* Part, int ldp, int r, int c4) {
    const float* pp = Part + r * ldp + c4 * 4;
    const size_t st = (size_t)(RB + 1) * ldp;
    const float4 p0 = *reinterpret_cast<const float4*>(pp);
    const float4 p1 = *reinterpret_cast<const float4*>(pp + st);
    const float4 p2 = *reinterpret_cast<const float4*>(pp + 2 * st);
    const float4 p3 = *reinterpret_cast<const float4*>(pp + 3 * st);
    return make_float4((p0.x + p1.x) + (p2.x + p3.x), (p0.y + p1.y) + (p2.y + p3.y), (p0.z + p1.z) + (p2.z + p3.z),
                       (p0.w + p1.w) + (p2.w + p3.w));
}

struct Sm {
    float *xs, *h1s, *h2s, *d2s, *outs, *dps, *part, *w3s, *refs, *behs, *acts, *advs;
    int ld_xs, ld_h1s, ld_h2s, ldp;
};

// hidden layer: dst_s[r][c] = relu(A . W + b), zero in the padding columns; copied to the global activation rows
__device__ __forceinline__ void hidden_layer(const Sm& sm, const float* As, int lda, int K, const float* W, int ldw, const float* bias,
                                             int N, float* dst_s, int ld_s, float* dst_g, int ld_g, int m0, int M) {
    const int nq = ldw >> 2;
    for (int c40 = 0; c40 < nq; c40 += 64) {
        rb_gemm<false>(As, lda, K, W, ldw, sm.part, sm.ldp, c40);
        __syncthreads();
        const int nc = min(64, nq - c40);
        for (int idx = threadIdx.x; idx < RB * nc; idx += E2T) {
            const int r = idx / nc, c4 = c40 + idx - r * nc;
            float4 o = part_sum(sm.part, sm.ldp, r, c4);
            const int c = c4 * 4;
            o.x = (c + 0 < N) ? fmaxf(o.x + __ldcg(bias + c + 0), 0.0f) : 0.0f;
            o.y = (c + 1 < N) ? fmaxf(o.y + __ldcg(bias + c + 1), 0.0f) : 0.0f;
            o.z = (c + 2 < N) ? fmaxf(o.z + __ldcg(bias + c + 2), 0.0f) : 0.0f;
            o.w = (c + 3 < N) ? fmaxf(o.w + __ldcg(bias + c + 3), 0.0f) : 0.0f;
            *reinterpret_cast<float4*>(dst_s + r * ld_s + c) = o;
            if (m0 + r < M) *reinterpret_cast<float4*>(dst_g + (long long)(m0 + r) * ld_g + c) = o;
        }
        __syncthreads();
    }
}

// ---- one batch row of the policy loss on a whole warp: lane j holds action dimension j (NO <= 32).  The Gaussian terms are
// those of ppo_loss.cu's policy_row / policy_dlogvar / row_kl, formed in parallel and summed in index order through
// shuffles (the serial version is a chain of ~1.5 K dependent instructions per row on one lane); the surrogate and c_kl
// come from ppo_loss_dev.cuh.
__device__ __forceinline__ float seq_sum(float term, int n) {
    float s = 0.0f;
    for (int j = 0; j < n; ++j) s += __shfl_sync(0xffffffffu, term, j);
    return s;
}
__device__ __forceinline__ float seq_sum_sq(float z, int n) {
    float s = 0.0f;
    for (int j = 0; j < n; ++j) {
        const float zj = __shfl_sync(0xffffffffu, z, j);
        s = fmaf(zj, zj, s);
    }
    return s;
}
// KL(ref || current) of one row (ppo_net.py:61-62)
__device__ __forceinline__ float row_kl_warp(const float* rp, const float* mu, const float* s_sig, int A, int lane) {
    const bool on = lane < A;
    const float m0 = on ? rp[lane] : 0.0f, s0 = on ? rp[A + lane] : 1.0f, m1 = on ? mu[lane] : 0.0f, s1 = on ? s_sig[lane] : 1.0f;
    const float d = m0 - m1;
    const float t1 = seq_sum(logf(s1 / s0), A);
    const float t2 = seq_sum((s0 * s0 + d * d) / (2.0f * s1 * s1), A);
    return t1 + t2 - 0.5f * (float)A;
}
struct RowOut {
    float surr, rowloss, dlogvar;             // dlogvar: this lane's dimension
};
__device__ __forceinline__ RowOut policy_row_warp(int mode, const float* mu_, const float* act_, const float* s_sig, const float* bp,
                                                  const float* rp, float ad, int A, float c0, double invB, const double* hyper,
                                                  float c_kl, float* dpre_row, int ldd, int lane) {
    const bool on = lane < A;
    const float a = on ? act_[lane] : 0.0f, mu = on ? mu_[lane] : 0.0f, sg = on ? s_sig[lane] : 1.0f;
    const float bm = on ? bp[lane] : 0.0f, bs = on ? bp[A + lane] : 1.0f, rm = on ? rp[lane] : 0.0f, rs = on ? rp[A + lane] : 1.0f;
    const float z = (a - mu) / sg;
    const float ll = -0.5f * seq_sum_sq(z, A) - c0 - seq_sum(logf(sg), A);
    const float zb = (a - bm) / bs;
    const float llb = -0.5f * seq_sum_sq(zb, A) - c0 - seq_sum(logf(bs), A);
    const ppo_dev::Surrogate sr = ppo_dev::surrogate(mode, expf(ll), expf(llb), ad, invB, hyper);
    // gradient w.r.t. the pre-tanh output (mean = tanh(pre)) and this dimension's share of d loss / d log_var
    float dmu = sr.g_ll * z / sg;
    float dl = sr.g_ll * (z * z - 1.0f);
    if (mode == 1) {
        const float d = rm - mu;
        dmu += c_kl * (-(rm - mu) / (sg * sg));
        dl += c_kl * (1.0f - (rs * rs + d * d) / (sg * sg));
    }
    if (lane < ldd) dpre_row[lane] = on ? dmu * (1.0f - mu * mu) : 0.0f;
    return {sr.surr, sr.rowloss, on ? dl : 0.0f};
}

// ---- P1a: forward of one row block; leaves xs / h1s / h2s / outs in shared memory and the KL partial in kl_part[rb]
__device__ void fwd_item(const Job& p, const Sm& sm, int rb, bool first_epoch, const float* s_sig, double* s_red, unsigned long long* cp) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    long long t0 = clock64();
    const int m0 = rb * RB, M = p.M, D = p.D, NO = p.NO;
    const float* W1 = p.params + p.w_off[0];
    const float* W2 = p.params + p.w_off[1];
    const float* W3 = p.params + p.w_off[2];
    const int ldw3 = p.ldw[2];
    for (int i = tid; i < (p.H2 * ldw3) >> 2; i += E2T) *reinterpret_cast<float4*>(sm.w3s + i * 4) = gt::ldcg4(W3 + i * 4);
    // the per-row operands of the loss come in with ONE cooperative round trip (a lane reading them row by row pays an L2
    // latency per element: 60 us per policy epoch in the first version of this kernel)
    if (p.mode != 2)
        for (int idx = tid; idx < RB * 2 * NO; idx += E2T) {
            const int r = idx / (2 * NO), j = idx - r * 2 * NO;
            sm.refs[r * 2 * E2_MAX_OUT + j] = (m0 + r < M) ? p.ref[(long long)(m0 + r) * p.ldr + j] : 1.0f;
        }
    // input rows (z_filter.py:59-79), zero padded
    {
        const float cnt = (p.zf != nullptr) ? p.zf[2 * D] : 1.0f;
        for (int idx = tid; idx < RB * sm.ld_xs; idx += E2T) {
            const int r = idx / sm.ld_xs, k = idx - r * sm.ld_xs;
            const int m = m0 + r;
            float v = 0.0f;
            if (m < M && k < D) {
                if (first_epoch) {
                    v = p.x[(long long)m * p.ldx + k];
                    if (p.zf != nullptr) {
                        const float mean = p.zf[k] / cnt;
                        const float var = p.zf[D + k] / cnt - mean * mean;
                        v = gt::zf1(v, mean, fmaxf(sqrtf(var), p.zf_eps));
                    }
                } else {
                    v = __ldcg(p.x_in + (long long)m * p.ld_x + k);
                }
            }
            sm.xs[idx] = v;
            if (first_epoch && m < M && k < p.ld_x) p.x_in[(long long)m * p.ld_x + k] = v;
        }
    }
    __syncthreads();
    hidden_layer(sm, sm.xs, sm.ld_xs, D, W1, p.ldw[0], p.params + p.b_off[0], p.H1, sm.h1s, sm.ld_h1s, p.h1, p.ld_h1, m0, M);
    hidden_layer(sm, sm.h1s, sm.ld_h1s, p.H1, W2, p.ldw[1], p.params + p.b_off[1], p.H2, sm.h2s, sm.ld_h2s, p.h2, p.ld_h2, m0, M);
    if (tid == 0) cp[3] += (unsigned long long)(clock64() - t0);
    // head, one warp per row (2 rows per warp); then lanes 0 / 1 of the warp take the KL(ref || current) rows together
    for (int r = warp; r < RB; r += E2W) {
        const int m = m0 + r;
        if (m >= M) continue;                                // warp-uniform
        const float* h2r = sm.h2s + r * sm.ld_h2s;
        for (int n8 = 0; n8 < NO; n8 += 8) {
            float s8[8];
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) s8[jj] = 0.0f;
            for (int k = lane; k < p.H2; k += 32) {
                const float hv = h2r[k];
                const float* wr = sm.w3s + k * ldw3 + n8;
                const float4 w0 = *reinterpret_cast<const float4*>(wr);
                s8[0] = fmaf(hv, w0.x, s8[0]); s8[1] = fmaf(hv, w0.y, s8[1]);
                s8[2] = fmaf(hv, w0.z, s8[2]); s8[3] = fmaf(hv, w0.w, s8[3]);
                if (n8 + 4 < ldw3) {
                    const float4 w1 = *reinterpret_cast<const float4*>(wr + 4);
                    s8[4] = fmaf(hv, w1.x, s8[4]); s8[5] = fmaf(hv, w1.y, s8[5]);
                    s8[6] = fmaf(hv, w1.z, s8[6]); s8[7] = fmaf(hv, w1.w, s8[7]);
                }
            }
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const float tt = warp_sum(s8[jj]);
                if (lane == 0 && n8 + jj < NO) {
                    float v = tt + __ldcg(p.params + p.b_off[2] + n8 + jj);
                    if (p.act_out == SB200_ACT_TANH) v = tanhf(v);
                    else if (p.act_out == SB200_ACT_RELU) v = fmaxf(v, 0.0f);
                    p.out[(long long)m * p.ld_out + n8 + jj] = v;
                    sm.outs[r * E2_MAX_OUT + n8 + jj] = v;
                }
            }
        }
    }
    __syncwarp();
    double klacc = 0.0;
    if (p.mode != 2)
        for (int r = warp; r < RB; r += E2W) {
            if (m0 + r >= M) continue;                       // warp-uniform
            const float kl = row_kl_warp(sm.refs + r * 2 * E2_MAX_OUT, sm.outs + r * E2_MAX_OUT, s_sig, NO, lane);
            if (lane == 0) klacc += (double)kl;
        }
    if (p.mode != 2) {
        const double t = block_sum(klacc, s_red);
        if (tid == 0) p.kl_part[rb] = t;
    }
    __syncthreads();
    if (tid == 0) cp[2] += (unsigned long long)(clock64() - t0);
}

// ---- P1b: loss rows, dpre, d2, d1 of one row block (activations resident in shared memory, or reloaded)
__device__ void bwd_item(const Job& p, const Sm& sm, int rb, bool resident, double kl_mean_now, const float* s_sig, double* s_red,
                         unsigned long long* cp) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    long long t0 = clock64();
    const int m0 = rb * RB, M = p.M, NO = p.NO;
    const float* W3 = p.params + p.w_off[2];
    const int ldw3 = p.ldw[2];
    const bool policy = p.mode != 2;
    if (policy) {
        for (int idx = tid; idx < RB * 2 * NO; idx += E2T) {
            const int r = idx / (2 * NO), j = idx - r * 2 * NO;
            const bool ok = m0 + r < M;
            sm.behs[r * 2 * E2_MAX_OUT + j] = ok ? p.behave[(long long)(m0 + r) * p.ldb + j] : 1.0f;
            if (!resident) sm.refs[r * 2 * E2_MAX_OUT + j] = ok ? p.ref[(long long)(m0 + r) * p.ldr + j] : 1.0f;
        }
        for (int idx = tid; idx < RB * NO; idx += E2T) {
            const int r = idx / NO, j = idx - r * NO;
            sm.acts[r * E2_MAX_OUT + j] = (m0 + r < M) ? p.actions[(long long)(m0 + r) * p.lda + j] : 0.0f;
        }
        if (tid < RB) sm.advs[tid] = (m0 + tid < M) ? p.adv[m0 + tid] : 0.0f;
    } else if (tid < RB) {
        sm.advs[tid] = (m0 + tid < M) ? p.returns[m0 + tid] : 0.0f;
    }
    if (!resident) {
        for (int i = tid; i < (p.H2 * ldw3) >> 2; i += E2T) *reinterpret_cast<float4*>(sm.w3s + i * 4) = gt::ldcg4(W3 + i * 4);
        for (int idx = tid; idx < RB * (sm.ld_h1s >> 2); idx += E2T) {
            const int r = idx / (sm.ld_h1s >> 2), q = idx - r * (sm.ld_h1s >> 2);
            float4 v = zero4();
            if (m0 + r < M && q * 4 < p.ld_h1) v = gt::ldcg4(p.h1 + (long long)(m0 + r) * p.ld_h1 + q * 4);
            *reinterpret_cast<float4*>(sm.h1s + r * sm.ld_h1s + q * 4) = v;
        }
        for (int idx = tid; idx < RB * (sm.ld_h2s >> 2); idx += E2T) {
            const int r = idx / (sm.ld_h2s >> 2), q = idx - r * (sm.ld_h2s >> 2);
            float4 v = zero4();
            if (m0 + r < M && q * 4 < p.ld_h2) v = gt::ldcg4(p.h2 + (long long)(m0 + r) * p.ld_h2 + q * 4);
            *reinterpret_cast<float4*>(sm.h2s + r * sm.ld_h2s + q * 4) = v;
        }
        for (int idx = tid; idx < RB * NO; idx += E2T) {
            const int r = idx / NO, j = idx - r * NO;
            sm.outs[r * E2_MAX_OUT + j] = (m0 + r < M) ? __ldcg(p.out + (long long)(m0 + r) * p.ld_out + j) : 0.0f;
        }
    }
    __syncthreads();
    const double invM = 1.0 / (double)M;
    const float c0 = (float)(0.5 * 1.8378770664093453 * (double)NO);
    const float c_kl = (p.mode == 1) ? ppo_dev::adapt_ckl(kl_mean_now, invM, p.hyper, p.eta, p.kl_target) : 0.0f;
    // loss rows.  Policy: a warp per row, lane j = action dimension j (policy_row_warp).  Value: lanes 0 / 1 of every warp take
    // rows warp / warp + 8 together.  Operands and results live in shared memory: no local arrays.
    double acc_slot[4] = {0.0, 0.0, 0.0, 0.0};
    double dl_acc = 0.0;                                     // policy: this lane's dimension of d loss / d log_var, both rows
    if (policy) {
        for (int r = warp; r < RB; r += E2W) {
            const int m = m0 + r;
            float* dp = sm.dps + r * E2_MAX_OUT;
            if (m >= M) {                                    // rows past the batch: no gradient (warp-uniform)
                if (lane < p.ld_out) dp[lane] = 0.0f;
                continue;
            }
            const RowOut o = policy_row_warp(p.mode, sm.outs + r * E2_MAX_OUT, sm.acts + r * E2_MAX_OUT, s_sig, sm.behs + r * 2 * E2_MAX_OUT,
                                             sm.refs + r * 2 * E2_MAX_OUT, sm.advs[r], NO, c0, invM, p.hyper, c_kl, dp, p.ld_out,
                                             lane);
            if (lane == 0) {
                acc_slot[0] += (double)o.surr;
                acc_slot[1] += (double)o.rowloss;
            }
            dl_acc += (double)o.dlogvar;
            __syncwarp();
            if (lane < p.ld_out) p.dpre[(long long)m * p.ld_out + lane] = dp[lane];
        }
    } else {
        const int my_r = warp + E2W * lane;
        if (lane < 2 && my_r < RB) {
            float* dp = sm.dps + my_r * E2_MAX_OUT;
            for (int j = 0; j < p.ld_out; ++j) dp[j] = 0.0f;
            if (m0 + my_r < M) {
                const ppo_dev::ValueRow vr = ppo_dev::value_row(sm.outs[my_r * E2_MAX_OUT], sm.advs[my_r], M);
                dp[0] = vr.dpre;
                acc_slot[0] = vr.d; acc_slot[1] = vr.d * vr.d; acc_slot[2] = vr.r; acc_slot[3] = vr.r * vr.r;
                for (int j = 0; j < p.ld_out; ++j) p.dpre[(long long)(m0 + my_r) * p.ld_out + j] = dp[j];
            }
        }
    }
    __syncwarp();
    // d2 = (dpre W3^T) * relu'(h2), a warp per row
    for (int r = warp; r < RB; r += E2W) {
        const int m = m0 + r;
        float* d2r = sm.d2s + r * sm.ld_h2s;
        if (m >= M) {                                        // rows past the batch contribute nothing
            for (int k = lane; k < sm.ld_h2s; k += 32) d2r[k] = 0.0f;
            continue;
        }
        const float* h2r = sm.h2s + r * sm.ld_h2s;
        const float* dp = sm.dps + r * E2_MAX_OUT;
        for (int k = lane; k < sm.ld_h2s; k += 32) {
            float g = 0.0f;
            if (k < p.H2) {
                const float* wr = sm.w3s + k * ldw3;
                for (int j = 0; j < NO; ++j) g = fmaf(dp[j], wr[j], g);
                if (!(h2r[k] > 0.0f)) g = 0.0f;
            }
            d2r[k] = g;
            if (k < p.ld_h2) p.d2[(long long)m * p.ld_h2 + k] = g;
        }
    }
    {
        double* part = p.loss_part + (size_t)rb * E2_SLOTS;
        const int ns = policy ? 2 : 4;                       // policy: [surr, rowloss, unused, unused] + dlog_var
        for (int s = 0; s < ns; ++s) {
            const double t = block_sum(acc_slot[s], s_red);
            if (tid == 0) part[s] = t;
        }
        if (policy) {                                        // d loss / d log_var: sum over the warps, dimension by dimension
            double* red = reinterpret_cast<double*>(sm.part);
            __syncthreads();
            red[warp * 32 + lane] = dl_acc;
            __syncthreads();
            if (tid < NO) {
                double t = 0.0;
                for (int w = 0; w < E2W; ++w) t += red[w * 32 + tid];
                part[4 + tid] = t;
            }
        }
    }
    __syncthreads();
    // this block's share of dW3 = h2^T dpre and db3 (16 rows, operands in shared memory): summed over the blocks in P2
    {
        float* wp = p.w3part + (size_t)rb * (p.H2 + 1) * ldw3;
        const int nq3 = ldw3 >> 2;
        for (int idx = tid; idx < (p.H2 + 1) * nq3; idx += E2T) {
            const int k = idx / nq3, q = idx - k * nq3;
            float4 acc = zero4();
#pragma unroll 4
            for (int r = 0; r < RB; ++r) {
                const float hv = (k < p.H2) ? sm.h2s[r * sm.ld_h2s + k] : 1.0f;
                const float4 dv = *reinterpret_cast<const float4*>(sm.dps + r * E2_MAX_OUT + q * 4);
                acc.x = fmaf(hv, dv.x, acc.x); acc.y = fmaf(hv, dv.y, acc.y);
                acc.z = fmaf(hv, dv.z, acc.z); acc.w = fmaf(hv, dv.w, acc.w);
            }
            *reinterpret_cast<float4*>(wp + (size_t)k * ldw3 + q * 4) = acc;
        }
    }
    if (tid == 0) {
        const long long t1 = clock64();
        cp[4] += (unsigned long long)(t1 - t0);
        t0 = t1;
    }
    // d1 = (d2 . W2^T) * relu'(h1)
    {
        const int nq = p.ld_h1 >> 2;
        for (int c40 = 0; c40 < nq; c40 += 64) {
            rb_gemm<false>(sm.d2s, sm.ld_h2s, p.H2, p.w2t, p.ld_h1, sm.part, sm.ldp, c40);
            __syncthreads();
            const int nc = min(64, nq - c40);
            for (int idx = tid; idx < RB * nc; idx += E2T) {
                const int r = idx / nc, c4 = c40 + idx - r * nc;
                if (m0 + r >= M) continue;
                float4 o = part_sum(sm.part, sm.ldp, r, c4);
                const float4 hv = *reinterpret_cast<const float4*>(sm.h1s + r * sm.ld_h1s + c4 * 4);
                if (!(hv.x > 0.0f)) o.x = 0.0f;
                if (!(hv.y > 0.0f)) o.y = 0.0f;
                if (!(hv.z > 0.0f)) o.z = 0.0f;
                if (!(hv.w > 0.0f)) o.w = 0.0f;
                *reinterpret_cast<float4*>(p.d1 + (long long)(m0 + r) * p.ld_h1 + c4 * 4) = o;
            }
            __syncthreads();
        }
    }
    if (tid == 0) cp[5] += (unsigned long long)(clock64() - t0);
}

// ---- P2: one weight-gradient item.  layer 1: dW2 rows [16 kb, 16 kb + 16) = h1^T d2;  layer 0: dW1 = x_in^T d1;
// row split z covers batch rows [z rps, (z+1) rps); the k-block 0 item also produces the bias gradient (column sums).
__device__ void dw_item(const Job& p, const Sm& sm, float* As, int layer, int kb, int z) {
    const int tid = threadIdx.x;
    const float* X = layer == 1 ? p.h1 : p.x_in;
    const int ldx = layer == 1 ? p.ld_h1 : p.ld_x;
    const float* dY = layer == 1 ? p.d2 : p.d1;
    const int ldy = layer == 1 ? p.ld_h2 : p.ld_h1;         // == ldw[layer]
    const int kdim = layer == 1 ? p.H1 : p.D;
    const int m_lo = z * p.rps, m_hi = min(p.M, m_lo + p.rps);
    const int Kz = max(0, m_hi - m_lo), Kzp = (Kz + 3) & ~3;
    const int lda = ((p.rps + 3) & ~3) + 4;
    const int k0 = kb * RB;
    for (int idx = tid; idx < Kzp * 4; idx += E2T) {
        const int mm = idx >> 2, q = idx & 3;
        float4 v = zero4();
        if (mm < Kz && k0 + q * 4 < ldx) v = gt::ldcg4(X + (long long)(m_lo + mm) * ldx + k0 + q * 4);
        As[(q * 4 + 0) * lda + mm] = v.x;
        As[(q * 4 + 1) * lda + mm] = v.y;
        As[(q * 4 + 2) * lda + mm] = v.z;
        As[(q * 4 + 3) * lda + mm] = v.w;
    }
    __syncthreads();
    float* slab = p.slabs + (long long)z * p.n_params;
    const int nq = ldy >> 2;
    const int N = layer == 1 ? p.H2 : p.H1;
    for (int c40 = 0; c40 < nq; c40 += 64) {
        if (kb == 0) rb_gemm<true>(As, lda, Kz, dY + (long long)m_lo * ldy, ldy, sm.part, sm.ldp, c40);
        else rb_gemm<false>(As, lda, Kz, dY + (long long)m_lo * ldy, ldy, sm.part, sm.ldp, c40);
        __syncthreads();
        const int nc = min(64, nq - c40);
        for (int idx = tid; idx < (RB + 1) * nc; idx += E2T) {
            const int r = idx / nc, c4 = c40 + idx - r * nc;
            if (r < RB) {
                if (k0 + r < kdim)
                    *reinterpret_cast<float4*>(slab + p.w_off[layer] + (long long)(k0 + r) * ldy + c4 * 4) = part_sum(sm.part, sm.ldp, r, c4);
            } else if (kb == 0) {
                const float4 o = part_sum(sm.part, sm.ldp, RB, c4);
                float* db = slab + p.b_off[layer] + c4 * 4;
                if (c4 * 4 + 0 < N) db[0] = o.x;
                if (c4 * 4 + 1 < N) db[1] = o.y;
                if (c4 * 4 + 2 < N) db[2] = o.z;
                if (c4 * 4 + 3 < N) db[3] = o.w;
            }
        }
        __syncthreads();
    }
}

// dW3 / db3 of row split z = sum of the row-block partials that P1 left in w3part, in block order (fixed -> deterministic)
__device__ void dw3_item(const Job& p, const Sm& sm, int z) {
    (void)sm;
    const int tid = threadIdx.x;
    const int ldw3 = p.ldw[2], nq3 = ldw3 >> 2;
    const int per = (p.n_rb + p.s - 1) / p.s;
    const int rb_lo = z * per, rb_hi = min(p.n_rb, rb_lo + per);
    const size_t stride = (size_t)(p.H2 + 1) * ldw3;
    float* slab = p.slabs + (long long)z * p.n_params;
    for (int idx = tid; idx < (p.H2 + 1) * nq3; idx += E2T) {
        const int k = idx / nq3, q = idx - k * nq3;
        float4 acc = zero4();
#pragma unroll 8
        for (int rb = rb_lo; rb < rb_hi; ++rb) {
            const float4 v = gt::ldcg4(p.w3part + (size_t)rb * stride + (size_t)k * ldw3 + q * 4);
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        if (k < p.H2) {
            *reinterpret_cast<float4*>(slab + p.w_off[2] + (long long)k * ldw3 + q * 4) = acc;
        } else {
            float* db = slab + p.b_off[2] + q * 4;
            if (q * 4 + 0 < p.NO) db[0] = acc.x;
            if (q * 4 + 1 < p.NO) db[1] = acc.y;
            if (q * 4 + 2 < p.NO) db[2] = acc.z;
            if (q * 4 + 3 < p.NO) db[3] = acc.w;
        }
    }
}

// phase timing (always on: two CTAs, one thread, a handful of clock reads per epoch)
#define E2_STAMP(slot)                                                                       \
    do {                                                                                     \
        if (tid == 0 && (c == 0 || c == G - 1)) {                                            \
            const long long now_ = clock64();                                                \
            P.prof[(c == 0 ? 0 : 16) + (slot)] += (unsigned long long)(now_ - prof_t);      \
            prof_t = now_;                                                                   \
        }                                                                                    \
    } while (0)

__global__ void __launch_bounds__(E2T, 1) ppo_epochs2_kernel(const __grid_constant__ E2Params P) {
    extern __shared__ __align__(16) float smem[];
    __shared__ float s_sig[ppo_dev::MAX_A];
    __shared__ double s_red[32];
    __shared__ optim_dev::AdamCoef s_adam[2];
    const int tid = threadIdx.x;
    const int G = (int)gridDim.x, c = (int)blockIdx.x;
    Sm sm;
    sm.xs = smem + P.o_xs; sm.h1s = smem + P.o_h1; sm.h2s = smem + P.o_h2; sm.d2s = smem + P.o_d2;
    sm.outs = smem + P.o_out; sm.dps = smem + P.o_dp; sm.part = smem + P.o_part; sm.w3s = smem + P.o_w3;
    sm.refs = smem + P.o_rows; sm.behs = sm.refs + RB * 2 * E2_MAX_OUT; sm.acts = sm.behs + RB * 2 * E2_MAX_OUT; sm.advs = sm.acts + RB * E2_MAX_OUT;
    sm.ld_xs = P.ld_xs; sm.ld_h1s = P.ld_h1s; sm.ld_h2s = P.ld_h2s; sm.ldp = P.ldp;
    unsigned int bar_target = 0;
    const int NJ = P.n_jobs;
    long long prof_t = clock64();

    // per-job loop state (identical in every CTA)
    bool left[2] = {false, false};        // no further training epochs
    int step0[2], steps_done[2] = {0, 0};
    unsigned int par_k[2] = {0u, 0u};
    int e_max = 0;
    for (int j = 0; j < NJ; ++j) {
        const Job& p = P.job[j];
        step0[j] = p.opt->step;
        if (p.stop != nullptr && *p.stop) left[j] = true;      // raised only behind a barrier every CTA has passed: uniform
        if (p.par.world > 1) par_k[j] = header_of(p.par, p.par.rank)->counter;
        const int last = (p.mode != 2) ? p.epochs : p.epochs - 1;
        e_max = max(e_max, last);
    }
    // ---- W2^T copies (refreshed by the Adam phase afterwards)
    for (int j = 0; j < NJ; ++j) {
        const Job& p = P.job[j];
        const float* W2 = p.params + p.w_off[1];
        for (long long i = (long long)c * E2T + tid; i < (long long)p.H1 * p.ldw[1]; i += (long long)G * E2T) {
            const int k = (int)(i / p.ldw[1]), n = (int)(i - (long long)k * p.ldw[1]);
            if (n < p.H2) p.w2t[(long long)n * p.ld_h1 + k] = W2[i];
        }
        for (long long i = (long long)c * E2T + tid; i < (long long)p.H2 * (p.ld_h1 - p.H1); i += (long long)G * E2T) {
            const int n = (int)(i / (p.ld_h1 - p.H1)), k = p.H1 + (int)(i - (long long)n * (p.ld_h1 - p.H1));
            p.w2t[(long long)n * p.ld_h1 + k] = 0.0f;
        }
    }
    grid_bar(P.bar, bar_target);
    E2_STAMP(0);

    for (int e = 0; e <= e_max; ++e) {
        bool fwd[2], train[2];
        int item0[2], n_items = 0;
        for (int j = 0; j < NJ; ++j) {
            const Job& p = P.job[j];
            const int last = (p.mode != 2) ? p.epochs : p.epochs - 1;
            fwd[j] = !left[j] && e <= last;
            train[j] = fwd[j] && e < p.epochs;
            item0[j] = n_items;
            if (fwd[j]) n_items += p.n_rb;
        }
        if (n_items == 0) break;                               // uniform
        // ---------------- P1: forward (+ loss and input gradients unless the loss must wait for the KL mean)
        int my_last_item = -1;
        long long cta_t = clock64();
        for (int it = c; it < n_items; it += G) {
            const int j = (NJ == 2 && fwd[1] && it >= item0[1]) ? 1 : 0;
            const Job& p = P.job[j];
            const int rb = it - item0[j];
            if (p.mode != 2 && tid < p.NO) s_sig[tid] = expf(__ldcg(p.params + p.extra_off + tid));      // builders.py:127
            __syncthreads();
            fwd_item(p, sm, rb, e == 0, s_sig, s_red, P.cta_prof + c * 8);
            if (train[j] && p.mode != 1) bwd_item(p, sm, rb, true, 0.0, s_sig, s_red, P.cta_prof + c * 8);
            my_last_item = it;
        }
        if (tid == 0) P.cta_prof[c * 8 + 0] += (unsigned long long)(clock64() - cta_t);
        E2_STAMP(1);
        grid_bar(P.bar, bar_target);
        E2_STAMP(2);
        // ---------------- gate (policy jobs): mean KL(ref || current) of the forward just done
        double klm[2] = {0.0, 0.0};
        for (int j = 0; j < NJ; ++j) {
            const Job& p = P.job[j];
            if (!fwd[j] || p.mode == 2) continue;
            {
                double a = 0.0;                                                // same tree in every CTA: identical result
                for (int k = tid; k < p.n_rb; k += E2T) a += __ldcg(&p.kl_part[k]);
                const double acc = block_sum(a, s_red);
                klm[j] = (double)(float)(acc * (1.0 / (double)p.M));           // .mean() in fp32 (kl_kernel)
            }
            if (p.par.world > 1) {                                             // average the scalar over ranks (CTA 0)
                ParHeader* par_me = header_of(p.par, p.par.rank);
                if (c == 0) {
                    const unsigned int k = par_k[j] + 1u;
                    double* mine = reinterpret_cast<double*>(slot_of(p.par, p.par.rank, k & 1u));
                    if (tid == 0) {
                        *mine = klm[j];
                        __threadfence_system();
                    }
                    publish_and_wait(p.par, par_me, 0, k);
                    if (tid == 0) {
                        double a = 0.0;
                        for (int q = 0; q < p.par.world; ++q)
                            a += ld_sys_f64(reinterpret_cast<const double*>(slot_of(p.par, q, k & 1u)));
                        *p.kl_global = (double)(float)(a * (1.0 / (double)p.par.world));
                    }
                }
                par_k[j] += 1u;
                grid_bar(P.bar, bar_target);
                klm[j] = __ldcg(p.kl_global);
            }
            bool stop_now = false;
            if (e > 0) {                                                       // post-step KL of epoch e-1 (ppo.py:553-556)
                stop_now = p.stop_threshold > 0.0 && klm[j] > p.stop_threshold;
                if (c == 0 && tid == 0) {
                    p.stats[SB200_STAT_KL_POST] = (float)klm[j];
                    p.stats[SB200_STAT_EPOCHS] += 1.0f;
                    if (stop_now && p.stop != nullptr) *p.stop = 1;
                }
            }
            if (stop_now || !train[j]) {
                left[j] = true;
                train[j] = false;
            }
        }
        // ---------------- adapt mode: the loss needs the KL mean (ppo.py:262-270) -> second half of P1 now
        {
            bool any = false;
            for (int j = 0; j < NJ; ++j) any = any || (train[j] && P.job[j].mode == 1);
            if (any) {
                for (int it = c; it < n_items; it += G) {
                    const int j = (NJ == 2 && fwd[1] && it >= item0[1]) ? 1 : 0;
                    const Job& p = P.job[j];
                    if (!(train[j] && p.mode == 1)) continue;
                    if (tid < p.NO) s_sig[tid] = expf(__ldcg(p.params + p.extra_off + tid));
                    __syncthreads();
                    bwd_item(p, sm, it - item0[j], it == my_last_item && n_items <= G, klm[j], s_sig, s_red, P.cta_prof + c * 8);
                }
                grid_bar(P.bar, bar_target);
            }
        }
        bool any_train = false;
        for (int j = 0; j < NJ; ++j) any_train = any_train || train[j];
        if (!any_train) continue;                              // uniform: e.g. only the policy's trailing forward ran
        // ---------------- loss statistics + dlog_var (CTA 0); the slab entry is consumed behind the next barriers
        if (c == 0) {
            for (int j = 0; j < NJ; ++j) {
                const Job& p = P.job[j];
                if (!train[j]) continue;
                const int NO = p.NO;
                const double invM = 1.0 / (double)p.M;
                if (p.mode != 2) {
                    if (tid < NO) s_sig[tid] = expf(__ldcg(p.params + p.extra_off + tid));
                    __syncthreads();
                    for (int s0 = 0; s0 < 4 + NO; s0 += E2T >> 3) {               // 8 lanes per statistic, uniform trip count
                        const int s = s0 + (tid >> 3);
                        const bool on = s < 4 + NO && (s < 2 || s >= 4);
                        double acc = 0.0;
                        if (on)
                            for (int k = tid & 7; k < p.n_rb; k += 8) acc += __ldcg(&p.loss_part[(size_t)k * E2_SLOTS + s]);
                        acc += __shfl_xor_sync(0xffffffffu, acc, 4);
                        acc += __shfl_xor_sync(0xffffffffu, acc, 2);
                        acc += __shfl_xor_sync(0xffffffffu, acc, 1);
                        if (!on || (tid & 7) != 0) continue;
                        if (s >= 4) p.slabs[p.extra_off + (s - 4)] = (float)acc;
                        else ppo_dev::loss_stats(p.mode, s, acc, invM, p.hyper, p.eta, p.kl_target, klm[j], p.stats);
                    }
                    if (tid == 0) p.stats[SB200_STAT_ENTROPY] = ppo_dev::gauss_entropy(s_sig, NO);
                    __syncthreads();
                } else if (tid < 32) {
                    double s[4] = {0, 0, 0, 0};
                    for (int k = tid; k < p.n_rb; k += 32)
                        for (int q = 0; q < 4; ++q) s[q] += __ldcg(&p.loss_part[(size_t)k * E2_SLOTS + q]);
                    for (int q = 0; q < 4; ++q) s[q] = warp_sum(s[q]);
                    if (tid == 0) ppo_dev::value_stats(s, (double)p.M, p.stats);
                }
            }
        }
        E2_STAMP(3);
        cta_t = clock64();
        // ---------------- P2: weight-gradient items
        {
            int w0[2], n_w = 0;
            for (int j = 0; j < NJ; ++j) {
                const Job& p = P.job[j];
                w0[j] = n_w;
                if (train[j]) n_w += (((p.H1 + RB - 1) / RB) + ((p.D + RB - 1) / RB) + 1) * p.s;
            }
            // CTA 0 spends this phase on the loss statistics (above, ~10 us of serial work): when the other CTAs cover the
            // items in as many rounds as the whole grid would (one round at the full grid, two on the learner's 68-SM budget)
            // it takes none, so that nobody waits for it at the barrier
            const int skip0 = (G > 1 && (n_w + G - 2) / (G - 1) == (n_w + G - 1) / G) ? 1 : 0;
            for (int it = c - skip0; it >= 0 && it < n_w; it += G - skip0) {
                const int j = (NJ == 2 && train[1] && it >= w0[1]) ? 1 : 0;
                const Job& p = P.job[j];
                int q = it - w0[j];
                const int nA = ((p.H1 + RB - 1) / RB) * p.s, nB = ((p.D + RB - 1) / RB) * p.s;
                if (q < nA) dw_item(p, sm, smem, 1, q / p.s, q % p.s);
                else if (q < nA + nB) dw_item(p, sm, smem, 0, (q - nA) / p.s, (q - nA) % p.s);
                else dw3_item(p, sm, q - nA - nB);
            }
        }
        if (tid == 0) P.cta_prof[c * 8 + 1] += (unsigned long long)(clock64() - cta_t);
        E2_STAMP(4);
        grid_bar(P.bar, bar_target);
        E2_STAMP(5);
        // ---------------- P3: slabs -> grad (fixed order), squared-norm partials of P.n_sq chunks (CTA c takes chunks
        // c, c + G, ...: every partial, and so the norm, is the same at any grid)
        for (int j = 0; j < NJ; ++j) {
            const Job& p = P.job[j];
            if (!train[j]) continue;
            for (int k = c; k < P.n_sq; k += G) {
                double sq = 0.0;
                for (long long i4 = (long long)k * E2T + tid; i4 < (p.n_params >> 2); i4 += (long long)P.n_sq * E2T) {    // one quad per thread
                    float4 g = gt::ldcg4(p.slabs + i4 * 4);
                    for (int z = 1; z < p.s; ++z) {
                        const float4 t4 = gt::ldcg4(p.slabs + (long long)z * p.n_params + i4 * 4);
                        g.x += t4.x; g.y += t4.y; g.z += t4.z; g.w += t4.w;
                    }
                    *reinterpret_cast<float4*>(p.grad + i4 * 4) = g;
                    sq += (double)g.x * (double)g.x;
                    sq += (double)g.y * (double)g.y;
                    sq += (double)g.z * (double)g.z;
                    sq += (double)g.w * (double)g.w;
                }
                const double t = block_sum(sq, s_red);
                if (tid == 0) p.sq_part[k] = (p.par.world > 1) ? 0.0 : t;
            }
        }
        E2_STAMP(6);
        grid_bar(P.bar, bar_target);
        E2_STAMP(7);
        {
            // ---------------- X (data-parallel): all-reduce (mean) of the flat gradients over NVLink peer memory
            bool any_dp = false;
            for (int j = 0; j < NJ; ++j) any_dp = any_dp || (train[j] && P.job[j].par.world > 1);
            if (any_dp) {
                const int PG = min(G / NJ, PAR_MAX_CTAS);
                for (int j = 0; j < NJ; ++j) {
                    const Job& p = P.job[j];
                    if (!(train[j] && p.par.world > 1)) continue;
                    const unsigned int k = par_k[j] + 1u;
                    par_k[j] += 1u;
                    const int cl = c - j * PG;                                 // this job's slice owners: CTAs [j PG, (j+1) PG)
                    if (cl < 0 || cl >= PG) continue;                          // block-uniform
                    ParHeader* par_me = header_of(p.par, p.par.rank);
                    double sq = 0.0;
                    long long per = (p.n_params + PG - 1) / PG;
                    per = (per + 3) & ~3ll;
                    const long long lo = (long long)cl * per;
                    const long long hi = (lo + per < p.n_params) ? lo + per : p.n_params;
                    float* mine = slot_of(p.par, p.par.rank, k & 1u);
                    for (long long i = lo + (long long)tid * 4; i < hi; i += (long long)E2T * 4)
                        *reinterpret_cast<float4*>(mine + i) = gt::ldcg4(p.grad + i);
                    __threadfence_system();
                    publish_and_wait(p.par, par_me, cl, k);
                    const float scale = 1.0f / (float)p.par.world;
                    if ((p.par.max_floats & 3) == 0) {
                        sq = peer_sum_slice<PAR_MAX_WORLD, 1>(p, lo, hi, k & 1u, scale);      // one path for every world size
                    } else {
                        for (long long i = lo + tid; i < hi; i += E2T) {
                            float a = 0.f;
                            for (int q = 0; q < p.par.world; ++q) a += ld_sys1(slot_of(p.par, q, k & 1u) + i);
                            a = __fmul_rn(a, scale);
                            p.grad[i] = a;
                            sq += (double)a * (double)a;
                        }
                    }
                    const double t = block_sum(sq, s_red);
                    if (tid == 0) p.sq_part[c] = t;
                }
                grid_bar(P.bar, bar_target);
            }
        }
        // ---------------- P4: global norm, clip, Adam; W2^T follows W2
        for (int j = 0; j < NJ; ++j) {
            const Job& p = P.job[j];
            if (!train[j]) continue;
            steps_done[j] += 1;
            double a = 0.0;
            for (int k = tid; k < P.n_sq; k += E2T) a += __ldcg(&p.sq_part[k]);
            const double acc = block_sum(a, s_red);                            // same tree in every CTA: identical coefficients
            if (tid == 0) {
                const float total_norm = (float)sqrt(acc);
                s_adam[j] = optim_dev::adam_coef(step0[j] + steps_done[j], p.lr[0], 0.9, 0.999, 1e-8, p.weight_decay, p.clip_mode,
                                                 p.clip_value, total_norm);
                if (c == 0) {
                    p.opt->step = step0[j] + steps_done[j];
                    p.opt->total_norm = total_norm;
                    if (p.norm_out != nullptr) *p.norm_out = total_norm;
                }
            }
        }
        __syncthreads();
        for (int j = 0; j < NJ; ++j) {
            const Job& p = P.job[j];
            if (!train[j]) continue;
            const optim_dev::AdamCoef ac = s_adam[j];
            const long long w2_lo = p.w_off[1], w2_hi = w2_lo + (long long)p.H1 * p.ldw[1];
            for (long long i4 = (long long)c * E2T + tid; i4 < (p.n_params >> 2); i4 += (long long)G * E2T) {    // one quad per thread
                const long long i = i4 * 4;
                float4 pq = gt::ldcg4(p.params + i), mq = *reinterpret_cast<const float4*>(p.m + i);
                float4 vq = *reinterpret_cast<const float4*>(p.v + i);
                const float4 gq = gt::ldcg4(p.grad + i);
                optim_dev::adam_apply(ac, gq.x, pq.x, mq.x, vq.x);
                optim_dev::adam_apply(ac, gq.y, pq.y, mq.y, vq.y);
                optim_dev::adam_apply(ac, gq.z, pq.z, mq.z, vq.z);
                optim_dev::adam_apply(ac, gq.w, pq.w, mq.w, vq.w);
                *reinterpret_cast<float4*>(p.params + i) = pq;
                *reinterpret_cast<float4*>(p.m + i) = mq;
                *reinterpret_cast<float4*>(p.v + i) = vq;
                if (i >= w2_lo && i < w2_hi) {                                   // W2 starts and its rows end on quad boundaries
                    const int k = (int)((i - w2_lo) / p.ldw[1]), n = (int)((i - w2_lo) - (long long)k * p.ldw[1]);
                    const float pv[4] = {pq.x, pq.y, pq.z, pq.w};
#pragma unroll
                    for (int u = 0; u < 4; ++u)
                        if (n + u < p.H2) p.w2t[(long long)(n + u) * p.ld_h1 + k] = pv[u];
                }
            }
        }
        E2_STAMP(8);
        grid_bar(P.bar, bar_target);
        E2_STAMP(9);
    }
    if (c == 0 && tid == 0)
        for (int j = 0; j < NJ; ++j)
            if (P.job[j].par.world > 1) header_of(P.job[j].par, P.job[j].par.rank)->counter = par_k[j];
}

bool e2_net_ok(const sb200_mlp* net) {
    if (net == nullptr || net->n_layers != 3 || net->aux_layer >= 0) return false;
    if (net->act[0] != SB200_ACT_RELU || net->act[1] != SB200_ACT_RELU) return false;
    const int D = net->dims[0], H1 = net->dims[1], H2 = net->dims[2], NO = net->dims[3];
    if (D < 1 || H1 < 1 || H2 < 1 || NO < 1 || NO > E2_MAX_OUT) return false;
    if (D > 512 || H1 > 512 || H2 > 512) return false;
    return true;
}

inline int ru4(int v) { return (v + 3) & ~3; }

struct Plan {
    int o_xs, o_h1, o_h2, o_d2, o_out, o_dp, o_part, o_w3, o_rows, ld_xs, ld_h1s, ld_h2s, ldp;
    size_t smem_bytes;
    int s[2], rps[2];
    int n_sq;
};

// SMs of the current device (at most E2_MAX_G): the full grid, and what the plan is sized for at any grid
int e2_n_sm() {
    static int n_sm = 0;
    if (n_sm == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n_sm = 132;
    }
    return std::min(n_sm, E2_MAX_G);
}

// shared-memory plan + row-split choice for up to two jobs.  Sized for one CTA per SM whatever grid the launch gets, so that a
// capped grid (a learner sharing the GPU with the actors) computes the same slabs and sums as the full one.
bool e2_plan(const sb200_epochs* const* a, int n_jobs, Plan* pl) {
    const int G = e2_n_sm();
    pl->n_sq = G;
    int ld_xs = 4, ld_h1 = 4, ld_h2 = 4, ldp = 4, max_as = 0, max_w3 = 4;
    int blocks = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const sb200_mlp* net = a[j]->net;
        if (!e2_net_ok(net) || sb200_mlp_has_ln(net)) return false;
        ld_xs = std::max(ld_xs, ru4(net->dims[0]));
        ld_h1 = std::max(ld_h1, ru4(net->dims[1]));
        ld_h2 = std::max(ld_h2, ru4(net->dims[2]));
        max_w3 = std::max(max_w3, net->dims[2] * ru4(net->dims[3]));
        blocks += (net->dims[1] + RB - 1) / RB + (net->dims[0] + RB - 1) / RB + 1;
    }
    ldp = std::max(ld_h1, ld_h2);
    for (int j = 0; j < n_jobs; ++j) {
        // one wave of weight-gradient items if possible; never more slabs than the trainer allocated
        int s = std::max(1, G / std::max(1, blocks));
        s = std::min(s, a[j]->splits);
        s = std::min(s, std::max(1, a[j]->M / 64));
        int rps = ((a[j]->M + s - 1) / s + 3) & ~3;
        pl->s[j] = s;
        pl->rps[j] = rps;
        max_as = std::max(max_as, RB * (ru4(rps) + 4));
    }
    long long off = 0;
    auto take = [&](long long n) { const long long o = off; off += (n + 3) / 4 * 4; return (int)o; };
    pl->ld_xs = ld_xs; pl->ld_h1s = ld_h1; pl->ld_h2s = ld_h2; pl->ldp = ldp;
    // the activation region doubles as the A operand of the weight-gradient items (smem offset 0)
    pl->o_xs = take((long long)RB * ld_xs);
    pl->o_h1 = take((long long)RB * ld_h1);
    pl->o_h2 = take((long long)RB * ld_h2);
    pl->o_d2 = take((long long)RB * ld_h2);
    pl->o_out = take((long long)RB * E2_MAX_OUT);
    pl->o_dp = take((long long)RB * E2_MAX_OUT);
    if (off < max_as) off = (max_as + 3) / 4 * 4;
    pl->o_part = take(4LL * (RB + 1) * ldp);
    pl->o_w3 = take(max_w3);
    pl->o_rows = take((long long)RB * (5 * E2_MAX_OUT + 1));       // ref | behave | action rows, advantages / returns
    pl->smem_bytes = (size_t)off * sizeof(float);
    return pl->smem_bytes <= 220 * 1024;
}

struct WsLayout {
    size_t bar, prof, cta_prof, w3part[2], w2t[2], kl_part[2], loss_part[2], sq_part[2], kl_global[2], total;
};

WsLayout e2_ws(const sb200_epochs* const* a, int n_jobs) {
    WsLayout w;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
    w.bar = take(256);
    w.prof = take(32 * sizeof(unsigned long long));
    w.cta_prof = take((size_t)E2_MAX_G * 8 * sizeof(unsigned long long));
    for (int j = 0; j < 2; ++j) {
        if (j >= n_jobs) {
            w.w3part[j] = w.w2t[j] = w.kl_part[j] = w.loss_part[j] = w.sq_part[j] = w.kl_global[j] = 0;
            continue;
        }
        const sb200_mlp* net = a[j]->net;
        const size_t n_rb = (size_t)(a[j]->M + RB - 1) / RB;
        w.w2t[j] = take((size_t)net->dims[2] * ru4(net->dims[1]) * sizeof(float));
        w.w3part[j] = take(n_rb * (size_t)(net->dims[2] + 1) * ru4(net->dims[3]) * sizeof(float));
        w.kl_part[j] = take(n_rb * sizeof(double));
        w.loss_part[j] = take(n_rb * E2_SLOTS * sizeof(double));
        w.sq_part[j] = take((size_t)E2_MAX_G * sizeof(double));
        w.kl_global[j] = take(sizeof(double));
    }
    w.total = off;
    return w;
}

int e2_fill_job(const sb200_epochs* a, Job* p, unsigned char* ws, const WsLayout& wl, int j, const Plan& pl) {
    const sb200_mlp* net = a->net;
    SB200_REQUIRE(a->params && a->n_params >= 1 && a->x && a->M >= 2 && a->ldx >= net->dims[0]);
    SB200_REQUIRE(a->x_in && a->h1 && a->h2 && a->out && a->d1 && a->d2 && a->dpre && a->slabs && a->grad && a->exp_avg && a->exp_avg_sq);
    SB200_REQUIRE(a->lr && a->opt_workspace && a->stats && a->splits >= 1 && a->epochs >= 1);
    SB200_REQUIRE(a->mode >= 0 && a->mode <= 2 && a->clip_mode >= 0 && a->clip_mode <= 2);
    SB200_REQUIRE((((uintptr_t)a->x_in) & 15) == 0 && (((uintptr_t)a->params) & 15) == 0 && (((uintptr_t)a->slabs) & 15) == 0);
    SB200_REQUIRE((((uintptr_t)a->h1) & 15) == 0 && (((uintptr_t)a->h2) & 15) == 0 && (((uintptr_t)a->d1) & 15) == 0);
    SB200_REQUIRE((((uintptr_t)a->d2) & 15) == 0 && (((uintptr_t)a->dpre) & 15) == 0 && a->n_params % 4 == 0);
    SB200_REQUIRE((((uintptr_t)a->grad) & 15) == 0 && (((uintptr_t)a->exp_avg) & 15) == 0 && (((uintptr_t)a->exp_avg_sq) & 15) == 0);
    p->params = a->params;
    p->n_params = a->n_params;
    for (int l = 0; l < 3; ++l) {
        SB200_REQUIRE(net->W[l] >= a->params && net->b[l] >= a->params && net->W[l] < a->params + a->n_params);
        p->w_off[l] = (int)(net->W[l] - a->params);
        p->b_off[l] = (int)(net->b[l] - a->params);
        p->ldw[l] = net->ldw[l];
        SB200_REQUIRE(p->ldw[l] % 4 == 0 && p->w_off[l] % 4 == 0 && p->ldw[l] == ru4(net->dims[l + 1]));
    }
    p->D = net->dims[0]; p->H1 = net->dims[1]; p->H2 = net->dims[2]; p->NO = net->dims[3];
    p->act_out = net->act[2];
    p->extra_off = a->extra_off;
    p->x = a->x; p->ldx = a->ldx; p->M = a->M;
    p->zf = a->zf_stats; p->zf_eps = (float)a->zf_eps;
    p->x_in = a->x_in; p->h1 = a->h1; p->h2 = a->h2; p->out = a->out; p->d1 = a->d1; p->d2 = a->d2; p->dpre = a->dpre;
    p->ld_x = ru4(p->D); p->ld_h1 = ru4(p->H1); p->ld_h2 = ru4(p->H2); p->ld_out = ru4(p->NO);
    p->slabs = a->slabs; p->grad = a->grad; p->m = a->exp_avg; p->v = a->exp_avg_sq;
    p->w2t = reinterpret_cast<float*>(ws + wl.w2t[j]);
    p->w3part = reinterpret_cast<float*>(ws + wl.w3part[j]);
    p->lr = a->lr; p->weight_decay = a->weight_decay; p->clip_value = a->clip_value; p->clip_mode = a->clip_mode;
    p->opt = (OptWs*)a->opt_workspace;
    p->norm_out = a->norm_out;
    p->mode = a->mode;
    p->actions = a->actions; p->lda = a->lda; p->adv = a->adv; p->behave = a->behave_pd; p->ldb = a->ldb;
    p->ref = a->ref_pd; p->ldr = a->ldr; p->returns = a->returns;
    p->hyper = a->hyper; p->eta = a->eta; p->kl_target = a->kl_target; p->stop_threshold = a->stop_threshold;
    p->stats = a->stats; p->stop = a->stop_flag; p->epochs = a->epochs;
    p->kl_part = reinterpret_cast<double*>(ws + wl.kl_part[j]);
    p->loss_part = reinterpret_cast<double*>(ws + wl.loss_part[j]);
    p->sq_part = reinterpret_cast<double*>(ws + wl.sq_part[j]);
    p->kl_global = reinterpret_cast<double*>(ws + wl.kl_global[j]);
    p->n_rb = (a->M + RB - 1) / RB;
    p->s = pl.s[j];
    p->rps = pl.rps[j];
    if (a->mode == 2) {
        SB200_REQUIRE(a->returns != nullptr && p->NO == 1);
    } else {
        SB200_REQUIRE(a->actions && a->adv && a->behave_pd && a->ref_pd && a->hyper);
        SB200_REQUIRE(a->lda >= p->NO && a->ldb >= 2 * p->NO && a->ldr >= 2 * p->NO);
        SB200_REQUIRE(a->extra_off >= 0 && a->extra_off + p->NO <= a->n_params);
    }
    p->par = sb200_par{};
    p->par.world = 1;
    if (a->par != nullptr && a->par->world > 1) {
        if (const int e = sb200_par_check(a->par, a->n_params)) return e;
        p->par = *a->par;
    }
    return SB200_OK;
}

int e2_grid(const sb200_epochs* a) {
    const int n_sm = e2_n_sm();
    return (a != nullptr && a->grid >= 1) ? std::min(a->grid, n_sm) : n_sm;
}

}  // namespace

int sb200_epochs2_init() {
    SB200_CUDA(cudaFuncSetAttribute(ppo_epochs2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    return SB200_OK;
}

extern "C" int sb200_ppo_epochs2_supported(const sb200_epochs* a, const sb200_epochs* b) {
    const sb200_epochs* jobs[2] = {a, b};
    const int n = (b != nullptr) ? 2 : 1;
    if (a == nullptr) return 0;
    Plan pl;
    return e2_plan(jobs, n, &pl) ? 1 : 0;
}

extern "C" int sb200_ppo_epochs2_plan(const sb200_epochs* a, const sb200_epochs* b, int* out6) {
    SB200_REQUIRE(a != nullptr && out6 != nullptr);
    const sb200_epochs* jobs[2] = {a, b};
    const int n = (b != nullptr) ? 2 : 1;
    Plan pl;
    if (!e2_plan(jobs, n, &pl)) return SB200_ERR_UNSUPPORTED;
    out6[0] = e2_grid(a);
    out6[1] = pl.n_sq;
    for (int j = 0; j < 2; ++j) {
        out6[2 + 2 * j] = j < n ? pl.s[j] : 0;
        out6[3 + 2 * j] = j < n ? pl.rps[j] : 0;
    }
    return SB200_OK;
}

extern "C" size_t sb200_ppo_epochs2_workspace_bytes(const sb200_epochs* a, const sb200_epochs* b) {
    const sb200_epochs* jobs[2] = {a, b};
    if (a == nullptr || a->net == nullptr || (b != nullptr && b->net == nullptr)) return 0;
    return e2_ws(jobs, (b != nullptr) ? 2 : 1).total;
}

extern "C" int sb200_ppo_epochs2_f32(const sb200_epochs* a, const sb200_epochs* b, void* workspace, void* stream) {
    SB200_REQUIRE(a != nullptr && a->net != nullptr && workspace != nullptr && (((uintptr_t)workspace) & 255) == 0);
    SB200_REQUIRE(b == nullptr || b->net != nullptr);
    const sb200_epochs* jobs[2] = {a, b};
    const int n = (b != nullptr) ? 2 : 1;
    const int G = e2_grid(a);
    Plan pl;
    if (!e2_plan(jobs, n, &pl)) return SB200_ERR_UNSUPPORTED;
    const WsLayout wl = e2_ws(jobs, n);
    E2Params P;
    P.n_jobs = n;
    P.n_sq = pl.n_sq;
    for (int j = 0; j < n; ++j) {
        const int rc = e2_fill_job(jobs[j], &P.job[j], (unsigned char*)workspace, wl, j, pl);
        if (rc != SB200_OK) return rc;
    }
    if (n == 1) P.job[1] = P.job[0];
    P.bar = reinterpret_cast<unsigned int*>((unsigned char*)workspace + wl.bar);
    P.prof = reinterpret_cast<unsigned long long*>((unsigned char*)workspace + wl.prof);
    P.cta_prof = reinterpret_cast<unsigned long long*>((unsigned char*)workspace + wl.cta_prof);
    P.o_xs = pl.o_xs; P.o_h1 = pl.o_h1; P.o_h2 = pl.o_h2; P.o_d2 = pl.o_d2; P.o_out = pl.o_out; P.o_dp = pl.o_dp; P.o_part = pl.o_part; P.o_w3 = pl.o_w3; P.o_rows = pl.o_rows;
    P.ld_xs = pl.ld_xs; P.ld_h1s = pl.ld_h1s; P.ld_h2s = pl.ld_h2s; P.ldp = pl.ldp;
    cudaStream_t st = (cudaStream_t)stream;
    SB200_CUDA(cudaMemsetAsync(P.bar, 0, sizeof(unsigned int), st));
    ppo_epochs2_kernel<<<G, E2T, pl.smem_bytes, st>>>(P);
    return sb200_launch_status();
}

/* Phase profile of the launches so far on this workspace: 2 x 16 accumulated clock64 cycles (CTA 0, last CTA); slots:
 * 0 setup, 1 P1, 2 barrier, 3 gate + statistics, 4 P2, 5 barrier, 6 P3, 7 barrier, 8 P4, 9 barrier.  reset != 0 clears them. */
extern "C" int sb200_ppo_epochs2_profile(void* workspace, uint64_t* out32, int reset, void* stream) {
    SB200_REQUIRE(workspace != nullptr && out32 != nullptr);
    unsigned char* ws = (unsigned char*)workspace;
    const size_t off = 256;                                   // WsLayout: bar (256 B) then the profile block
    SB200_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    SB200_CUDA(cudaMemcpy(out32, ws + off, 32 * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    if (reset) SB200_CUDA(cudaMemset(ws + off, 0, 32 * sizeof(uint64_t)));
    return SB200_OK;
}

/* per-CTA cycles (E2_MAX_G x 8 uint64: 0 P1, 1 P2, 2 forward, 3 forward GEMMs, 4 loss rows + d2, 5 d1 GEMM); cleared on read */
extern "C" int sb200_ppo_epochs2_cta_profile(void* workspace, uint64_t* out, void* stream) {
    SB200_REQUIRE(workspace != nullptr && out != nullptr);
    unsigned char* ws = (unsigned char*)workspace + 512;     // bar (256 B) | profile (256 B) | per-CTA block
    SB200_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    SB200_CUDA(cudaMemcpy(out, ws, (size_t)E2_MAX_G * 8 * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    SB200_CUDA(cudaMemset(ws, 0, (size_t)E2_MAX_G * 8 * sizeof(uint64_t)));
    return SB200_OK;
}
