// Fused MLP forward (z-filter -> [Linear + activation] x L) on row tiles, fp32 SIMT FFMA.
//
// One CTA owns BM = 8*TM rows and walks the layers; activations never leave shared memory (two
// ping-pong buffers), weights stream through a double-buffered cp.async stage of BK x 256 floats.
// Thread (ty = warp, tx = lane) accumulates a TM x 8 register tile: rows ty*TM.., columns
// n0 + tx*4 + {0..3} and n0 + 128 + tx*4 + {0..3}; A fragments are warp-broadcast LDS.128 along k,
// B fragments are conflict-free LDS.128.  Layers with <= 32 outputs (policy mean, value head) take a
// warp-per-row dot-product path instead of a 256-wide pass.
//
// Replaces the stock-torch calls of surreal/model/ppo_net.py:253-315, builders.py:114-132,160-175,
// 35-84 and the z-filter of z_filter.py:59-79.  Algorithmic HBM bytes per row: 4*D read + saved
// activations written (critic pass: 4 bytes); weights are L2-resident.
#include "common.cuh"
#include <stdlib.h>

namespace {

constexpr int PASS_N = 256;
// k-chunk rows per cp.async stage: 16 for the big-tile (compute-bound) variants, 64 for the small-row-tile
// variants whose wall time is a chain of L2 round trips (fewer, larger stages = fewer exposed latencies).

struct FwdParams {
    const float* x;
    const float* x_next;
    long long ldx;
    long long rows;
    int win_n;
    const float* aux;
    long long aux_ld;
    int aux_layer;
    int aux_dim;
    const float* zf;
    float zf_eps;
    float* save_x;
    long long ld_save_x;
    int n_layers;
    int dims[SB200_MAX_LAYERS + 1];
    int act[SB200_MAX_LAYERS];
    const float* W[SB200_MAX_LAYERS];
    const float* b[SB200_MAX_LAYERS];
    int ldw[SB200_MAX_LAYERS];
    float* save[SB200_MAX_LAYERS];
    long long ld_save[SB200_MAX_LAYERS];
    int ldh;
    int scratch_floats;
    const float* ln_g[SB200_MAX_LAYERS];     // LayerNorm after layer l (sb200_mlp.ln_g / ln_b), nullptr: none
    const float* ln_b[SB200_MAX_LAYERS];
    float ln_eps;
    float* ln_save[SB200_MAX_LAYERS];        // sb200_rows.ln_save / ln_stats
    long long ld_ln_save[SB200_MAX_LAYERS];
    float* ln_stats[SB200_MAX_LAYERS];
};

__host__ __device__ inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

__device__ __forceinline__ float apply_act(float v, int act) {
    if (act == SB200_ACT_RELU) return fmaxf(v, 0.0f);
    if (act == SB200_ACT_TANH) return tanhf(v);
    return v;
}

// LayerNorm epilogue of layer l on the tile's `rows` activation rows H[m][0, N) in shared memory, in place, a warp per
// row: two-pass mean / biased variance (exact for all-zero rows: y == b), y = fma((h - mean) * rstd, g, b).  Runs after
// the layer's barrier and before the next layer reads H; columns >= N are not touched.  Not inlined: the GEMM loops
// around it keep their register allocation.
__device__ __noinline__ void ln_epilogue(const FwdParams& p, int l, float* H, int ldh, int rows, long long row0) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int N = p.dims[l + 1];
    const float* __restrict__ g = p.ln_g[l];
    const float* __restrict__ b = p.ln_b[l];
    float* sv = p.ln_save[l];
    float* st = p.ln_stats[l];
    const long long lds = p.ld_ln_save[l];
    for (int m = warp; m < rows; m += SB200_THREADS / 32) {
        float* hr = H + m * ldh;
        float s = 0.0f;
        for (int j = lane; j < N; j += 32) s += hr[j];
        const float mean = warp_sum(s) / (float)N;
        float q = 0.0f;
        for (int j = lane; j < N; j += 32) {
            const float d = hr[j] - mean;
            q = fmaf(d, d, q);
        }
        const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)N + p.ln_eps);
        const long long r = row0 + m;
        const bool keep = r < p.rows;
        for (int j = lane; j < N; j += 32) {
            const float y = fmaf((hr[j] - mean) * rstd, __ldg(g + j), __ldg(b + j));
            hr[j] = y;
            if (sv != nullptr && keep) sv[r * lds + j] = y;
        }
        if (st != nullptr && keep && lane == 0) {
            st[2 * r] = mean;
            st[2 * r + 1] = rstd;
        }
    }
}

template <int TM, int BK>
__global__ void __launch_bounds__(SB200_THREADS, (TM <= 4 && BK == 16) ? 2 : 1) mlp_fwd_kernel(const __grid_constant__ FwdParams p) {
    constexpr int BM = 8 * TM;
    extern __shared__ __align__(16) float smem[];
    const int ldh = p.ldh;
    float* Hin = smem;
    float* Hout = smem + BM * ldh;
    float* Ws = smem + 2 * BM * ldh;   // [2][BK][PASS_N]
    const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
    const long long row0 = (long long)blockIdx.x * BM;

    // ---- stage 0: input tile (+ optional z-filter, + optional aux columns for layer 0)
    const int K0 = p.dims[0];
    if (p.zf != nullptr) {             // per-column mean / std once per CTA (scratch: the W stage)
        const float cnt = p.zf[2 * K0];
        for (int k = tid; k < K0; k += SB200_THREADS) {
            const float mean = p.zf[k] / cnt;
            const float var = p.zf[K0 + k] / cnt - mean * mean;
            Ws[k] = mean;
            Ws[K0 + k] = fmaxf(sqrtf(var), p.zf_eps);
        }
        __syncthreads();
    }
    {
        const int in_w = K0 + (p.aux_layer == 0 ? p.aux_dim : 0);
        const int in_wp = round_up(in_w, BK);
        for (int idx = tid; idx < BM * in_wp; idx += SB200_THREADS) {
            const int m = idx / in_wp, k = idx - m * in_wp;
            const long long r = row0 + m;
            float v = 0.0f;
            if (r < p.rows) {
                if (k < K0) {
                    const float* src;
                    if (p.win_n > 0) {
                        const long long b = r / (p.win_n + 1);
                        const int kk = (int)(r - b * (p.win_n + 1));
                        src = (kk < p.win_n) ? p.x + (b * p.win_n + kk) * p.ldx : p.x_next + b * p.ldx;
                    } else {
                        src = p.x + r * p.ldx;
                    }
                    v = src[k];
                    if (p.zf != nullptr) v = fminf(fmaxf((v - Ws[k]) / Ws[K0 + k], -5.0f), 5.0f);
                } else if (k < in_w) {
                    v = p.aux[r * p.aux_ld + (k - K0)];
                }
            }
            Hin[m * ldh + k] = v;
            if (p.save_x != nullptr && r < p.rows && k < K0) p.save_x[r * p.ld_save_x + k] = v;
        }
    }
    __syncthreads();

    for (int l = 0; l < p.n_layers; ++l) {
        const int K = p.dims[l] + (p.aux_layer == l ? p.aux_dim : 0);
        const int N = p.dims[l + 1];
        const float* __restrict__ W = p.W[l];
        const float* __restrict__ bias = p.b[l];
        const int ldw = p.ldw[l];
        const int act = p.act[l];
        const bool last = (l == p.n_layers - 1);
        float* sv = p.save[l];
        const long long lds = p.ld_save[l];

        if (N > 32) {
            // ------------------------------ wide path: 256-column passes ------------------------------
            const int nchunks = (K + BK - 1) / BK;
            const bool vec_ok = sv != nullptr && (lds % 4 == 0) && ((((uintptr_t)sv) & 15) == 0);
            for (int n0 = 0; n0 < N; n0 += PASS_N) {
                float acc[TM][8];
#pragma unroll
                for (int i = 0; i < TM; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
                const bool hi = (n0 + 128 < N);

                auto load_chunk = [&](int stage, int k0) {
                    float* dst = Ws + stage * (BK * PASS_N);
#pragma unroll
                    for (int i = 0; i < (BK * PASS_N / 4) / SB200_THREADS; ++i) {
                        const int f = tid + i * SB200_THREADS;
                        const int kr = f >> 6, c4 = f & 63;
                        const int k = k0 + kr, n = n0 + c4 * 4;
                        const bool ok = (k < K) && (n < ldw);
                        const float* src = ok ? (W + (long long)k * ldw + n) : W;
                        cp_async16(dst + kr * PASS_N + c4 * 4, src, ok ? 16 : 0);
                    }
                };

                load_chunk(0, 0);
                cp_async_commit();
                for (int c = 0; c < nchunks; ++c) {
                    if (c + 1 < nchunks) load_chunk((c + 1) & 1, (c + 1) * BK);
                    cp_async_commit();
                    cp_async_wait<1>();
                    __syncthreads();
                    const float* Wst = Ws + (c & 1) * (BK * PASS_N);
                    const float* A = Hin + (ty * TM) * ldh + c * BK;
#pragma unroll
                    for (int kk = 0; kk < BK; kk += 4) {
                        float4 a[TM];
#pragma unroll
                        for (int i = 0; i < TM; ++i) a[i] = *reinterpret_cast<const float4*>(A + i * ldh + kk);
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const float4 b0 = *reinterpret_cast<const float4*>(Wst + (kk + j) * PASS_N + tx * 4);
#pragma unroll
                            for (int i = 0; i < TM; ++i) {
                                const float av = (j == 0) ? a[i].x : (j == 1) ? a[i].y : (j == 2) ? a[i].z : a[i].w;
                                acc[i][0] = fmaf(av, b0.x, acc[i][0]);
                                acc[i][1] = fmaf(av, b0.y, acc[i][1]);
                                acc[i][2] = fmaf(av, b0.z, acc[i][2]);
                                acc[i][3] = fmaf(av, b0.w, acc[i][3]);
                            }
                            if (hi) {
                                const float4 b1 =
                                    *reinterpret_cast<const float4*>(Wst + (kk + j) * PASS_N + 128 + tx * 4);
#pragma unroll
                                for (int i = 0; i < TM; ++i) {
                                    const float av =
                                        (j == 0) ? a[i].x : (j == 1) ? a[i].y : (j == 2) ? a[i].z : a[i].w;
                                    acc[i][4] = fmaf(av, b1.x, acc[i][4]);
                                    acc[i][5] = fmaf(av, b1.y, acc[i][5]);
                                    acc[i][6] = fmaf(av, b1.z, acc[i][6]);
                                    acc[i][7] = fmaf(av, b1.w, acc[i][7]);
                                }
                            }
                        }
                    }
                    __syncthreads();
                }
                cp_async_wait<0>();

                // epilogue: bias + activation -> next activation buffer (+ optional global save)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int n = n0 + h * 128 + tx * 4;
                    if (n >= round_up(N, 4)) continue;
                    float bv[4];
#pragma unroll
                    for (int c = 0; c < 4; ++c) bv[c] = (n + c < N) ? bias[n + c] : 0.0f;
#pragma unroll
                    for (int i = 0; i < TM; ++i) {
                        const int m = ty * TM + i;
                        float4 o;
                        o.x = (n + 0 < N) ? apply_act(acc[i][h * 4 + 0] + bv[0], act) : 0.0f;
                        o.y = (n + 1 < N) ? apply_act(acc[i][h * 4 + 1] + bv[1], act) : 0.0f;
                        o.z = (n + 2 < N) ? apply_act(acc[i][h * 4 + 2] + bv[2], act) : 0.0f;
                        o.w = (n + 3 < N) ? apply_act(acc[i][h * 4 + 3] + bv[3], act) : 0.0f;
                        if (!last) *reinterpret_cast<float4*>(Hout + m * ldh + n) = o;
                        const long long r = row0 + m;
                        if (sv != nullptr && r < p.rows) {
                            float* dst = sv + r * lds + n;
                            if (vec_ok && n + 3 < N) {
                                *reinterpret_cast<float4*>(dst) = o;
                            } else {
                                if (n + 0 < N) dst[0] = o.x;
                                if (n + 1 < N) dst[1] = o.y;
                                if (n + 2 < N) dst[2] = o.z;
                                if (n + 3 < N) dst[3] = o.w;
                            }
                        }
                    }
                }
            }
        } else {
            // ------------------------------ narrow path: N <= 32 ------------------------------------
            // warp ty owns rows ty*TM..; lanes split k; 8 outputs at a time, shuffle-reduced.
            // The head's weights (K x ldw floats, e.g. 8 KB) are staged once per CTA in the (idle) W stage.
            const float* Wn = W;
            if (K * ldw <= 2 * BK * PASS_N) {
                for (int f = tid; f < (K * ldw) / 4; f += SB200_THREADS) cp_async16(Ws + f * 4, W + f * 4, 16);
                cp_async_commit();
                cp_async_wait<0>();
                __syncthreads();
                Wn = Ws;
            }
            for (int i = 0; i < TM; ++i) {
                const int m = ty * TM + i;
                const long long r = row0 + m;
                const float* hrow = Hin + m * ldh;
                for (int n8 = 0; n8 < N; n8 += 8) {
                    float s[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) s[j] = 0.0f;
                    const bool second = (n8 + 4 < ldw);
                    for (int k = tx; k < K; k += 32) {
                        const float hv = hrow[k];
                        const float* wr = Wn + (long long)k * ldw + n8;
                        const float4 w0 = *reinterpret_cast<const float4*>(wr);
                        s[0] = fmaf(hv, w0.x, s[0]);
                        s[1] = fmaf(hv, w0.y, s[1]);
                        s[2] = fmaf(hv, w0.z, s[2]);
                        s[3] = fmaf(hv, w0.w, s[3]);
                        if (second) {
                            const float4 w1 = *reinterpret_cast<const float4*>(wr + 4);
                            s[4] = fmaf(hv, w1.x, s[4]);
                            s[5] = fmaf(hv, w1.y, s[5]);
                            s[6] = fmaf(hv, w1.z, s[6]);
                            s[7] = fmaf(hv, w1.w, s[7]);
                        }
                    }
                    float mine = 0.0f;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float t = warp_sum(s[j]);
                        if (tx == j) mine = t;
                    }
                    const int n = n8 + tx;
                    if (tx < 8 && n < N) {
                        const float o = apply_act(mine + bias[n], act);
                        if (!last) Hout[m * ldh + n] = o;
                        if (sv != nullptr && r < p.rows) sv[r * lds + n] = o;
                    }
                }
            }
        }
        __syncthreads();
        if (!last) {
            if (p.ln_g[l] != nullptr) ln_epilogue(p, l, Hout, ldh, BM, row0);
            // columns [N, N+aux) <- aux input of the next layer; [.., pad16) <- 0
            const int auxd = (p.aux_layer == l + 1) ? p.aux_dim : 0;
            const int wp = round_up(N + auxd, BK);
            const int span = wp - N;
            if (span > 0) {
                for (int idx = tid; idx < BM * span; idx += SB200_THREADS) {
                    const int m = idx / span, c = N + (idx - m * span);
                    const long long r = row0 + m;
                    float v = 0.0f;
                    if (c < N + auxd && r < p.rows) v = p.aux[r * p.aux_ld + (c - N)];
                    Hout[m * ldh + c] = v;
                }
            }
            __syncthreads();
            float* t = Hin;
            Hin = Hout;
            Hout = t;
        }
    }
}


// ------------------------------------------------------------------------------------------------------
// Skinny variant for small batches (rows <= ~2K: one env step of all actors, one learner minibatch).
// There a forward is a chain of latency-bound steps, and the big-tile mapping re-reads every weight fragment
// from shared memory in all 8 warps.  Here a CTA owns R = 8 rows and thread t owns output column n0 + t:
// weights are read exactly once per CTA, coalesced (one 128-byte line per warp per k), straight from L2 with
// a register double buffer of 8 k-steps (no shared-memory staging, no barriers inside a layer); the 8 input
// rows are warp-broadcast LDS.128 along k.  Each CTA starts its k loop at a rotated offset (see below).
constexpr int SK_R = 8;
constexpr int SK_U = 8;      // k-steps per register stage
constexpr int SK_D = 4;      // register stages in flight

__global__ void __launch_bounds__(SB200_THREADS, 2) mlp_fwd_skinny_kernel(const __grid_constant__ FwdParams p) {
    extern __shared__ __align__(16) float smem[];
    const int ldh = p.ldh;
    float* Hin = smem;
    float* Hout = smem + SK_R * ldh;
    float* Wsc = smem + 2 * SK_R * ldh;                 // scratch: z-filter columns, then the narrow head's weights
    const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
    const long long row0 = (long long)blockIdx.x * SK_R;
    const int K0 = p.dims[0];
    if (p.zf != nullptr) {
        const float cnt = p.zf[2 * K0];
        for (int k = tid; k < K0; k += SB200_THREADS) {
            const float mean = p.zf[k] / cnt;
            const float var = p.zf[K0 + k] / cnt - mean * mean;
            Wsc[k] = mean;
            Wsc[K0 + k] = fmaxf(sqrtf(var), p.zf_eps);
        }
        __syncthreads();
    }
    {
        const int in_w = K0 + (p.aux_layer == 0 ? p.aux_dim : 0);
        const int in_wp = round_up(in_w, SK_U * SK_D);
        for (int idx = tid; idx < SK_R * in_wp; idx += SB200_THREADS) {
            const int m = idx / in_wp, k = idx - m * in_wp;
            const long long r = row0 + m;
            float v = 0.0f;
            if (r < p.rows) {
                if (k < K0) {
                    const float* src;
                    if (p.win_n > 0) {
                        const long long b = r / (p.win_n + 1);
                        const int kk = (int)(r - b * (p.win_n + 1));
                        src = (kk < p.win_n) ? p.x + (b * p.win_n + kk) * p.ldx : p.x_next + b * p.ldx;
                    } else {
                        src = p.x + r * p.ldx;
                    }
                    v = src[k];
                    if (p.zf != nullptr) v = fminf(fmaxf((v - Wsc[k]) / Wsc[K0 + k], -5.0f), 5.0f);
                } else if (k < in_w) {
                    v = p.aux[r * p.aux_ld + (k - K0)];
                }
            }
            Hin[m * ldh + k] = v;
            if (p.save_x != nullptr && r < p.rows && k < K0) p.save_x[r * p.ld_save_x + k] = v;
        }
    }
    __syncthreads();

    for (int l = 0; l < p.n_layers; ++l) {
        const int K = p.dims[l] + (p.aux_layer == l ? p.aux_dim : 0);
        const int N = p.dims[l + 1];
        const float* __restrict__ W = p.W[l];
        const float* __restrict__ bias = p.b[l];
        const int ldw = p.ldw[l];
        const int act = p.act[l];
        const bool last = (l == p.n_layers - 1);
        float* sv = p.save[l];
        const long long lds = p.ld_save[l];
        if (N > 32) {
            const int Kp = round_up(K, SK_U * SK_D);
            for (int n0 = 0; n0 < N; n0 += SB200_THREADS) {
                const int n = n0 + tid;
                const bool on = n < N;
                float acc[SK_R];
#pragma unroll
                for (int r = 0; r < SK_R; ++r) acc[r] = 0.0f;
                const float* wp = W + (on ? n : 0);
                // Register ring of SK_D stages x SK_U k-steps: ~24 weight loads per thread stay in flight, enough to
                // cover the L2 round trip (a single look-ahead stage left every iteration exposed to ~1 us of latency).
                // Every CTA needs the SAME weight rows; each starts its k loop at a different stage and wraps around
                // so that the CTAs do not hit the same L2 lines in lock-step.  The summation order of a row therefore
                // depends on its CTA index only (deterministic run to run).
                float w[SK_D][SK_U];
                const int nst = Kp / SK_U;                         // multiple of SK_D (Kp is padded to SK_U*SK_D)
                const int rot = (int)(((unsigned)blockIdx.x * 5u) % (unsigned)nst);
                auto stage_k0 = [&](int it) { int s_ = rot + it; if (s_ >= nst) s_ -= nst; return s_ * SK_U; };
                auto load_stage = [&](float (&dst)[SK_U], int it) {
                    const int k0 = stage_k0(it);
#pragma unroll
                    for (int u = 0; u < SK_U; ++u) {
                        const int k = k0 + u;
                        dst[u] = (on && it < nst && k < K) ? __ldg(wp + (long long)k * ldw) : 0.0f;
                    }
                };
                auto consume = [&](const float (&ws)[SK_U], int it) {
                    const int k0 = stage_k0(it);
#pragma unroll
                    for (int r = 0; r < SK_R; ++r) {
                        const float4 a0 = *reinterpret_cast<const float4*>(Hin + r * ldh + k0);
                        const float4 a1 = *reinterpret_cast<const float4*>(Hin + r * ldh + k0 + 4);
                        float t = acc[r];
                        t = fmaf(a0.x, ws[0], t); t = fmaf(a0.y, ws[1], t); t = fmaf(a0.z, ws[2], t); t = fmaf(a0.w, ws[3], t);
                        t = fmaf(a1.x, ws[4], t); t = fmaf(a1.y, ws[5], t); t = fmaf(a1.z, ws[6], t); t = fmaf(a1.w, ws[7], t);
                        acc[r] = t;
                    }
                };
#pragma unroll
                for (int d = 0; d < SK_D - 1; ++d) load_stage(w[d], d);
                for (int it = 0; it < nst; it += SK_D) {
#pragma unroll
                    for (int d = 0; d < SK_D; ++d) {
                        load_stage(w[(d + SK_D - 1) % SK_D], it + d + SK_D - 1);
                        consume(w[d], it + d);
                    }
                }
                if (on) {
                    const float bv = bias[n];
#pragma unroll
                    for (int r = 0; r < SK_R; ++r) {
                        const float o = apply_act(acc[r] + bv, act);
                        if (!last) Hout[r * ldh + n] = o;
                        const long long rr = row0 + r;
                        if (sv != nullptr && rr < p.rows) sv[rr * lds + n] = o;
                    }
                }
            }
        } else {
            // narrow head: warp ty owns row ty; weights staged once in shared memory
            const float* Wn = W;
            __syncthreads();                               // Wsc may still hold z-filter columns in use
            if (K * ldw <= p.scratch_floats) {
                for (int f = tid; f < (K * ldw) / 4; f += SB200_THREADS) cp_async16(Wsc + f * 4, W + f * 4, 16);
                cp_async_commit();
                cp_async_wait<0>();
                __syncthreads();
                Wn = Wsc;
            }
            const int m = ty;                              // SK_R == number of warps
            const long long r = row0 + m;
            const float* hrow = Hin + m * ldh;
            for (int n8 = 0; n8 < N; n8 += 8) {
                float s8[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) s8[j] = 0.0f;
                const bool second = (n8 + 4 < ldw);
                for (int k = tx; k < K; k += 32) {
                    const float hv = hrow[k];
                    const float* wr = Wn + (long long)k * ldw + n8;
                    const float4 w0 = *reinterpret_cast<const float4*>(wr);
                    s8[0] = fmaf(hv, w0.x, s8[0]); s8[1] = fmaf(hv, w0.y, s8[1]);
                    s8[2] = fmaf(hv, w0.z, s8[2]); s8[3] = fmaf(hv, w0.w, s8[3]);
                    if (second) {
                        const float4 w1 = *reinterpret_cast<const float4*>(wr + 4);
                        s8[4] = fmaf(hv, w1.x, s8[4]); s8[5] = fmaf(hv, w1.y, s8[5]);
                        s8[6] = fmaf(hv, w1.z, s8[6]); s8[7] = fmaf(hv, w1.w, s8[7]);
                    }
                }
                float mine = 0.0f;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float t = warp_sum(s8[j]);
                    if (tx == j) mine = t;
                }
                const int n = n8 + tx;
                if (tx < 8 && n < N) {
                    const float o = apply_act(mine + bias[n], act);
                    if (!last) Hout[m * ldh + n] = o;
                    if (sv != nullptr && r < p.rows) sv[r * lds + n] = o;
                }
            }
        }
        __syncthreads();
        if (!last) {
            if (p.ln_g[l] != nullptr) ln_epilogue(p, l, Hout, ldh, SK_R, row0);
            const int auxd = (p.aux_layer == l + 1) ? p.aux_dim : 0;
            const int wp2 = round_up(N + auxd, SK_U * SK_D);
            const int span = wp2 - N;
            if (span > 0) {
                for (int idx = tid; idx < SK_R * span; idx += SB200_THREADS) {
                    const int m = idx / span, c = N + (idx - m * span);
                    const long long r = row0 + m;
                    float v = 0.0f;
                    if (c < N + auxd && r < p.rows) v = p.aux[r * p.aux_ld + (c - N)];
                    Hout[m * ldh + c] = v;
                }
            }
            __syncthreads();
            float* t = Hin;
            Hin = Hout;
            Hout = t;
        }
    }
}

}  // namespace

#include "mlp_fwd_mma.cuh"
#include "mlp_fwd_pk.cuh"

namespace {

constexpr size_t SMEM_BUDGET = 200 * 1024;

template <int TM, int BK>
int launch_fwd(FwdParams p, int maxw, cudaStream_t st) {
    constexpr int BM = 8 * TM;
    p.ldh = round_up(maxw, BK) + 4;
    const size_t smem = (size_t)(2 * BM * p.ldh + 2 * BK * PASS_N) * sizeof(float);
    const long long grid = (p.rows + BM - 1) / BM;
    mlp_fwd_kernel<TM, BK><<<(unsigned)grid, SB200_THREADS, smem, st>>>(p);
    return sb200_launch_status();
}

}  // namespace

int g_forward_mode = [] { const char* e = getenv("SB200_MMA"); return e ? atoi(e) : 1; }();

extern "C" int sb200_set_forward_mode(int mode) {
    if (mode != 0 && mode != 1) return SB200_ERR_ARG;
    g_forward_mode = mode;
    return SB200_OK;
}

// called once from sb200_init(): opt every instantiation into the full dynamic shared-memory budget
int sb200_mlp_fwd_init() {
    SB200_CUDA(cudaFuncSetAttribute(mlp_fwd_mma_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BUDGET));
    SB200_CUDA(cudaFuncSetAttribute(mlp_fwd_mma_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BUDGET));
    SB200_CUDA(cudaFuncSetAttribute(mlp_fwd_mma_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BUDGET));
    SB200_CUDA(cudaFuncSetAttribute(mlp_fwd_pk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 225 * 1024));
    SB200_CUDA(cudaFuncSetAttribute(mlp_fwd_skinny_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    SB200_CUDA(cudaFuncSetAttribute(mlp_fwd_kernel<1, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BUDGET));
    SB200_CUDA(cudaFuncSetAttribute(mlp_fwd_kernel<2, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BUDGET));
    SB200_CUDA(cudaFuncSetAttribute(mlp_fwd_kernel<1, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BUDGET));
    SB200_CUDA(cudaFuncSetAttribute(mlp_fwd_kernel<2, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BUDGET));
    SB200_CUDA(cudaFuncSetAttribute(mlp_fwd_kernel<4, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BUDGET));
    SB200_CUDA(cudaFuncSetAttribute(mlp_fwd_kernel<8, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BUDGET));
    return SB200_OK;
}

// Validates the descriptors and fills the kernel parameter block; *maxw = widest layer input.
static int fill_fwd_params(const sb200_mlp* net, const sb200_zfilter* zf, const sb200_rows* in, float* const* save,
                           const int64_t* ld_save, FwdParams& p, int* maxw_out) {
    SB200_REQUIRE(net != nullptr && in != nullptr);
    SB200_REQUIRE(net->n_layers >= 1 && net->n_layers <= SB200_MAX_LAYERS);
    SB200_REQUIRE(in->rows >= 0 && in->x != nullptr);
    p.scratch_floats = 0;
    p.ldh = 0;
    p.x = in->x;
    p.x_next = in->x_next;
    p.ldx = in->ldx;
    p.rows = in->rows;
    p.win_n = in->win_n;
    SB200_REQUIRE(p.win_n == 0 || (p.x_next != nullptr && p.rows % (p.win_n + 1) == 0));
    p.aux = in->aux;
    p.aux_ld = in->aux_ld;
    p.aux_layer = net->aux_layer;
    p.aux_dim = (net->aux_layer >= 0) ? net->aux_dim : 0;
    SB200_REQUIRE(net->aux_layer < net->n_layers);
    SB200_REQUIRE(p.aux_layer < 0 || (p.aux != nullptr && p.aux_dim > 0));
    p.zf = (zf != nullptr) ? zf->stats : nullptr;
    p.zf_eps = (zf != nullptr) ? zf->eps : 0.0f;
    p.save_x = in->save_x;
    p.ld_save_x = in->ld_save_x;
    SB200_REQUIRE(p.save_x == nullptr || p.ld_save_x >= net->dims[0]);
    p.n_layers = net->n_layers;
    SB200_REQUIRE(net->dims[0] >= 1 && net->dims[0] <= 4096 && p.ldx >= net->dims[0]);
    int maxw = 0;
    for (int l = 0; l <= net->n_layers; ++l) p.dims[l] = net->dims[l];
    for (int l = 0; l < SB200_MAX_LAYERS; ++l) {
        const bool on = l < net->n_layers;
        p.act[l] = on ? net->act[l] : 0;
        p.W[l] = on ? net->W[l] : nullptr;
        p.b[l] = on ? net->b[l] : nullptr;
        p.ldw[l] = on ? net->ldw[l] : 0;
        p.save[l] = (on && save != nullptr) ? save[l] : nullptr;
        p.ld_save[l] = (on && save != nullptr && ld_save != nullptr) ? ld_save[l] : 0;
        p.ln_g[l] = on ? net->ln_g[l] : nullptr;
        p.ln_b[l] = on ? net->ln_b[l] : nullptr;
        p.ln_save[l] = p.ln_g[l] != nullptr ? in->ln_save[l] : nullptr;
        p.ld_ln_save[l] = p.ln_g[l] != nullptr ? in->ld_ln_save[l] : 0;
        p.ln_stats[l] = p.ln_g[l] != nullptr ? in->ln_stats[l] : nullptr;
        if (on) {
            SB200_REQUIRE(p.W[l] != nullptr && p.b[l] != nullptr);
            SB200_REQUIRE((p.ln_g[l] == nullptr) == (p.ln_b[l] == nullptr));
            SB200_REQUIRE(p.ln_g[l] == nullptr || (l + 1 < net->n_layers && net->ln_eps > 0.0f));
            SB200_REQUIRE(p.ln_save[l] == nullptr || p.ld_ln_save[l] >= p.dims[l + 1]);
            SB200_REQUIRE(p.dims[l + 1] >= 1 && p.ldw[l] >= p.dims[l + 1] && p.ldw[l] % 4 == 0);
            SB200_REQUIRE((((uintptr_t)p.W[l]) & 15) == 0);
            SB200_REQUIRE(p.save[l] == nullptr || p.ld_save[l] >= p.dims[l + 1]);
            const int w = p.dims[l] + (p.aux_layer == l ? p.aux_dim : 0);
            if (w > maxw) maxw = w;
        }
    }
    for (int l = net->n_layers; l < SB200_MAX_LAYERS; ++l) SB200_REQUIRE(net->ln_g[l] == nullptr && net->ln_b[l] == nullptr);
    p.ln_eps = net->ln_eps;
    *maxw_out = maxw;
    return SB200_OK;
}

// ---- packed small-batch inference path (mlp_fwd_pk.cuh) --------------------------------------------------------
static long long pack_layer_floats(const sb200_mlp* net, int l) {
    if (net->dims[l + 1] <= 32) return 0;
    const int K = net->dims[l] + (net->aux_layer == l ? net->aux_dim : 0);
    return (long long)PK_CS * pk_nst(K) * pk_ntl(net->dims[l + 1]) * 64;
}

// Shared-memory plan of mlp_fwd_pk_kernel (floats); false when the architecture does not fit one SM.
static bool pack_plan(const sb200_mlp* net, bool zf, PkParams* pp, size_t* smem_bytes) {
    if (net == nullptr || net->n_layers < 1 || net->n_layers > SB200_MAX_LAYERS) return false;
    if (sb200_mlp_has_ln(net)) return false;          // no LayerNorm epilogue in mlp_fwd_pk_kernel
    for (int l = 0; l + 1 < net->n_layers; ++l)
        if (net->dims[l + 1] <= 32) return false;        // wide layers first, a narrow layer only as the last one
    long long off = 0;
    int ldp = 4, head = 0;
    int offW[SB200_MAX_LAYERS] = {0}, offA[SB200_MAX_LAYERS] = {0};
    for (int l = 0; l < net->n_layers; ++l) {
        const int K = net->dims[l] + (net->aux_layer == l ? net->aux_dim : 0);
        if (net->dims[l + 1] > 32) {
            offW[l] = (int)off;
            off += pack_layer_floats(net, l) / PK_CS;
            offA[l] = (int)off;
            off += 2LL * PK_MT * pk_nst(K) * 128;
        } else {
            ldp = round_up(K, 4) + 4;
            head = K * net->ldw[l];
        }
    }
    const int offHp = (int)off;
    off += (long long)PK_ROWS * ldp;
    const int zf_floats = zf ? round_up(2 * net->dims[0], 4) : 0;
    const int scratch = round_up(zf_floats + ((head <= 16384) ? head : 0) + 4, 4);
    const int offScratch = (int)off;
    off += scratch;
    if ((size_t)off * sizeof(float) > 225 * 1024) return false;
    if (pp != nullptr) {
        for (int l = 0; l < SB200_MAX_LAYERS; ++l) {
            pp->offW[l] = offW[l];
            pp->offA[l] = offA[l];
        }
        pp->offHp = offHp;
        pp->offScratch = offScratch;
        pp->ldp = ldp;
        pp->f.scratch_floats = scratch;
    }
    if (smem_bytes != nullptr) *smem_bytes = (size_t)off * sizeof(float);
    return true;
}

extern "C" size_t sb200_mlp_pack_floats(const sb200_mlp* net) {
    if (!pack_plan(net, true, nullptr, nullptr)) return 0;
    long long tot = 0;
    for (int l = 0; l < net->n_layers; ++l) tot += pack_layer_floats(net, l);
    return (size_t)(tot > 0 ? tot : 4);
}

extern "C" int sb200_mlp_pack_tf32(const sb200_mlp* net, float* packed, void* stream) {
    SB200_REQUIRE(packed != nullptr && (((uintptr_t)packed) & 15) == 0);
    if (!pack_plan(net, true, nullptr, nullptr)) return SB200_ERR_UNSUPPORTED;
    long long off = 0;
    int launches = 0;
    for (int l = 0; l < net->n_layers; ++l) {
        const long long fl = pack_layer_floats(net, l);
        if (fl == 0) continue;
        const int K = net->dims[l] + (net->aux_layer == l ? net->aux_dim : 0);
        const long long items = fl / 2;
        mlp_pack_tf32_kernel<<<(unsigned)((items + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
            net->W[l], K, net->dims[l + 1], net->ldw[l], reinterpret_cast<float2*>(packed + off));
        off += fl;
        ++launches;
    }
    if (launches == 0) return SB200_OK;
    return sb200_launch_status(launches);
}

extern "C" int sb200_mlp_forward_packed_f32(const sb200_mlp* net, const float* packed, const sb200_zfilter* zf,
                                            const sb200_rows* in, float* out, int64_t ld_out, void* stream) {
    SB200_REQUIRE(packed != nullptr && out != nullptr && (((uintptr_t)packed) & 15) == 0);
    PkParams pp;
    int maxw = 0;
    const int rc = fill_fwd_params(net, zf, in, nullptr, nullptr, pp.f, &maxw);
    if (rc != SB200_OK) return rc;
    size_t smem = 0;
    if (!pack_plan(net, pp.f.zf != nullptr, &pp, &smem)) return SB200_ERR_UNSUPPORTED;
    if (in->rows == 0) return SB200_OK;
    SB200_REQUIRE(in->save_x == nullptr && ld_out >= net->dims[net->n_layers]);
    long long off = 0;
    for (int l = 0; l < SB200_MAX_LAYERS; ++l) {
        pp.P[l] = nullptr;
        if (l >= net->n_layers) continue;
        const long long fl = pack_layer_floats(net, l);
        if (fl > 0) {
            pp.P[l] = packed + off;
            off += fl;
        }
    }
    pp.out = out;
    pp.ld_out = ld_out;
    const long long clusters = (in->rows + PK_ROWS - 1) / PK_ROWS;
    mlp_fwd_pk_kernel<<<(unsigned)(PK_CS * clusters), SB200_THREADS, smem, (cudaStream_t)stream>>>(pp);
    return sb200_launch_status();
}

static int mlp_forward_impl(const sb200_mlp* net, const sb200_zfilter* zf, const sb200_rows* in, float* const* save,
                            const int64_t* ld_save, int variant, void* stream);

extern "C" int sb200_mlp_forward_f32(const sb200_mlp* net, const sb200_zfilter* zf, const sb200_rows* in,
                                     float* const* save, const int64_t* ld_save, void* stream) {
    return mlp_forward_impl(net, zf, in, save, ld_save, 0, stream);
}

extern "C" int sb200_mlp_forward_variant_f32(const sb200_mlp* net, const sb200_zfilter* zf, const sb200_rows* in,
                                             float* const* save, const int64_t* ld_save, int variant, void* stream) {
    SB200_REQUIRE(variant >= 0 && variant <= 2);
    return mlp_forward_impl(net, zf, in, save, ld_save, variant, stream);
}

static int mlp_forward_impl(const sb200_mlp* net, const sb200_zfilter* zf, const sb200_rows* in, float* const* save,
                            const int64_t* ld_save, int variant, void* stream) {
    FwdParams p;
    int maxw = 0;
    {
        const int rc = fill_fwd_params(net, zf, in, save, ld_save, p, &maxw);
        if (rc != SB200_OK) return rc;
    }
    if (in->rows == 0) return SB200_OK;
    const size_t budget = SMEM_BUDGET;
    auto fits = [&](int bm, int bk) {
        return (size_t)(2 * bm * (round_up(maxw, bk) + 4) + 2 * bk * PASS_N) * 4 <= budget;
    };
    SB200_REQUIRE(fits(8, 16));
    cudaStream_t st = (cudaStream_t)stream;
    // small batches: skinny kernel (8 rows per CTA, weights streamed once per CTA from L2)
    // default numerics: tensor-core 3xTF32 (fp32-level accuracy, ~1e-6 rel); SB200_MMA=0 selects the pure-FFMA kernels
    // explicit variants for the dual-pipe critic pass (ops.mlp_forward_dual): a tensor-core kernel and an FFMA kernel
    // that fit one SM TOGETHER (<= 128 registers per thread each, 67 KB + 99 KB of shared memory), so that the two
    // halves of a large batch keep the tensor pipe and the FMA pipe busy at the same time
    if (variant == 1) {
        const int rc = launch_fwd_mma<2>(p, maxw, net, st);
        if (rc != SB200_ERR_UNSUPPORTED) return rc;
    }
    if (variant == 2 && fits(32, 16)) return launch_fwd<4, 16>(p, maxw, st);
    // measured (tools/bench_kernels.py, 64-256-256-8): at 1024 rows the FFMA skinny kernel (19 us) beats mma<1> (26 us),
    // whose 64 CTAs leave most SMs idle; from ~4K rows the tensor-core tiles win
    if (g_forward_mode == 1 && p.rows > 2048) {
        // large M: 32-row tiles at 2 CTAs/SM (631 us on the 132 096-row critic pass) beat 64-row tiles at 1 CTA/SM
        // (774 us): the second resident CTA hides the first one's fragment-load and barrier latencies
        int rc = (p.rows <= 4096) ? launch_fwd_mma<1>(p, maxw, net, st) : launch_fwd_mma<2>(p, maxw, net, st);
        if (rc == SB200_ERR_UNSUPPORTED && p.rows > 4096) rc = launch_fwd_mma<4>(p, maxw, net, st);
        if (rc != SB200_ERR_UNSUPPORTED) return rc;
    }
    static const int no_skinny = [] { const char* e = getenv("SB200_NO_SKINNY"); return e ? atoi(e) : 0; }();
    if (p.rows <= 2048 && !no_skinny) {
        p.ldh = round_up(maxw, SK_U * SK_D) + 4;
        int scratch = 2 * net->dims[0];
        for (int l = 0; l < net->n_layers; ++l)
            if (net->dims[l + 1] <= 32) {
                const int kl = (net->dims[l] + (p.aux_layer == l ? p.aux_dim : 0)) * net->ldw[l];
                if (kl > scratch && kl <= 16384) scratch = kl;
            }
        p.scratch_floats = scratch;
        const size_t smem = (size_t)(2 * SK_R * p.ldh + scratch) * sizeof(float);
        if (smem <= 100 * 1024) {
            const long long grid = (p.rows + SK_R - 1) / SK_R;
            mlp_fwd_skinny_kernel<<<(unsigned)grid, SB200_THREADS, smem, st>>>(p);
            return sb200_launch_status();
        }
    }
    // tuning override for experiments (tools/bench_kernels.py): SB200_FWD_TM = 8 | 4 | 2 | 1
    static const int force_tm = [] { const char* e = getenv("SB200_FWD_TM"); return e ? atoi(e) : 0; }();
    if (force_tm == 8 && fits(64, 16)) return launch_fwd<8, 16>(p, maxw, st);
    if (force_tm == 4 && fits(32, 16)) return launch_fwd<4, 16>(p, maxw, st);
    if (force_tm == 2 && fits(16, 64)) return launch_fwd<2, 64>(p, maxw, st);
    if (force_tm == 1 && fits(8, 64)) return launch_fwd<1, 64>(p, maxw, st);
    // largest row tile that still yields >= ~1 CTA per SM; small batches take 16-row tiles with 64-row W stages
    const long long want = 120;
    // 32-row tiles at 2 CTAs/SM (16 warps hide the LDS->FFMA dependency chains) before 64-row tiles at 1 CTA/SM
    // (tools/bench_kernels.py critic times both)
    if (fits(32, 16) && (p.rows + 31) / 32 >= 2 * want) return launch_fwd<4, 16>(p, maxw, st);
    if (fits(64, 16) && (p.rows + 63) / 64 >= want) return launch_fwd<8, 16>(p, maxw, st);
    if (fits(32, 16) && (p.rows + 31) / 32 >= want) return launch_fwd<4, 16>(p, maxw, st);
    if (fits(16, 64)) return launch_fwd<2, 64>(p, maxw, st);
    if (fits(16, 16)) return launch_fwd<2, 16>(p, maxw, st);
    if (fits(8, 64)) return launch_fwd<1, 64>(p, maxw, st);
    return launch_fwd<1, 16>(p, maxw, st);
}
