// Tensor-core variant of the fused MLP forward: warp-level mma.sync m16n8k8 TF32 with the 3xTF32
// error-compensated split (x = hi + lo, hi = tf32(x), lo = tf32(x - hi);  A.B ~= A_lo.B_hi + A_hi.B_lo + A_hi.B_hi,
// fp32 accumulate), which restores fp32-level accuracy (~1e-6 relative) -- plain TF32 (~1e-3) would miss the 1e-5
// parity bar.  Included by mlp_fwd.cu (shares FwdParams / round_up).
//
// Why mma.sync and not wgmma here: these are skinny problems.  One env step of all actors is 1024 rows, a learner
// minibatch 1024-4096 rows; a wgmma tile is 64 rows per warpgroup fed through an mbarrier pipeline, which would leave
// most SMs idle and add microseconds of fixed latency to a kernel whose whole budget is a few microseconds.  m16n8k8 fragments give 16-row tiles, and -- the point of the exercise -- the A fragments are
// DISTRIBUTED over the lanes of a warp, so the activation rows are read from shared memory once per warp instead of
// once per thread (the FFMA version was bound by exactly that LDS return traffic).
//
// Tile: CTA = 8 warps, BM = 16*MT rows; warp w owns output columns [n0 + 32w, n0 + 32w + 32) of a 256-column pass
// (4 n-tiles) for all MT m-tiles.  B fragments (weights, kernel layout W[k][n]) are loaded straight from L2 into a
// register ring (each warp reads a different column slice: no redundancy inside a CTA); activations live in shared
// memory exactly as in the FFMA kernels.
#pragma once

namespace {

constexpr int MMA_D = 3;     // register stages of B fragments in flight (8 k-rows each)

__device__ __forceinline__ void mma_tf32(float (&d)[4], const unsigned (&a)[4], unsigned b0, unsigned b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int MT>
__global__ void __launch_bounds__(SB200_THREADS, (MT <= 2) ? 2 : 1) mlp_fwd_mma_kernel(const __grid_constant__ FwdParams p) {
    constexpr int BM = 16 * MT;
    extern __shared__ __align__(16) float smem[];
    const int ldh = p.ldh;
    float* Hin = smem;
    float* Hout = smem + BM * ldh;
    float* Wsc = smem + 2 * BM * ldh;                   // scratch: z-filter columns, then the narrow head's weights
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;              // mma fragment coordinates
    const long long row0 = (long long)blockIdx.x * BM;
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
        const int in_wp = round_up(in_w, 8);
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
            const int nst = (K + 7) >> 3;                           // k8 steps (Hin is zero-padded to 8)
            const int rot = (int)(((unsigned)blockIdx.x * 5u) % (unsigned)nst);   // de-phase the CTAs' walk over W
            for (int n0 = 0; n0 < N; n0 += 256) {
                float acc[MT][4][4];
#pragma unroll
                for (int mt = 0; mt < MT; ++mt)
#pragma unroll
                    for (int j = 0; j < 4; ++j)
#pragma unroll
                        for (int c = 0; c < 4; ++c) acc[mt][j][c] = 0.0f;
                const int nb = n0 + warp * 32 + g;                  // this lane's column in n-tile 0
                float breg[MMA_D][8];
                auto stage_k0 = [&](int it) { int s_ = rot + it; if (s_ >= nst) s_ -= nst; return s_ * 8; };
                auto load_stage = [&](float (&dst)[8], int it) {
                    const int k0 = stage_k0(it);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int n = nb + j * 8;
                        const bool okn = (it < nst) && (n < N);
                        dst[2 * j] = (okn && k0 + t < K) ? __ldg(W + (long long)(k0 + t) * ldw + n) : 0.0f;
                        dst[2 * j + 1] = (okn && k0 + t + 4 < K) ? __ldg(W + (long long)(k0 + t + 4) * ldw + n) : 0.0f;
                    }
                };
#pragma unroll
                for (int d = 0; d < MMA_D - 1; ++d) load_stage(breg[d], d);
                for (int it0 = 0; it0 < nst; it0 += MMA_D) {
#pragma unroll
                    for (int d = 0; d < MMA_D; ++d) {
                        const int it = it0 + d;
                        load_stage(breg[(d + MMA_D - 1) % MMA_D], it + MMA_D - 1);
                        if (it < nst) {
                            const int k0 = stage_k0(it);
                            unsigned bh[8], bl[8];
#pragma unroll
                            for (int q = 0; q < 8; ++q) split_tf32(breg[d][q], bh[q], bl[q]);
#pragma unroll
                            for (int mt = 0; mt < MT; ++mt) {
                                const float* ar = Hin + (mt * 16 + g) * ldh + k0 + t;
                                unsigned ah[4], al[4];
                                split_tf32(ar[0], ah[0], al[0]);
                                split_tf32(ar[8 * ldh], ah[1], al[1]);
                                split_tf32(ar[4], ah[2], al[2]);
                                split_tf32(ar[8 * ldh + 4], ah[3], al[3]);
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                    mma_tf32(acc[mt][j], al, bh[2 * j], bh[2 * j + 1]);     // small terms first
                                    mma_tf32(acc[mt][j], ah, bl[2 * j], bl[2 * j + 1]);
                                    mma_tf32(acc[mt][j], ah, bh[2 * j], bh[2 * j + 1]);
                                }
                            }
                        }
                    }
                }
                // epilogue: c0,c1 -> (row g, cols 2t, 2t+1); c2,c3 -> (row g+8, same cols)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int n = n0 + warp * 32 + j * 8 + 2 * t;
                    if (n >= N) continue;
                    const float b0v = bias[n];
                    const float b1v = (n + 1 < N) ? bias[n + 1] : 0.0f;
#pragma unroll
                    for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int m = mt * 16 + g + h * 8;
                            const float o0 = apply_act(acc[mt][j][2 * h] + b0v, act);
                            const float o1 = (n + 1 < N) ? apply_act(acc[mt][j][2 * h + 1] + b1v, act) : 0.0f;
                            if (!last) {
                                Hout[m * ldh + n] = o0;
                                Hout[m * ldh + n + 1] = o1;
                            }
                            const long long r = row0 + m;
                            if (sv != nullptr && r < p.rows) {
                                sv[r * lds + n] = o0;
                                if (n + 1 < N) sv[r * lds + n + 1] = o1;
                            }
                        }
                    }
                }
            }
        } else {
            // narrow head (<= 32 outputs): fp32 FFMA dot products, weights staged once in shared memory
            const float* Wn = W;
            __syncthreads();
            if (K * ldw <= p.scratch_floats) {
                for (int f = tid; f < (K * ldw) / 4; f += SB200_THREADS) cp_async16(Wsc + f * 4, W + f * 4, 16);
                cp_async_commit();
                cp_async_wait<0>();
                __syncthreads();
                Wn = Wsc;
            }
            for (int m = warp; m < BM; m += 8) {
                const long long r = row0 + m;
                const float* hrow = Hin + m * ldh;
                for (int n8 = 0; n8 < N; n8 += 8) {
                    float s8[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) s8[j] = 0.0f;
                    const bool second = (n8 + 4 < ldw);
                    for (int k = lane; k < K; k += 32) {
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
                        const float tt = warp_sum(s8[j]);
                        if (lane == j) mine = tt;
                    }
                    const int n = n8 + lane;
                    if (lane < 8 && n < N) {
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
            const int auxd = (p.aux_layer == l + 1) ? p.aux_dim : 0;
            const int wp2 = round_up(N + auxd, 8);
            const int span = wp2 - N;
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
            float* tp = Hin;
            Hin = Hout;
            Hout = tp;
        }
    }
}

template <int MT>
int launch_fwd_mma(FwdParams p, int maxw, const sb200_mlp* net, cudaStream_t st) {
    constexpr int BM = 16 * MT;
    p.ldh = round_up(maxw, 8) + 4;
    int scratch = 2 * net->dims[0];
    for (int l = 0; l < net->n_layers; ++l)
        if (net->dims[l + 1] <= 32) {
            const int kl = (net->dims[l] + (p.aux_layer == l ? p.aux_dim : 0)) * net->ldw[l];
            if (kl > scratch && kl <= 16384) scratch = kl;
        }
    p.scratch_floats = scratch;
    const size_t smem = (size_t)(2 * BM * p.ldh + scratch) * sizeof(float);
    if (smem > 200 * 1024) return SB200_ERR_UNSUPPORTED;
    const long long grid = (p.rows + BM - 1) / BM;
    mlp_fwd_mma_kernel<MT><<<(unsigned)grid, SB200_THREADS, smem, st>>>(p);
    return sb200_launch_status();
}

}  // namespace
