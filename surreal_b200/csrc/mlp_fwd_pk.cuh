// Inference forward for SMALL batches (one env step of all co-located actors: ~1K rows) on pre-packed weights.
//
// At this size the forward is a chain of dependent latencies, not a throughput problem: in the earlier variants
// every CTA pulled ALL the weights (330 KB) through a register ring that keeps only ~24 KB in flight per SM --
// the L2 round trip, not bandwidth or math, sets the time.  This kernel attacks exactly that:
//   * a thread-block CLUSTER of 4 CTAs owns 32 rows; each CTA computes a QUARTER of every layer's output
//     columns, so it needs only a quarter of the weights (~80 KB for 64-256-256), and it fetches that slice
//     with cp.async in one burst at kernel entry -- the whole slice is in flight at once and then RESIDENT in
//     shared memory; 1024 rows occupy 128 SMs and total L2->SM traffic drops 4x;
//   * the CTAs exchange layer outputs through distributed shared memory (st.shared::cluster into all four
//     copies), one cluster barrier per layer;
//   * weights are packed once per parameter version (sb200_mlp_pack_tf32) into mma.m16n8k8 B-fragment order
//     ({b0, b1} per lane: one conflict-free LDS.64 per k-step), activations are stored in A-fragment order and
//     already split for 3xTF32 (one LDS.128 for hi, one for lo, shared by all 8 warps).
// Numerics: the same 3xTF32 error-compensated products as mlp_fwd_mma.cuh (fp32-level accuracy); the main
// (hi*hi) and correction terms accumulate in separate registers to halve the dependent mma chain.
#pragma once
#include <cooperative_groups.h>

namespace {

namespace cg = cooperative_groups;

constexpr int PK_CS = 4;                // CTAs per cluster (column split)
constexpr int PK_MT = 2;                // 16-row m-tiles per cluster
constexpr int PK_ROWS = 16 * PK_MT;     // rows per cluster

struct PkParams {
    FwdParams f;
    const float* P[SB200_MAX_LAYERS];   // packed weights of wide layer l (NULL for the narrow head)
    int offW[SB200_MAX_LAYERS];         // shared-memory offsets (floats): resident weight slice of layer l
    int offA[SB200_MAX_LAYERS];         //   A-fragment planes (hi | lo) holding the INPUT of wide layer l
    int offHp;                          //   plain row-major input of the narrow head [PK_ROWS][ldp]
    int offScratch;                     //   z-filter columns, then the head's weights
    int ldp;
    float* out;
    long long ld_out;
};

__host__ __device__ inline int pk_nst(int K) { return (K + 7) >> 3; }
__host__ __device__ inline int pk_ntl(int N) { return (((N + 7) >> 3) + PK_CS - 1) / PK_CS; }   // n-tiles per CTA

__device__ __forceinline__ void mma_tf32u(float (&d)[4], const uint4& a, unsigned b0, unsigned b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "r"(b0), "r"(b1));
}

// distributed shared memory: a store to a cluster address (mapa_u32)
__device__ __forceinline__ void st_cluster_v4(unsigned addr, const float4& v) {
    asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}

// position of element (row m of PK_ROWS, column k) inside an A-fragment plane of a layer with `nst` k-steps:
// [m/16][k/8][lane = (m%8)*4 + k%4][slot = (m%16 >= 8) + 2*(k%8 >= 4)]
__device__ __forceinline__ int afrag_index(int m, int k, int nst) {
    const int kk = k & 7;
    return ((((m >> 4) * nst + (k >> 3)) * 32 + (m & 7) * 4 + (kk & 3)) << 2) + ((m >> 3) & 1) + ((kk >> 2) << 1);
}

// Pack kernel: P[((c*nst + s)*NTL + j)*32 + lane] = {b0, b1},  b0 = W[8s + t][8(c*NTL + j) + g],
// b1 = W[8s + t + 4][same column]  (g = lane / 4, t = lane % 4), zero outside [K) x [N): CTA c's slice is contiguous.
__global__ void __launch_bounds__(256) mlp_pack_tf32_kernel(const float* __restrict__ W, int K, int N, int ldw,
                                                            float2* __restrict__ P) {
    const int nst = pk_nst(K), NTL = pk_ntl(N);
    const int idx = blockIdx.x * 256 + threadIdx.x;
    if (idx >= PK_CS * nst * NTL * 32) return;
    const int lane = idx & 31;
    int q = idx >> 5;
    const int j = q % NTL;
    q /= NTL;
    const int s = q % nst, c = q / nst;
    const int g = lane >> 2, t = lane & 3;
    const int n = (c * NTL + j) * 8 + g, k0 = s * 8 + t, k1 = k0 + 4;
    const float b0 = (n < N && k0 < K) ? W[(long long)k0 * ldw + n] : 0.0f;
    const float b1 = (n < N && k1 < K) ? W[(long long)k1 * ldw + n] : 0.0f;
    P[idx] = make_float2(b0, b1);
}

__global__ void __cluster_dims__(PK_CS, 1, 1) __launch_bounds__(SB200_THREADS, 1)
    mlp_fwd_pk_kernel(const __grid_constant__ PkParams pp) {
    const FwdParams& p = pp.f;
    cg::cluster_group cluster = cg::this_cluster();
    const unsigned crank = cluster.block_rank();
    extern __shared__ __align__(16) float smem[];
    const unsigned smem_base = smem_u32(smem);
    unsigned peer_base[PK_CS - 1];                      // the three OTHER CTAs' copies of smem[0]
#pragma unroll
    for (int c = 1; c < PK_CS; ++c) peer_base[c - 1] = mapa_u32(smem_base, (crank + (unsigned)c) % PK_CS);
    float* Hp = smem + pp.offHp;
    float* Wsc = smem + pp.offScratch;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const long long row0 = (long long)(blockIdx.x / PK_CS) * PK_ROWS;
    const int K0 = p.dims[0];

    // ---- one burst: this CTA's weight slices of every wide layer + the head's weights -> shared memory.
    // group 0 = first layer (needed first), group 1 = everything else.
    const int zf_floats = (p.zf != nullptr) ? round_up(2 * K0, 4) : 0;
    float* Whead = Wsc + zf_floats;
    bool head_staged = false;
    for (int l = 0; l < p.n_layers; ++l) {
        const int K = p.dims[l] + (p.aux_layer == l ? p.aux_dim : 0);
        const int N = p.dims[l + 1];
        if (N > 32) {
            const int slice = pk_nst(K) * pk_ntl(N) * 64;                 // floats
            const float* src = pp.P[l] + (long long)crank * slice;
            float* dst = smem + pp.offW[l];
            for (int f = tid; f < slice / 4; f += SB200_THREADS) cp_async16(dst + f * 4, src + f * 4, 16);
        } else {
            const int kl = K * p.ldw[l];
            if (zf_floats + kl <= p.scratch_floats) {
                for (int f = tid; f < kl / 4; f += SB200_THREADS) cp_async16(Whead + f * 4, p.W[l] + f * 4, 16);
                head_staged = true;
            }
        }
        if (l == 0) cp_async_commit();
    }
    cp_async_commit();

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
    {   // input rows -> fragment order (every CTA of the cluster stages all PK_ROWS rows: 8 KB, cheaper than an exchange)
        const int in_w = K0 + (p.aux_layer == 0 ? p.aux_dim : 0);
        const int in_wp = round_up(in_w, 8);
        const bool first_narrow = (p.dims[1] <= 32);
        const int nst0 = in_wp >> 3;
        float* Ahi = smem + pp.offA[0];
        float* Alo = Ahi + PK_MT * nst0 * 128;
        for (int idx = tid; idx < PK_ROWS * in_wp; idx += SB200_THREADS) {
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
            if (first_narrow) {
                Hp[m * pp.ldp + k] = v;
            } else {
                unsigned hi, lo;
                split_tf32(v, hi, lo);
                const int a = afrag_index(m, k, nst0);
                Ahi[a] = __uint_as_float(hi);
                Alo[a] = __uint_as_float(lo);
            }
        }
    }
    cp_async_wait<1>();                                // first layer's weights have landed (this thread's copies)
    cluster.sync();                                    // ... everyone's; and every peer CTA is running (DSMEM is live)

    for (int l = 0; l < p.n_layers; ++l) {
        const int K = p.dims[l] + (p.aux_layer == l ? p.aux_dim : 0);
        const int N = p.dims[l + 1];
        const float* __restrict__ bias = p.b[l];
        const int act = p.act[l];
        const bool last = (l == p.n_layers - 1);
        if (N > 32) {
            const int nst = pk_nst(K), NTL = pk_ntl(N);
            const uint4* Ahi = reinterpret_cast<const uint4*>(smem + pp.offA[l]);
            const uint4* Alo = Ahi + PK_MT * nst * 32;
            const float2* Wl = reinterpret_cast<const float2*>(smem + pp.offW[l]);
            const bool next_narrow = !last && (p.dims[l + 2] <= 32);
            const int auxd = (!last && p.aux_layer == l + 1) ? p.aux_dim : 0;
            const int kp_next = round_up(N + auxd, 8);
            const int nst_next = kp_next >> 3;
            float* Ohi = (last || next_narrow) ? smem : smem + pp.offA[l + 1];   // only used when the next layer is wide
            float* Olo = Ohi + PK_MT * nst_next * 128;
            for (int j = warp; j < NTL; j += 8) {                          // warp-uniform; no block barrier inside
                float accM[PK_MT][4], accC[PK_MT][4];
#pragma unroll
                for (int mt = 0; mt < PK_MT; ++mt)
#pragma unroll
                    for (int c = 0; c < 4; ++c) accM[mt][c] = accC[mt][c] = 0.0f;
                const float2* bp = Wl + (long long)j * 32 + lane;
#pragma unroll 4
                for (int s = 0; s < nst; ++s) {
                    const float2 b = bp[(long long)s * NTL * 32];
                    unsigned bh0, bl0, bh1, bl1;
                    split_tf32(b.x, bh0, bl0);
                    split_tf32(b.y, bh1, bl1);
#pragma unroll
                    for (int mt = 0; mt < PK_MT; ++mt) {
                        const uint4 ah = Ahi[(mt * nst + s) * 32 + lane];
                        const uint4 al = Alo[(mt * nst + s) * 32 + lane];
                        mma_tf32u(accC[mt], al, bh0, bh1);
                        mma_tf32u(accC[mt], ah, bl0, bl1);
                        mma_tf32u(accM[mt], ah, bh0, bh1);
                    }
                }
                // epilogue: c0,c1 -> (row g, cols 2t, 2t+1); c2,c3 -> (row g+8, same cols).  The warp owns ALL 8 columns
                // of next-layer k-step `nt` for all rows: it writes them into its own CTA's copy with scalar stores, then
                // pushes the finished 512-byte chunks to the three peers with 16-byte DSMEM stores (scalar remote stores
                // cost ~1 SM-to-SM transaction each and dominated the first version of this kernel).
                const int nt = (int)crank * NTL + j;
                const bool keep = !last && (nt * 8 < kp_next);
#pragma unroll
                for (int mt = 0; mt < PK_MT; ++mt) {
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const int m = mt * 16 + g + 8 * (c >> 1);
                        const int n = nt * 8 + 2 * t + (c & 1);
                        const long long r = row0 + m;
                        float v = 0.0f;
                        if (n < N) v = apply_act(accM[mt][c] + accC[mt][c] + bias[n], act);
                        else if (n < N + auxd && r < p.rows) v = p.aux[r * p.aux_ld + (n - N)];
                        if (last) {
                            if (n < N && r < p.rows) pp.out[r * pp.ld_out + n] = v;
                        } else if (keep) {
                            if (next_narrow) {
                                Hp[m * pp.ldp + n] = v;
                            } else {
                                unsigned hi, lo;
                                split_tf32(v, hi, lo);
                                const int a = afrag_index(m, n, nst_next);
                                Ohi[a] = __uint_as_float(hi);
                                Olo[a] = __uint_as_float(lo);
                            }
                        }
                    }
                }
                if (keep) {
                    __syncwarp();
                    if (next_narrow) {                                     // 32 rows x 8 columns: lane = row, 2 x float4
                        const float* q = Hp + lane * pp.ldp + nt * 8;
                        const float4 v0 = *reinterpret_cast<const float4*>(q);
                        const float4 v1 = *reinterpret_cast<const float4*>(q + 4);
                        const unsigned off = smem_u32(q) - smem_base;
#pragma unroll
                        for (int cc = 1; cc < PK_CS; ++cc) {
                            const unsigned pb = peer_base[cc - 1] + off;
                            st_cluster_v4(pb, v0);
                            st_cluster_v4(pb + 16, v1);
                        }
                    } else {                                               // (hi, lo) x m-tile: 128 floats each
#pragma unroll
                        for (int mt = 0; mt < PK_MT; ++mt) {
                            const int a = ((mt * nst_next + nt) * 32 + lane) * 4;
                            const float4 vh = *reinterpret_cast<const float4*>(Ohi + a);
                            const float4 vl = *reinterpret_cast<const float4*>(Olo + a);
                            const unsigned oh = smem_u32(Ohi + a) - smem_base, ol = smem_u32(Olo + a) - smem_base;
#pragma unroll
                            for (int cc = 1; cc < PK_CS; ++cc) {
                                const unsigned pb = peer_base[cc - 1];
                                st_cluster_v4(pb + oh, vh);
                                st_cluster_v4(pb + ol, vl);
                            }
                        }
                    }
                }
            }
            if (!last) {
                // columns past the cluster's last n-tile (aux concatenation wider than the tile padding): local copy
                const int covered = PK_CS * NTL * 8;
                const int span = kp_next - covered;
                for (int idx = tid; idx < PK_ROWS * span; idx += SB200_THREADS) {
                    const int m = idx / span, k = covered + (idx - m * span);
                    const long long r = row0 + m;
                    float v = 0.0f;
                    if (k < N + auxd && r < p.rows) v = p.aux[r * p.aux_ld + (k - N)];
                    if (next_narrow) {
                        Hp[m * pp.ldp + k] = v;
                    } else {
                        unsigned hi, lo;
                        split_tf32(v, hi, lo);
                        const int a = afrag_index(m, k, nst_next);
                        Ohi[a] = __uint_as_float(hi);
                        Olo[a] = __uint_as_float(lo);
                    }
                }
                cp_async_wait<0>();                    // the remaining weight slices (issued at entry) have landed
                cluster.sync();
            }
        } else {
            // narrow head (<= 32 outputs): fp32 dot products on the plain activation copy; CTA c owns rows 8c..8c+7
            cp_async_wait<0>();
            __syncthreads();
            const float* Wn = head_staged ? Whead : p.W[l];
            const int ldw = p.ldw[l];
            const int m = (int)crank * 8 + warp;
            const long long r = row0 + m;
            const float* hrow = Hp + m * pp.ldp;
            for (int n8 = 0; n8 < N; n8 += 8) {
                float s8[8];
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) s8[jj] = 0.0f;
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
                for (int jj = 0; jj < 8; ++jj) {
                    const float tt = warp_sum(s8[jj]);
                    if (lane == jj) mine = tt;
                }
                const int n = n8 + lane;
                if (lane < 8 && n < N && r < p.rows) pp.out[r * pp.ld_out + n] = apply_act(mine + bias[n], act);
            }
        }
    }
    cluster.sync();                                    // no CTA may exit while a peer can still write into it
}

}  // namespace
