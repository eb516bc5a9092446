// Tensor-core fused MLP forward for LARGE row counts (the critic pass of _gae_and_return, ppo.py:376-387:
// B*(n+1) = 132 096 rows through 64 -> 256 -> 256 -> 1) on Hopper: wgmma (tf32, fp32 accumulators in registers), weights
// streamed by the TMA engine (cp.async.bulk + mbarrier ring), fp32-level accuracy through the 3xTF32 split
// (x = hi + lo;  a.b ~= a_lo.b_hi + a_hi.b_lo + a_hi.b_hi, fp32 accumulate).
//
// One persistent CTA per SM walks 128-row tiles; each of its two consumer warpgroups owns 64 rows of the tile, and the two
// share every weight stage.  A stage is one K-chunk of 32 of one column half (128 columns) of a layer's weights, hi and lo
// planes (2 x 16 KB), copied from a per-call "image" of the weights (already in the SWIZZLE_128B K-major operand layout,
// built by tc5_prep_kernel from the flat parameter buffer).  Per tile:
//
//   layer 1:  A = z-filtered observation columns, loaded from global memory straight into the wgmma A-fragment
//             registers and split there                                     -> acc1 (128 registers: 64 rows x 256 columns)
//   layer 2:  A = relu(acc1 + b1), taken from the accumulator registers as they are: the accumulator holds columns
//             8i + 2t, 8i + 2t + 1 where the A fragment wants k = t, t + 4, so the layer-2 weight image stores each group
//             of 8 k in the order (0 2 4 6 1 3 5 7) and the two agree      -> acc2 (64 registers, one column half at a time)
//   head   :  relu(acc2 + b2) . W3 + b3 on the CUDA cores after each column half, quad-reduced by shuffles (n_out <= 8)
//
// 8 warps = two consumer warpgroups; thread 0 also issues the bulk copies that refill the ring.
//
// Algorithmic HBM bytes per row: 4*D read + 4*n_out written; weights (640 KB of images per call) stay in L2.
#include "common.cuh"
#include "wgmma.cuh"

namespace {

using namespace wg;

constexpr int TM = 128;                    // rows per tile: 64 per consumer warpgroup
constexpr int KC = 32;                     // k per chunk = one 128-byte swizzle row
constexpr int MAXN = 256;                  // widest hidden layer
constexpr int HN = 128;                    // columns per wgmma (one half of the widest layer)
constexpr int MAX_OUT = 8;
constexpr int B_PLANE = MAXN * 128;        // 32 KB: one plane of one chunk of the image
constexpr int HALF_PLANE = HN * 128;       // 16 KB: one column half of it
constexpr int STAGE_BYTES = 2 * HALF_PLANE;            // hi | lo
constexpr int NSTAGE = 6;
constexpr int NTHREADS = 256;
constexpr int MAX_K0 = 256;

struct Tc5Params {
    const float* x;
    const float* x_next;
    long long ldx;
    long long rows;
    int win_n;
    const float* zf;            // running_sum[K0] | running_sumsq[K0] | count, or null
    float zf_eps;
    int K0, N1, N2, n_out;
    int act_out;
    const float* b1;
    const float* b2;
    const float* W3;            // [N2][ldw3]
    int ldw3;
    const float* b3;
    const unsigned char* wimg;  // chunk images: [NC][hi plane B_PLANE | lo plane B_PLANE]
    float* out;
    long long ld_out;
    long long n_tiles;
};

struct SmemSmall {
    uint64_t full[NSTAGE], empty[NSTAGE];
    alignas(16) float zmean[MAX_K0];
    alignas(16) float zstd[MAX_K0];
    alignas(16) float b1[MAXN];             // zero past N1
    alignas(16) float b2[MAXN];             // zero past N2
    alignas(16) float w3[MAXN * MAX_OUT];   // w3[col][8], zero-padded
    float b3[MAX_OUT];
};

// ---- weight images ------------------------------------------------------------------------------------------------------
// W is the kernel layout [K][ldw] (k-major rows, n contiguous).  Chunk c of a layer covers k in [32c, 32c+32); its image is
// the operand tile B[n][kk] = W[32c + kk'][n] in the SWIZZLE_128B K-major layout, as a hi plane and a lo plane, rows past N
// zero.  Layer 1: kk' = kk.  Layer 2: within each group of 8, kk' = (0 2 4 6 1 3 5 7)[kk % 8] (see the header comment).
__global__ void __launch_bounds__(256) tc5_prep_kernel(const float* __restrict__ W1, int ldw1, int K0, int N1,
                                                       const float* __restrict__ W2, int ldw2, int N2,
                                                       unsigned char* __restrict__ img) {
    const int NC1 = K0 / KC, NC2 = N1 / KC;
    const long long units = (long long)(NC1 + NC2) * MAXN * 8;          // one unit = 16 bytes of one row of one chunk
    for (long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x; u < units; u += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(u % MAXN);
        const int c16 = (int)((u / MAXN) % 8);
        const int c = (int)(u / (MAXN * 8));
        const bool l1 = c < NC1;
        const float* W = l1 ? W1 : W2;
        const int ldw = l1 ? ldw1 : ldw2;
        const int N = l1 ? N1 : N2;
        const int kb = (l1 ? c : c - NC1) * KC;
        int k[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) k[j] = l1 ? kb + c16 * 4 + j : kb + (c16 >> 1) * 8 + 2 * j + (c16 & 1);
        uint32_t hi[4] = {0u, 0u, 0u, 0u}, lo[4] = {0u, 0u, 0u, 0u};
        if (n < N) {
#pragma unroll
            for (int j = 0; j < 4; ++j) split_tf32(W[(long long)k[j] * ldw + n], hi[j], lo[j]);
        }
        unsigned char* base = img + (size_t)c * 2 * B_PLANE;
        const uint32_t off = sw128_off((uint32_t)n, (uint32_t)(c16 * 4));
        *reinterpret_cast<uint4*>(base + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
        *reinterpret_cast<uint4*>(base + B_PLANE + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    }
}

__device__ __forceinline__ const float* row_ptr(const Tc5Params& p, long long r) {
    if (p.win_n > 0) {
        const long long b = r / (p.win_n + 1);
        const int kk = (int)(r - b * (p.win_n + 1));
        return (kk < p.win_n) ? p.x + (b * p.win_n + kk) * p.ldx : p.x_next + b * p.ldx;
    }
    return p.x + r * p.ldx;
}

// the three products of one k-slice, small terms first; `first` starts the accumulator
__device__ __forceinline__ void mma3(float (&d)[64], const uint32_t (&ah)[4], const uint32_t (&al)[4], uint64_t bh, uint64_t bl,
                                     bool first) {
    wgmma_m64n128k8_tf32_rs(d, al[0], al[1], al[2], al[3], bh, first ? 0u : 1u);
    wgmma_m64n128k8_tf32_rs(d, ah[0], ah[1], ah[2], ah[3], bl, 1u);
    wgmma_m64n128k8_tf32_rs(d, ah[0], ah[1], ah[2], ah[3], bh, 1u);
}

// MO: output columns the head keeps per row (1 for the critic, MAX_OUT otherwise)
template <int MO>
__global__ void __launch_bounds__(NTHREADS, 1) mlp3_wgmma_kernel(const __grid_constant__ Tc5Params p) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* stage_base = smem_raw;
    if ((smem_u32(smem_raw) & 1023u) != 0u) __trap();      // the dynamic segment must start 1024-aligned (no static smem here)
    SmemSmall* sm = reinterpret_cast<SmemSmall*>(stage_base + NSTAGE * STAGE_BYTES);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int NC1 = p.K0 / KC, NC2 = p.N1 / KC;
    const int nh1 = (p.N1 + HN - 1) / HN, nh2 = (p.N2 + HN - 1) / HN;

    // ---- one-time setup ---------------------------------------------------------------------------------------------
    if (tid == 0) {
        for (int s = 0; s < NSTAGE; ++s) {
            mbar_init(&sm->full[s], 1);            // thread 0's arrive.expect_tx (both planes' bytes)
            mbar_init(&sm->empty[s], 8);           // every consumer warp, after its wgmmas on the stage completed
        }
        mbar_init_fence();
    }
    for (int i = tid; i < MAXN; i += NTHREADS) {
        sm->b1[i] = (i < p.N1) ? p.b1[i] : 0.0f;
        sm->b2[i] = (i < p.N2) ? p.b2[i] : 0.0f;
    }
    for (int i = tid; i < MAXN * MAX_OUT; i += NTHREADS) {
        const int k = i / MAX_OUT, o = i - k * MAX_OUT;
        sm->w3[i] = (k < p.N2 && o < p.n_out) ? p.W3[(long long)k * p.ldw3 + o] : 0.0f;
    }
    if (tid < MAX_OUT) sm->b3[tid] = (tid < p.n_out) ? p.b3[tid] : 0.0f;
    if (p.zf != nullptr) {
        const float cnt = p.zf[2 * p.K0];
        for (int k = tid; k < p.K0; k += NTHREADS) {
            const float mean = p.zf[k] / cnt;
            const float var = p.zf[p.K0 + k] / cnt - mean * mean;
            sm->zmean[k] = mean;
            sm->zstd[k] = 1.0f / fmaxf(sqrtf(var), p.zf_eps);       // reciprocal: the filter multiplies (1 ulp vs the division)
        }
    }
    __syncthreads();
    const long long my_tiles = (p.n_tiles > (long long)blockIdx.x) ? (p.n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    // ================= consumer warpgroups =================
    const int wgi = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3;
    float acc1[2][64];
    float acc2[64];
    // stage q of this CTA: tile q / QT; within a tile, layer 1 runs chunk-major (c, h) and layer 2 half-major (h, c)
    const int QT = NC1 * nh1 + nh2 * NC2;
    const long long n_stages = my_tiles * QT;
    // thread 0 also feeds the ring: stage q + NSTAGE goes into the slot stage q leaves, once all 8 consumer warps left it
    auto load = [&](long long qq) {
        const int r = (int)(qq % QT);
        const int chunk = (r < NC1 * nh1) ? r / nh1 : NC1 + (r - NC1 * nh1) % NC2;
        const int h = (r < NC1 * nh1) ? r % nh1 : (r - NC1 * nh1) / NC2;
        const int s = (int)(qq % NSTAGE);
        unsigned char* st = stage_base + (size_t)s * STAGE_BYTES;
        const unsigned char* src = p.wimg + (size_t)chunk * 2 * B_PLANE + (size_t)h * HALF_PLANE;
        mbar_arrive_expect_tx(&sm->full[s], 2 * HALF_PLANE);
        bulk_g2s(st, src, HALF_PLANE, &sm->full[s]);
        bulk_g2s(st + HALF_PLANE, src + B_PLANE, HALF_PLANE, &sm->full[s]);
    };
    if (tid == 0)
        for (long long qq = 0; qq < NSTAGE && qq < n_stages; ++qq) load(qq);
    long long q = 0;
    // waits for the next stage; returns the descriptors of its hi / lo planes at k-slice 0
    auto acquire = [&](uint64_t& dh, uint64_t& dl) {
        const int s = (int)(q % NSTAGE);
        mbar_wait(&sm->full[s], (uint32_t)(q / NSTAGE) & 1u);
        const uint32_t a = smem_u32(stage_base + (size_t)s * STAGE_BYTES);
        dh = smem_desc_sw128(a);
        dl = smem_desc_sw128(a + HALF_PLANE);
    };
    auto release = [&]() {
        __syncwarp();
        const int s = (int)(q % NSTAGE);
        if (lane == 0) mbar_arrive(&sm->empty[s]);
        if (tid == 0 && q + NSTAGE < n_stages) {
            mbar_wait(&sm->empty[s], (uint32_t)(q / NSTAGE) & 1u);
            load(q + NSTAGE);
        }
        ++q;
    };

    for (long long it = 0; it < my_tiles; ++it) {
        const long long tile = (long long)blockIdx.x + it * gridDim.x;
        const long long ra = tile * TM + wgi * 64 + w * 16 + g, rb = ra + 8;
        const float* xa = (ra < p.rows) ? row_ptr(p, ra) : nullptr;
        const float* xb = (rb < p.rows) ? row_ptr(p, rb) : nullptr;

        // ---- layer 1 ------------------------------------------------------------------------------------------------
#pragma unroll 1
        for (int c = 0; c < NC1; ++c) {
            uint32_t ah[4][4], al[4][4];
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const int k0 = c * KC + ks * 8 + t;
                float v[4] = {xa ? __ldg(xa + k0) : 0.0f, xb ? __ldg(xb + k0) : 0.0f,
                              xa ? __ldg(xa + k0 + 4) : 0.0f, xb ? __ldg(xb + k0 + 4) : 0.0f};
                if (p.zf != nullptr) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int k = k0 + (j >> 1) * 4;
                        v[j] = fminf(fmaxf((v[j] - sm->zmean[k]) * sm->zstd[k], -5.0f), 5.0f);
                    }
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) split_tf32(v[j], ah[ks][j], al[ks][j]);
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (h < nh1) {
                    uint64_t dh, dl;
                    acquire(dh, dl);
                    wgmma_fence();
#pragma unroll
                    for (int ks = 0; ks < 4; ++ks)
                        mma3(acc1[h], ah[ks], al[ks], dh + 2 * ks, dl + 2 * ks, c == 0 && ks == 0);   // +32 bytes per k-slice
                    wgmma_commit();
                    wgmma_wait_all();
                    fence_regs(acc1[h]);
                    release();
                }
            }
        }
        // hidden activations in place: acc1[h][4i + e] holds column 128h + 8i + 2t + (e & 1)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const float2 bb = *reinterpret_cast<const float2*>(sm->b1 + h * HN + 8 * i + 2 * t);
                acc1[h][4 * i + 0] = fmaxf(acc1[h][4 * i + 0] + bb.x, 0.0f);
                acc1[h][4 * i + 1] = fmaxf(acc1[h][4 * i + 1] + bb.y, 0.0f);
                acc1[h][4 * i + 2] = fmaxf(acc1[h][4 * i + 2] + bb.x, 0.0f);
                acc1[h][4 * i + 3] = fmaxf(acc1[h][4 * i + 3] + bb.y, 0.0f);
            }

        // ---- layer 2 + head -----------------------------------------------------------------------------------------
        float o[2][MO];
#pragma unroll
        for (int k = 0; k < MO; ++k) o[0][k] = o[1][k] = 0.0f;
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
            if (h2 >= nh2) break;
#pragma unroll
            for (int c = 0; c < MAXN / KC; ++c) {
                if (c < NC2) {
                    uint64_t dh, dl;
                    acquire(dh, dl);
                    wgmma_fence();
#pragma unroll
                    for (int ks = 0; ks < 4; ++ks) {
                        const int sl = c * 4 + ks, hs = sl >> 4, i = sl & 15;       // source k-slice = 8 columns of acc1
                        uint32_t ah[4], al[4];
                        split_tf32(acc1[hs][4 * i + 0], ah[0], al[0]);
                        split_tf32(acc1[hs][4 * i + 2], ah[1], al[1]);
                        split_tf32(acc1[hs][4 * i + 1], ah[2], al[2]);
                        split_tf32(acc1[hs][4 * i + 3], ah[3], al[3]);
                        mma3(acc2, ah, al, dh + 2 * ks, dl + 2 * ks, c == 0 && ks == 0);
                    }
                    wgmma_commit();
                    wgmma_wait_all();
                    fence_regs(acc2);
                    release();
                }
            }
#pragma unroll
            for (int i = 0; i < 16; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = h2 * HN + 8 * i + 2 * t + e;
                    const float bb = sm->b2[col];
                    const float ya = fmaxf(acc2[4 * i + e] + bb, 0.0f), yb = fmaxf(acc2[4 * i + 2 + e] + bb, 0.0f);
#pragma unroll
                    for (int k = 0; k < MO; ++k) {
                        const float wk = sm->w3[col * MAX_OUT + k];
                        o[0][k] = fmaf(ya, wk, o[0][k]);
                        o[1][k] = fmaf(yb, wk, o[1][k]);
                    }
                }
        }
        // the 4 lanes of a quad hold disjoint columns of the same two rows
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int k = 0; k < MO; ++k) {
                o[r][k] += __shfl_xor_sync(0xffffffffu, o[r][k], 1);
                o[r][k] += __shfl_xor_sync(0xffffffffu, o[r][k], 2);
            }
        if (t == 0) {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const long long gr = r ? rb : ra;
                if (gr < p.rows) {
#pragma unroll
                    for (int k = 0; k < MO; ++k)
                        if (k < p.n_out) {
                            float y = o[r][k] + sm->b3[k];
                            if (p.act_out == SB200_ACT_RELU) y = fmaxf(y, 0.0f);
                            else if (p.act_out == SB200_ACT_TANH) y = tanhf(y);
                            p.out[gr * p.ld_out + k] = y;
                        }
                }
            }
        }
    }
}

constexpr size_t TC5_SMEM = (size_t)NSTAGE * STAGE_BYTES + sizeof(SmemSmall);

}  // namespace

int sb200_mlp_tc5_init() {
    SB200_CUDA(cudaFuncSetAttribute(mlp3_wgmma_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC5_SMEM));
    SB200_CUDA(cudaFuncSetAttribute(mlp3_wgmma_kernel<MAX_OUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC5_SMEM));
    return SB200_OK;
}

static bool tc5_net_ok(const sb200_mlp* net) {
    if (net == nullptr || net->n_layers != 3 || net->aux_layer >= 0 || sb200_mlp_has_ln(net)) return false;
    const int K0 = net->dims[0], N1 = net->dims[1], N2 = net->dims[2], NO = net->dims[3];
    if (K0 % KC != 0 || K0 < KC || K0 > MAX_K0) return false;
    if (N1 % KC != 0 || N1 < KC || N1 > MAXN) return false;
    if (N2 % KC != 0 || N2 < KC || N2 > MAXN) return false;
    if (NO < 1 || NO > MAX_OUT) return false;
    if (net->act[0] != SB200_ACT_RELU || net->act[1] != SB200_ACT_RELU) return false;
    return true;
}

extern "C" int sb200_mlp_tc5_supported(const sb200_mlp* net, int64_t rows) {
    return (tc5_net_ok(net) && rows >= TM) ? 1 : 0;
}

extern "C" size_t sb200_mlp_tc5_workspace_bytes(const sb200_mlp* net) {
    if (!tc5_net_ok(net)) return 0;
    return (size_t)(net->dims[0] / KC + net->dims[1] / KC) * 2 * B_PLANE;
}

extern "C" int sb200_mlp_forward_tc5_f32(const sb200_mlp* net, const sb200_zfilter* zf, const sb200_rows* in, float* out,
                                         int64_t ld_out, void* workspace, int max_grid, void* stream) {
    SB200_REQUIRE(net && in && out && workspace);
    if (!tc5_net_ok(net)) return SB200_ERR_UNSUPPORTED;
    SB200_REQUIRE(in->x != nullptr && in->rows >= 0 && in->aux == nullptr && in->save_x == nullptr);
    SB200_REQUIRE(in->win_n == 0 || in->x_next != nullptr);
    SB200_REQUIRE((((uintptr_t)workspace) & 15) == 0 && ld_out >= net->dims[3]);
    if (in->rows == 0) return SB200_OK;
    cudaStream_t st = (cudaStream_t)stream;
    static int n_sm = 0;
    if (n_sm == 0) {
        int dev = 0;
        SB200_CUDA(cudaGetDevice(&dev));
        SB200_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    }
    Tc5Params p;
    p.x = in->x; p.x_next = in->x_next; p.ldx = in->ldx; p.rows = in->rows; p.win_n = in->win_n;
    p.zf = (zf != nullptr) ? zf->stats : nullptr;
    p.zf_eps = (zf != nullptr) ? zf->eps : 0.0f;
    p.K0 = net->dims[0]; p.N1 = net->dims[1]; p.N2 = net->dims[2]; p.n_out = net->dims[3];
    p.act_out = net->act[2];
    p.b1 = net->b[0]; p.b2 = net->b[1]; p.W3 = net->W[2]; p.ldw3 = net->ldw[2]; p.b3 = net->b[2];
    p.wimg = (const unsigned char*)workspace;
    p.out = out; p.ld_out = ld_out;
    p.n_tiles = (in->rows + TM - 1) / TM;
    const int units = (p.K0 / KC + p.N1 / KC) * MAXN * 8;
    tc5_prep_kernel<<<(units + 255) / 256, 256, 0, st>>>(net->W[0], net->ldw[0], p.K0, p.N1, net->W[1], net->ldw[1], p.N2,
                                                        (unsigned char*)workspace);
    const int cap = (max_grid >= 1 && max_grid < n_sm) ? max_grid : n_sm;
    const long long grid = p.n_tiles < cap ? p.n_tiles : cap;
    if (p.n_out == 1) mlp3_wgmma_kernel<1><<<(unsigned)grid, NTHREADS, TC5_SMEM, st>>>(p);
    else mlp3_wgmma_kernel<MAX_OUT><<<(unsigned)grid, NTHREADS, TC5_SMEM, st>>>(p);
    return sb200_launch_status(2);
}
