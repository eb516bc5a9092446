// Backward of the LayerNorm that follows a hidden layer's activation (ActorNetworkX / CriticNetworkX with use_layernorm,
// builders.py:42-48,64-77; torch.nn.LayerNorm's autograd in ddpg.py:306,330).
//
// One launch, two kinds of CTA that read the same inputs and write disjoint outputs:
//   - row CTAs (a warp per row): dX = rstd * (g*dY - mean(g*dY) - x^ * mean(g*dY*x^)) [* relu'(h)], x^ = (h - mean) * rstd
//     recomputed from the forward's saved (mean, rstd), so it has the forward's bits;
//   - column CTAs (one per 64-column block and split): dg = sum dY*x^, db = sum dY over the split's rows, 4 row groups
//     added in fixed order -> the split's slab.  No atomics: bit-reproducible run to run.
// Why a kernel of its own and not an epilogue of the dX GEMM: the row reductions need whole rows, while a 64x64 dX tile
// holds a quarter of a 300-wide row; fusing would need a second pass over the GEMM output anyway.  The extra traffic is
// three [M][N] reads and one write (about 26 MB at M = 4096, N = 400), small next to the GEMMs around it.
#include "common.cuh"
#include "gemm_tiles.cuh"

namespace {

constexpr int LN_COLS = 64;                    // columns per column CTA
constexpr int LN_RG = SB200_THREADS / LN_COLS;  // row groups per column CTA

__global__ void __launch_bounds__(SB200_THREADS) layernorm_bwd_kernel(
    const float* __restrict__ dY, long long ldy, const float* __restrict__ h, long long ldh,
    const float* __restrict__ stats, const float* __restrict__ g, int M, int N, int relu, float* __restrict__ dX,
    long long lddx, float* __restrict__ dg_slabs, float* __restrict__ db_slabs, long long slab_stride, int rps,
    int row_ctas) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if ((int)blockIdx.x < row_ctas) {
        const int m = blockIdx.x * (SB200_THREADS / 32) + warp;
        if (m >= M) return;
        const float mean = stats[2LL * m], rstd = stats[2LL * m + 1];
        const float* dy = dY + (long long)m * ldy;
        const float* hr = h + (long long)m * ldh;
        float s1 = 0.0f, s2 = 0.0f;
        for (int j = lane; j < N; j += 32) {
            const float gd = dy[j] * __ldg(g + j);
            s1 += gd;
            s2 = fmaf(gd, (hr[j] - mean) * rstd, s2);
        }
        const float m1 = warp_sum(s1) / (float)N, m2 = warp_sum(s2) / (float)N;
        float* dx = dX + (long long)m * lddx;
        for (int j = lane; j < N; j += 32) {
            const float hv = hr[j];
            const float xh = (hv - mean) * rstd;
            float v = rstd * (dy[j] * __ldg(g + j) - m1 - xh * m2);
            if (relu && !(hv > 0.0f)) v = 0.0f;
            dx[j] = v;
        }
        return;
    }
    // column CTA: block (cb, z) of the dg / db slabs
    __shared__ float red[2][LN_RG][LN_COLS];
    const int c = blockIdx.x - row_ctas;
    const int ncb = (N + LN_COLS - 1) / LN_COLS;
    const int z = c / ncb, cb = c - z * ncb;
    const int col = cb * LN_COLS + (tid % LN_COLS), rg = tid / LN_COLS;
    const int mb = z * rps, me = min(M, mb + rps);
    float sg = 0.0f, sb = 0.0f;
    if (col < N) {
        for (int m = mb + rg; m < me; m += LN_RG) {
            const float d = dY[(long long)m * ldy + col];
            const float xh = (h[(long long)m * ldh + col] - stats[2LL * m]) * stats[2LL * m + 1];
            sg = fmaf(d, xh, sg);
            sb += d;
        }
    }
    red[0][rg][tid % LN_COLS] = sg;
    red[1][rg][tid % LN_COLS] = sb;
    __syncthreads();
    if (rg == 0 && col < N) {
        for (int r = 1; r < LN_RG; ++r) {
            sg += red[0][r][tid];
            sb += red[1][r][tid];
        }
        dg_slabs[(long long)z * slab_stride + col] = sg;
        db_slabs[(long long)z * slab_stride + col] = sb;
    }
}

}  // namespace

extern "C" int sb200_layernorm_bwd_f32(const float* dY, int64_t ldy, const float* h, int64_t ldh, const float* stats,
                                       const float* g, int M, int N, int relu, float* dX, int64_t lddx, float* dg_slabs,
                                       float* db_slabs, int64_t slab_stride, int splits, void* stream) {
    SB200_REQUIRE(dY && h && stats && g && dX && M >= 1 && N >= 1);
    SB200_REQUIRE(ldy >= N && ldh >= N && lddx >= N);
    SB200_REQUIRE((dg_slabs == nullptr) == (db_slabs == nullptr));
    SB200_REQUIRE(dg_slabs == nullptr || (splits >= 1 && slab_stride >= N));
    const int row_ctas = (M + SB200_THREADS / 32 - 1) / (SB200_THREADS / 32);
    // the rows of split z, as sb200_linear_bwd_dw_f32 splits them
    const int rps = dg_slabs != nullptr ? ((M + splits - 1) / splits + gt::RK - 1) / gt::RK * gt::RK : 0;
    const int col_ctas = dg_slabs != nullptr ? splits * ((N + LN_COLS - 1) / LN_COLS) : 0;
    layernorm_bwd_kernel<<<(unsigned)(row_ctas + col_ctas), SB200_THREADS, 0, (cudaStream_t)stream>>>(
        dY, (long long)ldy, h, (long long)ldh, stats, g, M, N, relu, dX, (long long)lddx, dg_slabs, db_slabs,
        (long long)slab_stride, rps, row_ctas);
    return sb200_launch_status();
}
