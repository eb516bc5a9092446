// Windowed GAE + n-step return (surreal/learner/ppo.py:372-374, 387-418; SURVEY Appendix A.1).
//
// One warp per window: lanes stride over the n steps with coalesced loads of the window's
// rewards / values / dones rows, products are formed exactly as the reference does
// ((td * gamma^k) * lam^k with fp32 tables), the window sums are accumulated in fp64 and reduced with
// warp shuffles.  The horizon-truncated (RNN-mode) variant stages td / r through shared memory.
// Batch normalisation of the advantages (unbiased std, floor 1e-4) is fused through a last-block
// ticket: the last CTA to finish reduces all B*E advantages in a fixed order (deterministic).
//
// Algorithmic HBM bytes per window: (3n+1)*4 read + 2*E*4 written (SURVEY §8d: 1548 B at n=128).
#include "common.cuh"

namespace {

constexpr int GAE_WARPS = 8;
constexpr int GAE_MAX_GRID = 1056;          // persistent grid: 132 SMs x 8 resident CTAs
constexpr int GAE_FUSED_NORM_MAX = 16384;   // up to here the last CTA normalises alone (one launch); above: a parallel pass

struct GaeWs {
    unsigned int counter;
    unsigned int pad;
    float mean, denom;                      // batch statistics of the large-batch path (read by gae_normalize_kernel)
    double partial[2 * GAE_MAX_GRID];       // per-CTA (sum, sum of squares) of the advantages
};

__device__ __forceinline__ float pow_table(float base_f32, int k) {
    // torch.pow(python_float, fp32 tensor): base rounded to fp32, result within 1 ulp (ppo.py:373-374)
    return (float)pow((double)base_f32, (double)k);
}

__device__ void normalize_all(float* adv, long long total, double* sh) {
    // mean and UNBIASED std over all advantages (torch .mean() / .std(), ppo.py:413-416), two-pass fp64
    double s = 0.0;
    for (long long i = threadIdx.x; i < total; i += blockDim.x) s += (double)adv[i];
    const double mean = block_sum(s, sh) / (double)total;
    double q = 0.0;
    for (long long i = threadIdx.x; i < total; i += blockDim.x) {
        const double d = (double)adv[i] - mean;
        q += d * d;
    }
    const double var = block_sum(q, sh) / (double)(total - 1);
    const float mean_f = (float)mean;
    const float std_f = (float)sqrt(var);
    const float denom = (std_f > 1e-4f) ? std_f : 1e-4f;   // Python max(std, 1e-4)
    for (long long i = threadIdx.x; i < total; i += blockDim.x) adv[i] = (adv[i] - mean_f) / denom;
}

// One window with n == 32 * ITER, everything in registers: ALL loads of the window are issued before the first use (the
// generic loop below exposes one DRAM round trip per 32 steps: 1.76 TB/s at 2^18 windows), the NEXT window of the warp is
// loaded while the current one is reduced (two windows in flight per warp), and the shifted operands
// V[k+1] / done[k-1] come from the neighbouring lane by shuffle instead of a second load.  Same operations on the same
// operands in the same order as the generic loop -> bit-identical results.
template <int ITER>
struct GaeRegs {
    float rr[ITER], vv[ITER], dd[ITER], v_last;
};
template <int ITER>
__device__ __forceinline__ void gae_window_load(const float* __restrict__ r, const float* __restrict__ v, const float* __restrict__ d,
                                                int lane, GaeRegs<ITER>& g) {
    constexpr int n = 32 * ITER;
#pragma unroll
    for (int i = 0; i < ITER; ++i) {
        g.rr[i] = __ldg(r + lane + 32 * i);
        g.dd[i] = __ldg(d + lane + 32 * i);
        g.vv[i] = __ldg(v + lane + 32 * i);
    }
    g.v_last = (lane == 31) ? __ldg(v + n) : 0.0f;
}
template <int ITER>
__device__ __forceinline__ void gae_window_regs(const GaeRegs<ITER>& g, const float* __restrict__ tab, int lane, float gamma_f,
                                                float rscale, double& a_sum, double& r_sum, float& vn) {
    constexpr int n = 32 * ITER;
    float vm[ITER + 1];                               // masked values V[k] (1 - done[k-1]) of this lane's steps
#pragma unroll
    for (int i = 0; i < ITER; ++i) {
        float dprev = __shfl_up_sync(0xffffffffu, g.dd[i], 1);
        if (i > 0) {
            const float wrap = __shfl_sync(0xffffffffu, g.dd[i - 1], 31);
            if (lane == 0) dprev = wrap;
        }
        vm[i] = (i == 0 && lane == 0) ? g.vv[0] : __fmul_rn(g.vv[i], __fsub_rn(1.0f, dprev));
    }
    vm[ITER] = __fmul_rn(g.v_last, __fsub_rn(1.0f, g.dd[ITER - 1]));     // lane 31: V[n] (1 - done[n-1])
    a_sum = 0.0;
    r_sum = 0.0;
#pragma unroll
    for (int i = 0; i < ITER; ++i) {
        const int k = lane + 32 * i;
        float v1 = __shfl_down_sync(0xffffffffu, vm[i], 1);
        const float wrap = __shfl_sync(0xffffffffu, vm[i + 1], 0);
        if (lane == 31) v1 = (i + 1 < ITER) ? wrap : vm[ITER];
        const float gk = tab[k], l = tab[n + k];
        const float rk = __fmul_rn(g.rr[i], rscale);
        const float td = __fsub_rn(__fadd_rn(rk, __fmul_rn(gamma_f, v1)), vm[i]);
        a_sum += (double)__fmul_rn(__fmul_rn(td, gk), l);
        r_sum += (double)__fmul_rn(gk, rk);
    }
    vn = __shfl_sync(0xffffffffu, vm[ITER], 31);
}

// MLP branch: horizon == n, one (adv, ret) per window.  ITER > 0: n == 32 * ITER, register-resident windows.
template <int ITER>
__global__ void __launch_bounds__(GAE_WARPS * 32) gae_full_kernel(const float* __restrict__ rewards,
                                                                   const float* __restrict__ values,
                                                                   const float* __restrict__ dones, int B, int n,
                                                                   float gamma_f, float lam_f, float gamma_pow_n, float rscale,
                                                                   int norm_adv, float* __restrict__ adv,
                                                                   float* __restrict__ ret, GaeWs* ws) {
    __shared__ double sh[32];
    extern __shared__ __align__(16) float tab[];       // [n] gamma^k, [n] lam^k (fp32 tables, ppo.py:373-374)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = threadIdx.x; k < n; k += blockDim.x) {
        tab[k] = pow_table(gamma_f, k);
        tab[n + k] = pow_table(lam_f, k);
    }
    __syncthreads();
    double blk_s = 0.0, blk_q = 0.0;               // this warp's share of sum(adv), sum(adv^2) (large-batch path)
    const int b_first = blockIdx.x * GAE_WARPS + warp, b_step = gridDim.x * GAE_WARPS;
    GaeRegs<(ITER > 0 ? ITER : 1)> cur, nxt;
    if constexpr (ITER > 0) {
        if (b_first < B)
            gae_window_load<ITER>(rewards + (long long)b_first * n, values + (long long)b_first * (n + 1), dones + (long long)b_first * n, lane, cur);
    }
    for (int b = b_first; b < B; b += b_step) {
        const float* r = rewards + (long long)b * n;
        const float* v = values + (long long)b * (n + 1);
        const float* d = dones + (long long)b * n;
        double a_sum = 0.0, r_sum = 0.0;
        float vn = 0.0f;
        if constexpr (ITER > 0) {
            const int bn = b + b_step;
            if (bn < B)
                gae_window_load<ITER>(rewards + (long long)bn * n, values + (long long)bn * (n + 1), dones + (long long)bn * n, lane, nxt);
            gae_window_regs<ITER>(cur, tab, lane, gamma_f, rscale, a_sum, r_sum, vn);
            cur = nxt;
        } else {
            for (int k = lane; k < n; k += 32) {
                const float g = tab[k], l = tab[n + k];
                const float rk = __fmul_rn(r[k], rscale);   // ppo.py:452 (x reward_scale, rounded to fp32)
                const float v0 = (k > 0) ? __fmul_rn(v[k], __fsub_rn(1.0f, d[k - 1])) : v[0];
                const float v1 = __fmul_rn(v[k + 1], __fsub_rn(1.0f, d[k]));
                // td = r + gamma*V[k+1] - V[k]; each op rounded separately like the eager reference
                const float td = __fsub_rn(__fadd_rn(rk, __fmul_rn(gamma_f, v1)), v0);
                a_sum += (double)__fmul_rn(__fmul_rn(td, g), l);
                r_sum += (double)__fmul_rn(g, rk);
            }
            if (lane == 0) vn = __fmul_rn(v[n], __fsub_rn(1.0f, d[n - 1]));
        }
        a_sum = warp_sum(a_sum);
        r_sum = warp_sum(r_sum);
        if (lane == 0) {
            const float af = (float)a_sum;
            adv[b] = af;
            ret[b] = __fadd_rn((float)r_sum, __fmul_rn(vn, gamma_pow_n));
            blk_s += (double)af;
            blk_q += (double)af * (double)af;
        }
    }
    if (norm_adv == 1) {
        if (last_block_ticket(&ws->counter, gridDim.x)) normalize_all(adv, (long long)B, sh);
    } else if (norm_adv == 2) {
        // large batch: per-CTA fp64 partials in a fixed order; the last CTA turns them into (mean, max(std, 1e-4)) and
        // gae_normalize_kernel applies them with the whole grid
        const double ts = block_sum((lane == 0) ? blk_s : 0.0, sh);
        const double tq = block_sum((lane == 0) ? blk_q : 0.0, sh);
        if (threadIdx.x == 0) {
            ws->partial[2 * blockIdx.x] = ts;
            ws->partial[2 * blockIdx.x + 1] = tq;
        }
        if (last_block_ticket(&ws->counter, gridDim.x)) {
            if (threadIdx.x == 0) {
                double S = 0.0, Q = 0.0;
                for (unsigned int k = 0; k < gridDim.x; ++k) { S += ws->partial[2 * k]; Q += ws->partial[2 * k + 1]; }
                const double mean = S / (double)B;
                const double var = (Q - S * S / (double)B) / (double)(B - 1);
                const float std_f = (float)sqrt(var > 0.0 ? var : 0.0);
                ws->mean = (float)mean;
                ws->denom = (std_f > 1e-4f) ? std_f : 1e-4f;
            }
        }
    }
}

__global__ void __launch_bounds__(256) gae_normalize_kernel(float* __restrict__ adv, long long total, const GaeWs* __restrict__ ws) {
    const float mean = ws->mean, denom = ws->denom;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        adv[i] = (adv[i] - mean) / denom;
}

// RNN branch: E = n - H + 1 outputs per window, each an H-term sum (ppo.py:389-406).
__global__ void __launch_bounds__(GAE_WARPS * 32) gae_horizon_kernel(const float* __restrict__ rewards,
                                                                      const float* __restrict__ values,
                                                                      const float* __restrict__ dones, int B, int n,
                                                                      int H, float gamma_f, float lam_f,
                                                                      float gamma_pow_h, float rscale, int norm_adv,
                                                                      float* __restrict__ adv,
                                                                      float* __restrict__ ret, GaeWs* ws) {
    extern __shared__ __align__(16) float sm[];
    __shared__ double sh[32];
    const int E = n - H + 1;
    float* gl = sm;                       // [H] gamma^k * ... tables: g[k], then l[k]
    float* ll = sm + H;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* w_r = sm + 2 * H + warp * (3 * n + 1);    // per-warp: r[n], td[n], vm[n+1]
    float* w_td = w_r + n;
    float* w_v = w_td + n;
    for (int k = threadIdx.x; k < H; k += blockDim.x) {
        gl[k] = pow_table(gamma_f, k);
        ll[k] = pow_table(lam_f, k);
    }
    const int b = blockIdx.x * GAE_WARPS + warp;
    if (b < B) {
        const float* r = rewards + (long long)b * n;
        const float* v = values + (long long)b * (n + 1);
        const float* d = dones + (long long)b * n;
        for (int k = lane; k <= n; k += 32) w_v[k] = (k > 0) ? __fmul_rn(v[k], __fsub_rn(1.0f, d[k - 1])) : v[0];
        for (int k = lane; k < n; k += 32) w_r[k] = __fmul_rn(r[k], rscale);
    }
    __syncthreads();
    if (b < B) {
        for (int k = lane; k < n; k += 32)
            w_td[k] = __fsub_rn(__fadd_rn(w_r[k], __fmul_rn(gamma_f, w_v[k + 1])), w_v[k]);
    }
    __syncthreads();
    if (b < B) {
        for (int s = lane; s < E; s += 32) {
            double a_sum = 0.0, r_sum = 0.0;
            for (int k = 0; k < H; ++k) {
                a_sum += (double)__fmul_rn(__fmul_rn(w_td[s + k], gl[k]), ll[k]);
                r_sum += (double)__fmul_rn(gl[k], w_r[s + k]);
            }
            adv[(long long)b * E + s] = (float)a_sum;
            ret[(long long)b * E + s] = __fadd_rn((float)r_sum, __fmul_rn(w_v[s + H], gamma_pow_h));
        }
    }
    if (norm_adv) {
        if (last_block_ticket(&ws->counter, gridDim.x)) normalize_all(adv, (long long)B * E, sh);
    }
}

}  // namespace

static size_t tab_bytes_of(int n) { return (size_t)2 * n * sizeof(float); }

template <int IT>
static int gae_occ(size_t smem) {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gae_full_kernel<IT>, GAE_WARPS * 32, smem) != cudaSuccess || per_sm < 1) per_sm = 4;
    return per_sm;
}

// CTAs of the MLP-branch kernel that are resident at once on this device (cached per window length class)
static int gae_resident_ctas(int n, size_t smem) {
    static int n_sm = 0;
    static int cache[5] = {0, 0, 0, 0, 0};
    if (n_sm == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n_sm = 132;
    }
    const int cls = (n == 32) ? 1 : (n == 64) ? 2 : (n == 128) ? 3 : (n == 256) ? 4 : 0;
    if (cache[cls] == 0) {
        const int per_sm = (cls == 1) ? gae_occ<1>(smem) : (cls == 2) ? gae_occ<2>(smem) : (cls == 3) ? gae_occ<4>(smem)
                         : (cls == 4) ? gae_occ<8>(smem) : gae_occ<0>(smem);
        cache[cls] = per_sm;
    }
    const int cap = n_sm * cache[cls];
    return cap < GAE_MAX_GRID ? cap : GAE_MAX_GRID;
}

int sb200_gae_init() {
    // the generic MLP-branch kernel takes up to 48 KB of tables (n <= 6144) on top of its static reduction scratch, past
    // the 48 KB a kernel gets without opting in
    SB200_CUDA(cudaFuncSetAttribute(gae_full_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 48 * 1024));
    SB200_CUDA(cudaFuncSetAttribute(gae_horizon_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    return SB200_OK;
}

extern "C" size_t sb200_gae_workspace_bytes(int B, int n, int horizon) {
    (void)B; (void)n; (void)horizon;
    return sizeof(GaeWs);
}


extern "C" int sb200_gae_window_f32(const float* rewards, const float* values, const float* dones, int B, int n,
                                    int horizon, double gamma, double lam, double reward_scale, int norm_adv, float* adv,
                                    float* ret, void* workspace, void* stream) {
    SB200_REQUIRE(rewards && values && dones && adv && ret && workspace);
    SB200_REQUIRE(B >= 1 && n >= 1 && horizon >= 1 && horizon <= n);
    cudaStream_t st = (cudaStream_t)stream;
    const float gamma_f = (float)gamma, lam_f = (float)lam;
    const int grid = (B + GAE_WARPS - 1) / GAE_WARPS;
    if (horizon == n) {
        const float gpn = (float)pow(gamma, (double)n);          // Python `gamma ** n_step` (double) -> fp32 scalar
        SB200_REQUIRE((size_t)2 * n * sizeof(float) <= 48 * 1024);
        // persistent grid: the gamma^k / lam^k tables (2n double-precision pow) are built once per CTA, not once per 8
        // windows; windows are walked grid-stride
        // one resident wave: SM count x the occupancy the runtime reports for this instantiation (48 registers -> 5 CTAs per
        // SM, not the 8 the first version assumed: 1184 CTAs ran as 1.6 waves, 0.41 of HBM peak at 2^18 windows)
        const int cap = gae_resident_ctas(n, tab_bytes_of(n));
        const int pgrid = grid < cap ? grid : cap;
        const int mode = !norm_adv ? 0 : (B <= GAE_FUSED_NORM_MAX ? 1 : 2);
        const size_t tab_bytes = (size_t)2 * n * sizeof(float);
#define SB200_GAE_LAUNCH(IT)                                                                                                      \
    gae_full_kernel<IT><<<pgrid, GAE_WARPS * 32, tab_bytes, st>>>(rewards, values, dones, B, n, gamma_f, lam_f, gpn,             \
                                                                  (float)reward_scale, mode, adv, ret, (GaeWs*)workspace)
        if (n == 32) SB200_GAE_LAUNCH(1);
        else if (n == 64) SB200_GAE_LAUNCH(2);
        else if (n == 128) SB200_GAE_LAUNCH(4);
        else if (n == 256) SB200_GAE_LAUNCH(8);
        else SB200_GAE_LAUNCH(0);
#undef SB200_GAE_LAUNCH
        if (mode == 2) {
            const long long nb = ((long long)B + 256 * 4 - 1) / (256 * 4);
            gae_normalize_kernel<<<(unsigned)(nb < 2048 ? nb : 2048), 256, 0, st>>>(adv, (long long)B, (const GaeWs*)workspace);
            return sb200_launch_status(2);
        }
    } else {
        const float gph = (float)pow(gamma, (double)horizon);
        const size_t smem = (size_t)(2 * horizon + GAE_WARPS * (3 * n + 1)) * sizeof(float);
        SB200_REQUIRE(smem <= 200 * 1024);
        gae_horizon_kernel<<<grid, GAE_WARPS * 32, smem, st>>>(rewards, values, dones, B, n, horizon, gamma_f, lam_f,
                                                             gph, (float)reward_scale, norm_adv, adv, ret, (GaeWs*)workspace);
    }
    return sb200_launch_status();
}
