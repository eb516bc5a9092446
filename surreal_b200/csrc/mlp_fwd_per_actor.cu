// Per-actor MLP forward: row k of the batch runs through actor k's own parameter image (parameter-space exploration
// noise, surreal/agent/param_noise.py:9-74, where every agent process acts with its own perturbed copy of the policy).
// Replaces the batch-1 `self.model(obs_tensor)` of ddpg_agent.py:173 for N perturbed actors at once, and the
// `original_model` forward of AdaptiveNormalParameterNoise.compute_action_distance (param_noise.py:42-47).
//
// Nothing is shared between rows, so every weight byte crosses HBM once per step: the kernel is bound by HBM
// bandwidth, not by math.  One CTA owns one row.  Each thread streams float4 columns of W (layout [K][ldw], read once,
// no L1 allocation) and keeps its FMAs in registers; with 8 resident CTAs of 256 threads per SM and 4 independent 16-byte
// loads in flight per thread, about 128 KB per SM are outstanding, well above the bandwidth-delay product of HBM3.
// Staging through shared memory would add a write and a read per byte with nothing to reuse.
//
// Arithmetic: fp32 FFMA.  Output column j of a layer is split into S slices of the K inputs; each slice accumulates its
// inputs in ascending order, and the slices are added in ascending order, then the bias.  S depends only on the layer
// shape, so the result does not change from run to run or with N.
#include "common.cuh"

namespace {

constexpr int PT = 256;
constexpr int PART_FLOATS = 4 * PT;

struct PaLayout {
    int L;
    int dims[SB200_MAX_LAYERS + 1];
    int act[SB200_MAX_LAYERS];
    int ldw[SB200_MAX_LAYERS];
    long long w[SB200_MAX_LAYERS];   // offsets in floats from the image base
    long long b[SB200_MAX_LAYERS];
    long long g[SB200_MAX_LAYERS];   // LayerNorm gain / bias after layer l, -1: none
    long long beta[SB200_MAX_LAYERS];
    float ln_eps;
};

// One Linear + activation of one row: hout[0:N) = act(hin[0:K) @ W + b).  W / b point into the row's image.
__device__ __forceinline__ void layer_row(const float* __restrict__ W, const float* __restrict__ b, int K, int N,
                                          int ldw, int act, const float* hin, float* hout, float* part) {
    const int G = ldw >> 2;
    int S = PT / G;
    S = S < 1 ? 1 : (S > K ? K : S);
    const int kper = (K + S - 1) / S;
    for (int item = threadIdx.x; item < G * S; item += PT) {
        const int s = item / G, g = item - s * G;
        const int k0 = s * kper, k1 = min(K, k0 + kper);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        const float* wp = W + (long long)k0 * ldw + 4 * g;
#pragma unroll 4
        for (int k = k0; k < k1; ++k) {
            const float4 w = ld_stream4(wp);
            wp += ldw;
            const float h = hin[k];
            acc.x = fmaf(h, w.x, acc.x);
            acc.y = fmaf(h, w.y, acc.y);
            acc.z = fmaf(h, w.z, acc.z);
            acc.w = fmaf(h, w.w, acc.w);
        }
        *reinterpret_cast<float4*>(part + (long long)s * ldw + 4 * g) = acc;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < N; j += PT) {
        float v = part[j];
        for (int s = 1; s < S; ++s) v = __fadd_rn(v, part[s * ldw + j]);
        hout[j] = apply_act(__fadd_rn(v, __ldg(b + j)), act);
    }
    __syncthreads();
}

// LayerNorm of one row h[0:N) in place (g / b point into the row's image).  Warp 0 reduces in a fixed order (lanes
// stride the row, then a butterfly), two passes, biased variance; an all-zero row gives exactly b.
__device__ __forceinline__ void layernorm_row(const float* __restrict__ g, const float* __restrict__ b, int N, float eps,
                                              float* h, float* part) {
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        float s = 0.0f;
        for (int j = lane; j < N; j += 32) s = __fadd_rn(s, h[j]);
        const float mean = __fdiv_rn(warp_sum(s), (float)N);
        float q = 0.0f;
        for (int j = lane; j < N; j += 32) {
            const float d = __fsub_rn(h[j], mean);
            q = fmaf(d, d, q);
        }
        const float var = __fdiv_rn(warp_sum(q), (float)N);
        if (lane == 0) {
            part[0] = mean;
            part[1] = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var, eps)));
        }
    }
    __syncthreads();
    const float mean = part[0], rstd = part[1];
    for (int j = threadIdx.x; j < N; j += PT) h[j] = fmaf(__fmul_rn(__fsub_rn(h[j], mean), rstd), __ldg(g + j), __ldg(b + j));
    __syncthreads();
}

// Whole network on one row; returns the shared-memory buffer that holds the output.
__device__ __forceinline__ float* net_row(const PaLayout& P, const float* __restrict__ base, float* h0, float* h1,
                                          float* part) {
    float* in = h0;
    float* out = h1;
    for (int l = 0; l < P.L; ++l) {
        layer_row(base + P.w[l], base + P.b[l], P.dims[l], P.dims[l + 1], P.ldw[l], P.act[l], in, out, part);
        if (P.g[l] >= 0) layernorm_row(base + P.g[l], base + P.beta[l], P.dims[l + 1], P.ln_eps, out, part);
        float* t = in;
        in = out;
        out = t;
    }
    return in;
}

__global__ void __launch_bounds__(PT) mlp_fwd_per_actor_kernel(PaLayout P, const float* __restrict__ images,
                                                              long long actor_stride, const float* __restrict__ x,
                                                              long long ldx, float* __restrict__ out, long long ld_out,
                                                              const float* __restrict__ shared, float* __restrict__ dist,
                                                              int dist_interval, sb200_param_noise_state* state,
                                                              int part_floats, int wpad) {
    extern __shared__ __align__(16) float sm[];
    float* part = sm;                       // [part | h0 | h1 | pert]
    float* h0 = part + part_floats;
    float* h1 = h0 + wpad;
    float* pert = h1 + wpad;
    const int row = blockIdx.x;
    const int A = P.dims[P.L];
    // the act counter is read before this CTA's ticket, so every CTA sees the value of this launch
    const unsigned long long acts = (state != nullptr) ? *(volatile unsigned long long*)&state->acts : 0ull;
    for (int k = threadIdx.x; k < P.dims[0]; k += PT) h0[k] = x[(long long)row * ldx + k];
    __syncthreads();
    const float* y = net_row(P, images + (long long)row * actor_stride, h0, h1, part);
    for (int j = threadIdx.x; j < A; j += PT) {
        out[(long long)row * ld_out + j] = y[j];
        pert[j] = y[j];
    }
    if (shared != nullptr && dist != nullptr && state != nullptr && acts % (unsigned long long)dist_interval == 0ull) {
        // compute_action_distance (param_noise.py:42-47): sqrt(sum((pi_orig(s) - pi_pert(s))^2)), overwritten
        __syncthreads();
        for (int k = threadIdx.x; k < P.dims[0]; k += PT) h0[k] = x[(long long)row * ldx + k];
        __syncthreads();
        const float* yo = net_row(P, shared, h0, h1, part);
        if (threadIdx.x == 0) {
            float s = 0.0f;
            for (int j = 0; j < A; ++j) {
                const float d = __fsub_rn(yo[j], pert[j]);
                s = __fadd_rn(s, __fmul_rn(d, d));
            }
            dist[row] = sqrtf(s);
        }
    }
    if (state != nullptr) {
        if (last_block_ticket(&state->ticket, gridDim.x) && threadIdx.x == 0) state->acts = acts + 1ull;   // i += 1
    }
}

}  // namespace

// Shared memory of one CTA: partial sums (S * ldw <= max(4 * PT, ldw) floats), two activation rows, the perturbed output.
static size_t per_actor_smem_bytes(const sb200_mlp* net, int* part_out, int* wpad_out) {
    int maxw = 0, maxldw = 0;
    for (int l = 0; l <= net->n_layers; ++l) maxw = net->dims[l] > maxw ? net->dims[l] : maxw;
    for (int l = 0; l < net->n_layers; ++l) maxldw = net->ldw[l] > maxldw ? net->ldw[l] : maxldw;
    *wpad_out = 4 * ((maxw + 3) / 4);
    *part_out = PART_FLOATS > maxldw ? PART_FLOATS : maxldw;
    return (size_t)(*part_out + 3 * *wpad_out) * sizeof(float);
}

extern "C" int sb200_mlp_forward_per_actor_f32(const sb200_mlp* net, int64_t actor_stride, const float* x, int64_t ldx,
                                               int N, float* out, int64_t ld_out, const sb200_mlp* shared, float* dist,
                                               int dist_interval, sb200_param_noise_state* state, void* stream) {
    SB200_REQUIRE(net != nullptr && x != nullptr && out != nullptr && N >= 1);
    SB200_REQUIRE(net->n_layers >= 1 && net->n_layers <= SB200_MAX_LAYERS && net->aux_layer < 0);
    SB200_REQUIRE(actor_stride >= 0 && actor_stride % 4 == 0 && ldx >= net->dims[0] && ld_out >= net->dims[net->n_layers]);
    SB200_REQUIRE(shared == nullptr || (dist != nullptr && state != nullptr && dist_interval >= 1));
    PaLayout P;
    P.L = net->n_layers;
    const float* base = net->W[0];
    for (int l = 0; l <= net->n_layers; ++l) P.dims[l] = net->dims[l];
    for (int l = 0; l < net->n_layers; ++l) {
        SB200_REQUIRE(net->dims[l] >= 1 && net->dims[l + 1] >= 1 && net->ldw[l] >= net->dims[l + 1] && net->ldw[l] % 4 == 0);
        P.act[l] = net->act[l];
        P.ldw[l] = net->ldw[l];
        P.w[l] = (long long)(net->W[l] - base);
        P.b[l] = (long long)(net->b[l] - base);
        SB200_REQUIRE(P.w[l] % 4 == 0 && P.b[l] >= 0);
        SB200_REQUIRE((net->ln_g[l] == nullptr) == (net->ln_b[l] == nullptr));
        SB200_REQUIRE(net->ln_g[l] == nullptr || (l + 1 < net->n_layers && net->ln_eps > 0.0f));
        P.g[l] = net->ln_g[l] != nullptr ? (long long)(net->ln_g[l] - base) : -1;
        P.beta[l] = net->ln_b[l] != nullptr ? (long long)(net->ln_b[l] - base) : -1;
        SB200_REQUIRE(net->ln_g[l] == nullptr || (P.g[l] >= 0 && P.beta[l] >= 0));
        if (shared != nullptr)     // the unperturbed net must have the image's layout
            SB200_REQUIRE(shared->n_layers == net->n_layers && shared->W[l] - shared->W[0] == P.w[l] &&
                          shared->b[l] - shared->W[0] == P.b[l] && shared->ldw[l] == net->ldw[l] &&
                          shared->dims[l + 1] == net->dims[l + 1] &&
                          (shared->ln_g[l] == nullptr ? -1 : shared->ln_g[l] - shared->W[0]) == P.g[l] &&
                          (shared->ln_b[l] == nullptr ? -1 : shared->ln_b[l] - shared->W[0]) == P.beta[l]);
    }
    P.ln_eps = net->ln_eps;
    SB200_REQUIRE(((uintptr_t)base & 15u) == 0 && (shared == nullptr || ((uintptr_t)shared->W[0] & 15u) == 0));
    int part = 0, wpad = 0;
    const size_t smem = per_actor_smem_bytes(net, &part, &wpad);
    if (smem > 48 * 1024) return SB200_ERR_UNSUPPORTED;
    mlp_fwd_per_actor_kernel<<<N, PT, smem, (cudaStream_t)stream>>>(
        P, base, (long long)actor_stride, x, (long long)ldx, out, (long long)ld_out,
        shared != nullptr ? shared->W[0] : nullptr, dist, dist_interval, state, part, wpad);
    return sb200_launch_status();
}
