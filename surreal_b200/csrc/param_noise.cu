// Parameter-space exploration noise of the DDPG actors (surreal/agent/param_noise.py:9-74, ddpg_agent.py:136-153):
// per-actor perturbed parameter images, the adaptive sigma update, and the host-observation act that runs on them.
//
// Image k of N is the actor's flat FlatNet buffer, perturbed:  W' = fl32((double)W + sigma_k * z),  z ~ N(0,1) in
// float64 -- numpy's `p + np.random.normal(0, sigma, shape)` on a float32 array, rounded to float32 once by
// ModuleDict.load (module_dict.py:47-63).  Images are [N][actor_stride] floats; padding columns stay zero.
#include "common.cuh"

namespace {

constexpr int NT = 256;
// Philox key of the perturbation stream: the agent seed XOR this constant.  The action noise (rollout.cu) keys on the
// agent seed itself, the synthetic envs and the pixel stream on other constants, so no two streams share a key.
constexpr unsigned long long PN_KEY = 0xC2B2AE3D27D4EB4Full;

struct PnLayout {
    int L;
    int N[SB200_MAX_LAYERS];
    int ldw[SB200_MAX_LAYERS];
    long long w[SB200_MAX_LAYERS], wend[SB200_MAX_LAYERS], b[SB200_MAX_LAYERS];
    long long g[SB200_MAX_LAYERS], beta[SB200_MAX_LAYERS];    // LayerNorm gain / bias segments, -1: none
};

// Is flat offset p a parameter (true) or a padding column / the tail up to actor_stride (false)?  LayerNorm gains and
// biases are parameters too: the reference perturbs every entry of the state dict (param_noise.py:14-23,61-69).
__device__ __forceinline__ bool is_param(const PnLayout& P, long long p) {
    for (int l = 0; l < P.L; ++l) {
        if (p >= P.w[l] && p < P.wend[l]) return (int)((p - P.w[l]) % P.ldw[l]) < P.N[l];
        if (p >= P.b[l] && p < P.b[l] + P.ldw[l]) return (int)(p - P.b[l]) < P.N[l];
        if (P.g[l] >= 0 && p >= P.g[l] && p < P.g[l] + P.ldw[l]) return (int)(p - P.g[l]) < P.N[l];
        if (P.beta[l] >= 0 && p >= P.beta[l] && p < P.beta[l] + P.ldw[l]) return (int)(p - P.beta[l]) < P.N[l];
    }
    return false;
}

// Two N(0,1) in float64 from two 32-bit words (Box-Muller, double precision: the noise is added in float64).
__device__ __forceinline__ double2 box_muller_f64(unsigned int a, unsigned int b) {
    const double u1 = ((double)a + 1.0) * 2.3283064365386963e-10;      // (0, 1]
    const double u2 = (double)b * 2.3283064365386963e-10;              // [0, 1)
    const double rad = sqrt(-2.0 * log(u1));
    double s, c;
    sincos(__dmul_rn(6.283185307179586, u2), &s, &c);
    return make_double2(__dmul_rn(rad, c), __dmul_rn(rad, s));
}

// AdaptiveNormalParameterNoise.apply (param_noise.py:49-60): when i > 0, mean = dist / i in float32 (torch arithmetic,
// compared with target in float32), sigma /= alpha if mean > target else sigma *= alpha, in float64.
__device__ __forceinline__ double adapted_sigma(double sg, float d, unsigned long long i, double alpha, float target) {
    if (i == 0ull) return sg;
    const float mean = __fdiv_rn(d, (float)i);
    return (mean > target) ? __ddiv_rn(sg, alpha) : __dmul_rn(sg, alpha);
}

// grid (ceil(stride / (4 * NT)), N): each thread writes 4 consecutive entries of one image from one Philox call.
__global__ void __launch_bounds__(NT) param_noise_apply_kernel(PnLayout P, const float* __restrict__ W, int N,
                                                              float* __restrict__ images, long long stride,
                                                              double* __restrict__ sigma,
                                                              const double* __restrict__ unit_noise,
                                                              unsigned long long key, unsigned long long fetch,
                                                              const float* __restrict__ dist,
                                                              sb200_param_noise_state* state, double alpha,
                                                              float target) {
    const int k = blockIdx.y;
    const unsigned long long i = (state != nullptr) ? *(volatile unsigned long long*)&state->acts : 0ull;
    const double sg = (state != nullptr) ? adapted_sigma(sigma[k], dist[k], i, alpha, target) : sigma[k];
    const long long p0 = ((long long)blockIdx.x * NT + threadIdx.x) * 4;
    if (p0 < stride) {
        double z[4] = {0.0, 0.0, 0.0, 0.0};
        if (unit_noise == nullptr) {
            const Philox4 r = philox4x32_10(key, fetch, ((unsigned long long)k << 32) | (unsigned long long)(p0 >> 2));
            const double2 a = box_muller_f64(r.x, r.y), b = box_muller_f64(r.z, r.w);
            z[0] = a.x; z[1] = a.y; z[2] = b.x; z[3] = b.y;
        }
        float v[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const long long p = p0 + c;
            v[c] = 0.0f;
            if (is_param(P, p)) {
                const double zz = (unit_noise != nullptr) ? unit_noise[(long long)k * stride + p] : z[c];
                v[c] = __double2float_rn(__dadd_rn((double)W[p], __dmul_rn(sg, zz)));
            }
        }
        *reinterpret_cast<float4*>(images + (long long)k * stride + p0) = make_float4(v[0], v[1], v[2], v[3]);
    }
    if (state != nullptr && last_block_ticket(&state->ticket, gridDim.x * gridDim.y)) {
        // every CTA has drawn with the old sigma / counter: publish the new sigma and reset the act counter (i = 0)
        for (int a = threadIdx.x; a < N; a += NT) sigma[a] = adapted_sigma(sigma[a], dist[a], i, alpha, target);
        if (threadIdx.x == 0) state->acts = 0ull;
    }
}

}  // namespace

extern "C" int sb200_ddpg_param_noise_apply_f32(const sb200_mlp* net, int N, float* images, int64_t actor_stride,
                                                double* sigma, const double* unit_noise, uint64_t seed,
                                                uint64_t fetch_index, const float* dist, sb200_param_noise_state* state,
                                                double alpha, double target_stddev, void* stream) {
    SB200_REQUIRE(net != nullptr && images != nullptr && sigma != nullptr && N >= 1 && N <= 65535);
    SB200_REQUIRE(net->n_layers >= 1 && net->n_layers <= SB200_MAX_LAYERS && net->aux_layer < 0);
    SB200_REQUIRE(actor_stride >= 4 && actor_stride % 32 == 0 && ((uintptr_t)images & 127u) == 0);
    SB200_REQUIRE(state == nullptr || (dist != nullptr && alpha > 0.0));
    PnLayout P;
    P.L = net->n_layers;
    const float* base = net->W[0];
    for (int l = 0; l < net->n_layers; ++l) {
        SB200_REQUIRE(net->ldw[l] >= net->dims[l + 1]);
        P.N[l] = net->dims[l + 1];
        P.ldw[l] = net->ldw[l];
        P.w[l] = (long long)(net->W[l] - base);
        P.wend[l] = P.w[l] + (long long)net->dims[l] * net->ldw[l];
        P.b[l] = (long long)(net->b[l] - base);
        SB200_REQUIRE(P.w[l] >= 0 && P.b[l] >= 0 && P.wend[l] <= actor_stride && P.b[l] + net->ldw[l] <= actor_stride);
        SB200_REQUIRE((net->ln_g[l] == nullptr) == (net->ln_b[l] == nullptr));
        P.g[l] = net->ln_g[l] != nullptr ? (long long)(net->ln_g[l] - base) : -1;
        P.beta[l] = net->ln_b[l] != nullptr ? (long long)(net->ln_b[l] - base) : -1;
        SB200_REQUIRE(net->ln_g[l] == nullptr || (P.g[l] >= 0 && P.beta[l] >= 0 && P.g[l] + net->ldw[l] <= actor_stride &&
                                                  P.beta[l] + net->ldw[l] <= actor_stride));
    }
    const dim3 grid((unsigned)((actor_stride + 4 * NT - 1) / (4 * NT)), (unsigned)N);
    param_noise_apply_kernel<<<grid, NT, 0, (cudaStream_t)stream>>>(
        P, base, N, images, (long long)actor_stride, sigma, unit_noise, (unsigned long long)seed ^ PN_KEY,
        (unsigned long long)fetch_index, dist, state, alpha, (float)target_stddev);
    return sb200_launch_status();
}
