// LSTM stem of RNN-mode PPO (the reference's DEFAULT config: surreal/model/ppo_net.py:143-152,277-279,342-351 -- a
// torch.nn.LSTM(batch_first=True) shared by actor and critic; learner BPTT over eff_len = n_step - horizon + 1 steps,
// ppo.py:389-406,507-525).  Split so that everything GEMM-shaped reuses the MLP kernels:
//
//   pre_x  = z-filter(x) . W_ih^T + b_ih           rows_zfilter_kernel (gather + filter) + sb200_mlp_forward_f32 (1 layer)
//   h_t    = LSTM cell recurrence over time          lstm_fwd_kernel: one CTA per sequence, one thread per gate unit
//   dpre_t = backward through the cell recurrence    lstm_bwd_kernel
//   dW_ih, db_ih = sum dpre^T x ;  dW_hh, db_hh = sum dpre^T h_{t-1}          sb200_linear_bwd_dw_f32 (slabs)
//
// Gate order i, f, g, o (torch).  Weights in the kernel layout: WhhT[k][4H] (transpose of torch's weight_hh_l0 [4H][H]).
// Sequences are tiny here (B = 64 windows x <= 26 steps x H = 100): latency-bound, weights come from L2 every step.
#include "common.cuh"
#include "lstm_dev.cuh"

namespace {

// out[(b*L + t)][0..D) = zfilter(x[b*batch_stride + t*row_stride + 0..D))   (z_filter.py:59-79); zf == nullptr: plain gather
__global__ void __launch_bounds__(256) rows_zfilter_kernel(const float* __restrict__ x, long long row_stride, long long batch_stride,
                                                           int B, int L, int D, const float* __restrict__ zf, float eps,
                                                           float* __restrict__ out, long long ldo) {
    const long long total = (long long)B * L * D;
    const float cnt = (zf != nullptr) ? zf[2 * D] : 1.0f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int d = (int)(i % D);
        const long long r = i / D;
        const int t = (int)(r % L);
        const long long b = r / L;
        float v = x[b * batch_stride + (long long)t * row_stride + d];
        if (zf != nullptr) {
            const float mean = zf[d] / cnt;
            const float var = zf[D + d] / cnt - mean * mean;
            const float sd = fmaxf(sqrtf(var), eps);
            v = fminf(fmaxf((v - mean) / sd, -5.0f), 5.0f);
        }
        out[r * ldo + d] = v;
    }
}

// One CTA per sequence b; thread j < 4H owns gate unit j.
__global__ void __launch_bounds__(1024) lstm_fwd_kernel(const float* __restrict__ pre_x, const float* __restrict__ WhhT,
                                                        const float* __restrict__ b_hh, const float* __restrict__ h0,
                                                        const float* __restrict__ c0, long long ld_cells, int L, int H, int ldh,
                                                        float* __restrict__ h_out, float* __restrict__ h_prev,
                                                        float* __restrict__ gates, float* __restrict__ c_seq,
                                                        float* __restrict__ h_last, float* __restrict__ c_last) {
    extern __shared__ float sm[];
    float* hs = sm;              // [H]
    float* cs = sm + H;          // [H]
    float* gs = sm + 2 * H;      // [4H] gate pre-activations
    const int b = blockIdx.x, j = threadIdx.x, G = 4 * H;
    if (j < H) {
        hs[j] = (h0 != nullptr) ? h0[(long long)b * ld_cells + j] : 0.0f;
        cs[j] = (c0 != nullptr) ? c0[(long long)b * ld_cells + j] : 0.0f;
    }
    __syncthreads();
    for (int t = 0; t < L; ++t) {
        const long long r = (long long)b * L + t;
        if (h_prev != nullptr && j < H) h_prev[r * ldh + j] = hs[j];
        if (j < G) {
            float acc = 0.0f;
            for (int k = 0; k < H; ++k) acc = fmaf(hs[k], WhhT[(long long)k * G + j], acc);
            gs[j] = lstm_gate_pre(pre_x[r * G + j], acc, b_hh[j]);
        }
        __syncthreads();
        if (j < H) {
            LstmGates q;
            float c = cs[j];
            const float h = lstm_cell(gs[j], gs[H + j], gs[2 * H + j], gs[3 * H + j], c, q);
            cs[j] = c;
            hs[j] = h;
            h_out[r * ldh + j] = h;
            if (gates != nullptr) {
                gates[r * G + j] = q.i; gates[r * G + H + j] = q.f; gates[r * G + 2 * H + j] = q.g; gates[r * G + 3 * H + j] = q.o;
            }
            if (c_seq != nullptr) c_seq[r * H + j] = c;
        }
        __syncthreads();
    }
    if (j < H) {
        if (h_last != nullptr) h_last[(long long)b * H + j] = hs[j];
        if (c_last != nullptr) c_last[(long long)b * H + j] = cs[j];
    }
}

// Backward through the recurrence: dh_out[b, t] (gradient w.r.t. h_t from the head) -> dpre[b, t] (w.r.t. the 4H gate
// pre-activations).  The initial cells are detached (ppo.py:507-510): no gradient flows out of t = 0.
__global__ void __launch_bounds__(1024) lstm_bwd_kernel(const float* __restrict__ dh_out, long long ldd,
                                                        const float* __restrict__ gates, const float* __restrict__ c_seq,
                                                        const float* __restrict__ c0, long long ld_cells,
                                                        const float* __restrict__ WhhT, int L, int H, float* __restrict__ dpre) {
    extern __shared__ float sm[];
    float* dh = sm;              // [H] gradient flowing into h_t from the future
    float* dc = sm + H;          // [H]
    float* dg = sm + 2 * H;      // [4H] this step's dpre
    const int b = blockIdx.x, j = threadIdx.x, G = 4 * H;
    const int lane = j & 31, warp = j >> 5, nw = blockDim.x >> 5;
    if (j < H) { dh[j] = 0.0f; dc[j] = 0.0f; }
    __syncthreads();
    for (int t = L - 1; t >= 0; --t) {
        const long long r = (long long)b * L + t;
        if (j < H) {
            const float ig = gates[r * G + j], fg = gates[r * G + H + j], gg = gates[r * G + 2 * H + j], og = gates[r * G + 3 * H + j];
            const float c = c_seq[r * H + j];
            const float cp = (t > 0) ? c_seq[(r - 1) * H + j] : ((c0 != nullptr) ? c0[(long long)b * ld_cells + j] : 0.0f);
            const float tc = tanhf(c);
            const float dht = dh_out[r * ldd + j] + dh[j];
            const float dct = dht * og * (1.0f - tc * tc) + dc[j];
            const float d_i = dct * gg * ig * (1.0f - ig);
            const float d_f = dct * cp * fg * (1.0f - fg);
            const float d_g = dct * ig * (1.0f - gg * gg);
            const float d_o = dht * tc * og * (1.0f - og);
            dg[j] = d_i; dg[H + j] = d_f; dg[2 * H + j] = d_g; dg[3 * H + j] = d_o;
            dpre[r * G + j] = d_i; dpre[r * G + H + j] = d_f; dpre[r * G + 2 * H + j] = d_g; dpre[r * G + 3 * H + j] = d_o;
            dc[j] = dct * fg;
        }
        __syncthreads();
        // dh_{t-1}[k] = sum_j dpre[j] * W_hh[j][k] = sum_j dpre[j] * WhhT[k][j]: a warp per k, lanes over j (coalesced)
        if (t > 0) {
            for (int k = warp; k < H; k += nw) {
                float s = 0.0f;
                for (int q = lane; q < G; q += 32) s = fmaf(dg[q], WhhT[(long long)k * G + q], s);
                s = warp_sum(s);
                if (lane == 0) dh[k] = s;
            }
        }
        __syncthreads();
    }
}

}  // namespace

extern "C" int sb200_rows_zfilter_f32(const float* x, int64_t row_stride, int64_t batch_stride, int B, int L, int D,
                                      const float* zf_stats, double eps, float* out, int64_t ldo, void* stream) {
    SB200_REQUIRE(x && out && B >= 1 && L >= 1 && D >= 1 && ldo >= D);
    const long long total = (long long)B * L * D;
    int grid = (int)((total + 255) / 256);
    if (grid > 132 * 8) grid = 132 * 8;
    rows_zfilter_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, row_stride, batch_stride, B, L, D, zf_stats, (float)eps, out, ldo);
    return sb200_launch_status();
}

static int lstm_threads(int H) { return ((4 * H + 31) / 32) * 32; }

extern "C" int sb200_lstm_forward_f32(const float* pre_x, const float* WhhT, const float* b_hh, const float* h0, const float* c0,
                                      int64_t ld_cells, int B, int L, int H, int ldh, float* h_out, float* h_prev, float* gates,
                                      float* c_seq, float* h_last, float* c_last, void* stream) {
    SB200_REQUIRE(pre_x && WhhT && b_hh && h_out && B >= 1 && L >= 1 && H >= 1 && 4 * H <= 1024 && ldh >= H);
    lstm_fwd_kernel<<<B, lstm_threads(H), (size_t)6 * H * sizeof(float), (cudaStream_t)stream>>>(
        pre_x, WhhT, b_hh, h0, c0, ld_cells, L, H, ldh, h_out, h_prev, gates, c_seq, h_last, c_last);
    return sb200_launch_status();
}

extern "C" int sb200_lstm_backward_f32(const float* dh_out, int64_t ldd, const float* gates, const float* c_seq, const float* c0,
                                       int64_t ld_cells, const float* WhhT, int B, int L, int H, float* dpre, void* stream) {
    SB200_REQUIRE(dh_out && gates && c_seq && WhhT && dpre && B >= 1 && L >= 1 && H >= 1 && 4 * H <= 1024 && ldd >= H);
    lstm_bwd_kernel<<<B, lstm_threads(H), (size_t)6 * H * sizeof(float), (cudaStream_t)stream>>>(dh_out, ldd, gates, c_seq, c0,
                                                                                               ld_cells, WhhT, L, H, dpre);
    return sb200_launch_status();
}
