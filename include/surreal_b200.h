/* libsurreal_b200 -- C-ABI of the H100-native actor -> replay -> learner hot path.
 *
 * The reference (SurrealAI/surreal) is pure Python and has NO FFI / operator registry: its plugin
 * surface is three Python base classes (Agent / Replay / Learner, SURVEY.md §8b).  This header is
 * therefore the boundary a maintainer would bind from those classes (ctypes stub in
 * INTEGRATION.md); every entry point cites the reference code whose arithmetic it replaces.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _h; fp32, row-major, contiguous
 *     unless a leading dimension is given; `stream` is a cudaStream_t passed as void*.
 *   - every call is asynchronous on `stream`, allocates nothing, and returns SB200_OK (0) or a
 *     negative sb200 status; no exceptions cross the ABI.  Workspaces are caller-owned.
 *   - weights use the KERNEL LAYOUT: W[l] is [in_l][ldw_l] (ldw = out rounded up to 4), i.e. the
 *     transpose of torch.nn.Linear.weight, zero in the padding columns; b[l] is [ldw_l].
 *   - there is no CPU fallback: without a CUDA device every compute entry fails.
 */
#ifndef SURREAL_B200_H
#define SURREAL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB200_OK 0
#define SB200_ERR_ARG (-1)
#define SB200_ERR_CUDA (-2)
#define SB200_ERR_UNSUPPORTED (-3)

#define SB200_ACT_NONE 0
#define SB200_ACT_RELU 1
#define SB200_ACT_TANH 2
#define SB200_MAX_LAYERS 4

int sb200_version(void);
/* One-time per-process setup on the current device (kernel attributes); fails on devices other than sm_90 (H100).
 * Must run before any compute entry (and before CUDA-graph capture). */
int sb200_init(void);
const char* sb200_status_string(int status);
/* SM count / compute capability of the current device (fails without a GPU). */
int sb200_device_info(int* sm_count, int* cc_major, int* cc_minor);
/* Number of CUDA kernels this library has launched so far (optionally reset) -- bench.py's gpu_launches. */
uint64_t sb200_launch_counter(int reset);
/* Account for kernels submitted through a replayed CUDA graph (counted once at capture time). */
void sb200_launch_counter_add(uint64_t kernels);

/* ---------------------------------------------------------------------------------------------
 * Networks.  One descriptor covers PPO_ActorNetwork / PPO_CriticNetwork
 * (surreal/model/model_builders/builders.py:86-175), ActorNetworkX / CriticNetworkX (:35-84).
 * `aux_layer` >= 0 concatenates `aux` columns to the input of that layer (the DDPG critic's
 * cat(h, action), builders.py:80-83). */
typedef struct {
    int n_layers;                       /* 1..SB200_MAX_LAYERS */
    int dims[SB200_MAX_LAYERS + 1];     /* dims[0] = input width (without aux), dims[l+1] = out of layer l */
    int act[SB200_MAX_LAYERS];          /* SB200_ACT_* applied after layer l */
    const float* W[SB200_MAX_LAYERS];   /* [in_l(+aux)][ldw_l] */
    const float* b[SB200_MAX_LAYERS];   /* [ldw_l] */
    int ldw[SB200_MAX_LAYERS];
    int aux_layer;                      /* -1: none */
    int aux_dim;
    /* LayerNorm after layer l's activation (ActorNetworkX / CriticNetworkX with use_layernorm, builders.py:42-48,64-77):
     * y = (h - mean) * rsqrt(var + ln_eps) * ln_g[l] + ln_b[l] over the dims[l+1] columns of a row, biased variance
     * (torch.nn.LayerNorm).  ln_g[l] = ln_b[l] = NULL: none (a zero-initialised descriptor has no LayerNorm).  Hidden
     * layers only.  Only the entries that say so implement it; every other entry rejects such a descriptor. */
    const float* ln_g[SB200_MAX_LAYERS];    /* [ldw_l] gain */
    const float* ln_b[SB200_MAX_LAYERS];    /* [ldw_l] bias */
    float ln_eps;
} sb200_mlp;

/* ZFilter (surreal/model/z_filter.py:59-79): stats = running_sum[D] | running_sumsq[D] | count[1]. */
typedef struct {
    const float* stats;                 /* NULL: no filter */
    float eps;                          /* 1e-5 in the reference */
} sb200_zfilter;

/* Input rows of a forward pass.  Either a plain matrix (x, ldx, rows) or, when win_n > 0, the
 * virtual concatenation cat([obs, obs_next], dim=1).view(-1, D) of ppo.py:376-383 WITHOUT copying:
 * row r -> (b, k) = (r / (win_n+1), r % (win_n+1)); k < win_n ? x[(b*win_n+k)*ldx] : x_next[b*ldx]. */
typedef struct {
    const float* x;
    const float* x_next;                /* only when win_n > 0 */
    int64_t ldx;
    int64_t rows;                       /* total rows ( = B*(win_n+1) when win_n > 0 ) */
    int win_n;
    const float* aux;                   /* [rows][aux_ld] or NULL */
    int64_t aux_ld;
    float* save_x;                      /* optional: receives the z-filtered input rows [rows][ld_save_x] */
    int64_t ld_save_x;
    /* optional, layers with LayerNorm: ln_save[l] receives the LayerNorm output [rows][ld_ln_save[l]] (the next layer's
     * input; save[l] then holds the activation BEFORE the LayerNorm), ln_stats[l] the per-row (mean, rstd) [rows][2] */
    float* ln_save[SB200_MAX_LAYERS];
    int64_t ld_ln_save[SB200_MAX_LAYERS];
    float* ln_stats[SB200_MAX_LAYERS];
} sb200_rows;

/* Fused forward of a whole MLP on row tiles (z-filter -> Linear/act x n_layers): activations stay in
 * shared memory; `save[l]` (may be NULL) receives layer l's post-activation output [rows][ld_save[l]]
 * (needed by the backward pass); save[n_layers-1] is the network output.
 * Replaces: ppo_net.py:253-315 (forward_actor / forward_critic), builders.py:114-132,160-175,
 * ddpg_net.py:63-91. */
int sb200_mlp_forward_f32(const sb200_mlp* net, const sb200_zfilter* zf, const sb200_rows* in,
                          float* const* save, const int64_t* ld_save, void* stream);
/* Same, with the kernel family chosen by the caller: variant 0 = default dispatch, 1 = tensor-core 3xTF32 tiles of
 * 32 rows, 2 = fp32 FFMA tiles of 32 rows (both <= 128 registers per thread, 2 CTAs/SM).  Variant 1 is what large
 * batches get by default (631 us on the 132 096-row critic pass).  Launching 1 and 2 on two streams over the two
 * halves of a batch -- tensor pipe and FMA pipe at once -- was measured SLOWER (700-760 us): both kernels are bound
 * by instruction issue, not by their math pipes; it stays available as an experiment (ops.mlp_forward_dual). */
int sb200_mlp_forward_variant_f32(const sb200_mlp* net, const sb200_zfilter* zf, const sb200_rows* in,
                                  float* const* save, const int64_t* ld_save, int variant, void* stream);
/* Small-batch inference on PRE-PACKED weights (the actors' per-step policy forward, ppo_agent.py:138-141 /
 * ddpg_agent.py:170-176): pack once per parameter version, then every step's forward reads the weights in
 * mma-fragment order and a 4-CTA cluster shares each 32-row tile (each CTA keeps a quarter of the weights resident in
 * shared memory and exchanges layer outputs through distributed shared memory).
 *   pack_floats: size of `packed` in floats (0: this architecture is not supported -- use sb200_mlp_forward_f32;
 *     supported = every layer but the last wider than 32 outputs).
 *   pack_tf32: (re)builds `packed` from net->W.  Must be re-run after ANY change of the parameters.
 *   forward_packed: out[rows][ld_out] = network output; same numerics class as forward mode 1. */
size_t sb200_mlp_pack_floats(const sb200_mlp* net);
int sb200_mlp_pack_tf32(const sb200_mlp* net, float* packed, void* stream);
int sb200_mlp_forward_packed_f32(const sb200_mlp* net, const float* packed, const sb200_zfilter* zf,
                                 const sb200_rows* in, float* out, int64_t ld_out, void* stream);
/* Hopper large-batch forward (csrc/mlp_fwd_tc5.cu): wgmma tf32 tiles of 128 rows (two warpgroups of 64) with the
 * accumulators in registers, weights streamed by the TMA engine (cp.async.bulk), 3xTF32 split for fp32-level
 * accuracy, both hidden layers and the narrow head fused in one persistent kernel (one CTA per SM).  The critic pass of
 * PPOLearner._gae_and_return (ppo.py:376-387: B*(n+1) rows through D-256-256-1) is its customer.
 *   supported: 3 layers, ReLU-ReLU-any, dims[0] a multiple of 32 up to 256, dims[1] and dims[2] multiples of 32 (both
 *     <= 256), dims[3] <= 8, no aux input, rows >= 128.  Returns 1 / 0.
 *   workspace_bytes: caller-owned scratch for the per-call weight images (hi / lo planes in operand layout); 0 when
 *     unsupported.  One workspace must not be shared by calls that may run concurrently.
 *   forward: out[rows][ld_out] = network output (only the last layer is written: no saved activations, no save_x).
 *     SB200_ERR_UNSUPPORTED for other shapes -- callers then use sb200_mlp_forward_f32.  max_grid >= 1 caps the
 *     persistent grid below one CTA per SM (0: no cap); tiles and their arithmetic do not depend on it. */
int sb200_mlp_tc5_supported(const sb200_mlp* net, int64_t rows);
size_t sb200_mlp_tc5_workspace_bytes(const sb200_mlp* net);
int sb200_mlp_forward_tc5_f32(const sb200_mlp* net, const sb200_zfilter* zf, const sb200_rows* in, float* out,
                              int64_t ld_out, void* workspace, int max_grid, void* stream);
/* ---------------------------------------------------------------------------------------------
 * CNN stem of the pixel path (CNNStemNetwork, builders.py:8-33; used by PPOModel / DDPGModel with pixel input,
 * ppo_net.py:136-140,268-273,368-375): Conv2d(16, k8, s4)+ReLU -> Conv2d(32, k4, s2)+ReLU -> Flatten -> Linear+ReLU.
 * The two convolutions (csrc/stem.cu); the Linear layer is an ordinary sb200_mlp layer.
 *   frames [rows][C][H][W] (uint8 scaled by in_scale = 1/255, or float); outputs [rows][COUT][HO][WO] (torch order);
 *   Wk: kernel layout [(c*KS + ky)*KS + kx][COUT] = transpose of torch's [COUT][C][KS][KS]; bias [COUT].
 *   layer 1 = Conv2d(16, k8, s4), layer 2 = Conv2d(32, k4, s2) (the reference's fixed stem).
 *   forward: y = relu(conv(x * in_scale) + bias).
 *   backward_dw: partial gradients of `frames` frames w.r.t. Wk / bias, written into `splits` slabs at
 *     slab_w + s*slab_stride / slab_b + s*slab_stride (reduce with sb200_grad_reduce_norm_f32); dy = gradient w.r.t. the
 *     PRE-activation output.
 *   backward_dx (layer 2 only): dx = relu'(act) * conv_transpose(dy), act = layer 1's output (may be NULL: no mask). */
int sb200_conv_forward_f32(int layer, const void* x, int in_u8, int64_t frames, int CIN, int H, int W, const float* Wk,
                           const float* bias, double in_scale, float* y, void* stream);
int sb200_conv_backward_dw_f32(int layer, const void* x, int in_u8, const float* dy, int64_t frames, int CIN, int H, int W,
                               double in_scale, float* slab_w, float* slab_b, int64_t slab_stride, int splits, void* stream);
int sb200_conv_backward_dx_f32(int layer, const float* dy, const float* Wk, const float* act, int64_t frames, int CIN, int H,
                               int W, float* dx, void* stream);

/* ---------------------------------------------------------------------------------------------
 * One-shot all-reduce over NVLink peer memory (csrc/peer_allreduce.cu) for the small exchanges of the data-parallel
 * learner (SURVEY §8e; the reference has no collective at all): every rank maps every other rank's "symmetric" buffer
 * (cudaMalloc + CUDA IPC), one kernel per all-reduce publishes its slice, waits for the peers' flags and sums the slots
 * in rank order (bit-identical result on all ranks).
 *   par_alloc / par_open / par_close: allocate + export (64-byte IPC handle) / map a peer's buffer / release.
 *   par_allreduce_f32: out = scale * sum over ranks of x (n <= max_floats); with opt_workspace != NULL it also does
 *     the gradient-norm / step bookkeeping of sb200_grad_reduce_norm_f32 on the result.  EVERY rank must issue the
 *     same sequence of calls on one sb200_par (use separate ones for streams that run concurrently).
 *   par_allreduce_f64: the same for a few float64 scalars. */
typedef struct {
    void* peers[8];                     /* device pointers of every rank's symmetric buffer, valid in THIS process */
    int world;
    int rank;
    int64_t max_floats;                 /* capacity of one slot */
} sb200_par;
size_t sb200_par_buffer_bytes(int64_t max_floats);
int sb200_par_alloc(int64_t max_floats, void** ptr_out, void* handle_out);
int sb200_par_open(const void* handle, void** ptr_out);
int sb200_par_close(void* ptr, int own);
int sb200_par_allreduce_f32(const sb200_par* ctx, const float* x, float* out, int64_t n, double scale, int bump_step,
                            void* opt_workspace, const int* stop_flag, void* stream);
int sb200_par_allreduce_f64(const sb200_par* ctx, const double* x, double* out, int n, double scale, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Persistent learner kernel (csrc/epoch2.cu): ALL minibatch epochs of BOTH optimisers of PPOLearner._optimize
 * (surreal/learner/ppo.py:194-353 losses + updates, 541-557 epoch loops + KL early stop) in ONE launch of one CTA per SM --
 * forward, loss, backward, slab reduction, gradient clip, Adam, post-step forward and KL of every epoch; row blocks of 16 run
 * forward -> loss -> input gradients without grid barriers, weight gradients are a second wave, an epoch costs 4 grid
 * barriers (5 in adapt mode).  It writes the same buffers and statistics as the launch chain it replaces
 * (sb200_mlp_forward_f32 + sb200_ppo_policy_loss_f32 / sb200_value_loss_f32 + sb200_linear_bwd_* +
 * sb200_grad_reduce_norm_f32 + sb200_clip_adam_f32 + sb200_ppo_kl_f32).
 *   sb200_epochs = the argument block of ONE optimiser: 3 layers ReLU-ReLU-any, no aux input, head <= 32 wide, widths <= 512.
 *   net->W / net->b must point INTO `params` (the flat buffer Adam updates); x_in/h1/h2/out/d1/d2/dpre are [M][ru4(width)]
 *   with zero padding columns (x_in receives the z-filtered input rows).
 *   mode 0 clip / 1 adapt (policy: out = tanh mean, log_var at params[extra_off..+A), early stop above stop_threshold),
 *   mode 2 value (MSE on `returns`).  grid: upper bound on the CTAs to launch (0: one per SM); cta_shift and workspace of the
 *   block are unused (the call takes the workspace).
 *   par != NULL with world > 1: data-parallel -- the KL scalar and the flat gradient are averaged over the ranks inside
 *   the kernel through the symmetric buffers of `par` (every rank must launch the same sequence). */
typedef struct {
    const sb200_mlp* net;
    float* params;
    int64_t n_params;
    int extra_off;
    const float* x;
    int64_t ldx;
    int M;
    const float* zf_stats;              /* NULL: no z-filter */
    double zf_eps;
    float *x_in, *h1, *h2, *out, *d1, *d2, *dpre;
    float* slabs;                       /* [splits][n_params] */
    int splits;
    float *grad, *exp_avg, *exp_avg_sq;
    const double* lr;
    double weight_decay;
    int clip_mode;
    double clip_value;
    void* opt_workspace;                /* sb200_optim_workspace_bytes(): holds the Adam step count */
    float* norm_out;                    /* optional: global gradient norm of the last step */
    int mode;
    const float* actions; int64_t lda;
    const float* adv;
    const float* behave_pd; int64_t ldb;
    const float* ref_pd; int64_t ldr;
    const float* returns;
    const double* hyper;                /* device: [clip_epsilon, beta] */
    double eta, kl_target, stop_threshold;
    float* stats;
    int* stop_flag;
    int epochs;
    void* workspace;                    /* unused (kept for layout) */
    int grid;
    int cta_shift;
    const sb200_par* par;
} sb200_epochs;
/* `policy` (mode 0 / 1) and `value` (mode 2, may be NULL) in one launch; `workspace` must hold
 * sb200_ppo_epochs2_workspace_bytes() bytes, 256-byte aligned, zero-initialised once.  Data-parallel: the two blocks must use
 * DIFFERENT sb200_par channels (both exchange in the same phase). */
int sb200_ppo_epochs2_supported(const sb200_epochs* policy, const sb200_epochs* value);
size_t sb200_ppo_epochs2_workspace_bytes(const sb200_epochs* policy, const sb200_epochs* value);
/* the launch plan: {grid, squared-norm chunks, s, rows per split (policy), s, rows per split (value; 0 without one)}.
 * `grid` caps the launch below one CTA per SM; everything else is sized for one CTA per SM, so results do not depend on it. */
int sb200_ppo_epochs2_plan(const sb200_epochs* policy, const sb200_epochs* value, int* out6);
int sb200_ppo_epochs2_f32(const sb200_epochs* policy, const sb200_epochs* value, void* workspace, void* stream);
/* accumulated clock64 cycles per phase of the launches on `workspace` (2 x 16: CTA 0, last CTA; see epoch2.cu) */
int sb200_ppo_epochs2_profile(void* workspace, uint64_t* out32, int reset, void* stream);
int sb200_ppo_epochs2_cta_profile(void* workspace, uint64_t* out_192x8, void* stream);

/* ---------------------------------------------------------------------------------------------
 * LSTM stem of RNN-mode PPO (csrc/lstm.cu; nn.LSTM(batch_first=True) of ppo_net.py:143-152,277-279,342-351; BPTT over
 * eff_len = n_step - horizon + 1 steps, ppo.py:389-406,507-525).  Gate order i, f, g, o; WhhT = [H][4H].
 *   rows_zfilter: out[b*L + t][0..D) = zfilter(x[b*batch_stride + t*row_stride + 0..D)) (plain gather if zf_stats NULL).
 *   lstm_forward: pre_x [B*L][4H] = x W_ih^T + b_ih (an MLP-kernel call); h0 / c0 row b at element b*ld_cells (NULL: zeros);
 *     h_out [B*L][ldh]; optional saves for the backward pass: h_prev (h_{t-1}, [B*L][ldh]), gates (post-activation), c_seq; optional
 *     final cells h_last / c_last [B][H].
 *   lstm_backward: dh_out [B*L][ldd] (gradient w.r.t. h_t) -> dpre [B*L][4H] (w.r.t. the gate pre-activations); the
 *     weight gradients are then sb200_linear_bwd_dw_f32(x, dpre) and sb200_linear_bwd_dw_f32(h_prev, dpre). */
int sb200_rows_zfilter_f32(const float* x, int64_t row_stride, int64_t batch_stride, int B, int L, int D,
                           const float* zf_stats, double eps, float* out, int64_t ldo, void* stream);
int sb200_lstm_forward_f32(const float* pre_x, const float* WhhT, const float* b_hh, const float* h0, const float* c0,
                           int64_t ld_cells, int B, int L, int H, int ldh, float* h_out, float* h_prev, float* gates,
                           float* c_seq, float* h_last, float* c_last, void* stream);
int sb200_lstm_backward_f32(const float* dh_out, int64_t ldd, const float* gates, const float* c_seq, const float* c0,
                            int64_t ld_cells, const float* WhhT, int B, int L, int H, float* dpre, void* stream);

/* Kernel family of the wide layers of sb200_mlp_forward_f32: 1 (default) = tensor-core mma.sync TF32 with the 3xTF32
 * error-compensated split (fp32-level accuracy, ~1e-6 relative) for batches above 2048 rows, fp32 FFMA below (where
 * the FFMA kernel is faster: 19 us vs 26 us at 1024 rows); 0 = fp32 FFMA kernels everywhere.  Env SB200_MMA overrides
 * the initial value. */
int sb200_set_forward_mode(int mode);

/* Backward of one Linear layer (kernel layout), replacing torch autograd in ppo.py:242,347 and
 * ddpg.py:306,330.
 *   dx: dX[M,K] = (dY[M,N] . W^T), multiplied by relu'(x_act) when x_act != NULL (x_act = the layer's
 *       saved post-ReLU input, so dX is directly the previous layer's pre-activation gradient).
 *   dw: `splits` partial slabs, slab z covering rows [z*rps, (z+1)*rps): dW_slabs + z*slab_stride is a
 *       [K][ldw] matrix, db_slabs + z*slab_stride a [ldw] vector (db_slabs may be NULL).  The slabs are
 *       summed in fixed order by sb200_grad_reduce_norm_f32 (deterministic, no atomics). */
int sb200_linear_bwd_dx_f32(const float* dY, int64_t ldy, const float* W, int ldw, const float* x_act,
                            int64_t ld_xact, float* dX, int64_t lddx, int M, int N, int K, void* stream);
int sb200_linear_bwd_dw_f32(const float* X, int64_t ldx, const float* dY, int64_t ldy, float* dW_slabs,
                            float* db_slabs, int64_t slab_stride, int splits, int ldw, int M, int K, int N,
                            void* stream);
/* Backward of a LayerNorm that follows an activation (csrc/layernorm.cu).  dY [M][ldy]: gradient w.r.t. the LayerNorm
 * output (sb200_linear_bwd_dx_f32 of the next layer with x_act = NULL); h [M][ldh]: the saved activation before the
 * LayerNorm; stats [M][2]: the forward's (mean, rstd); g [N]: the gain.  With x^ = (h - mean) * rstd:
 *   dX = rstd * (g*dY - mean(g*dY) - x^ * mean(g*dY*x^)), times relu'(h) when relu != 0  ->  dX [M][lddx]
 *   dg_slabs + z*slab_stride / db_slabs + z*slab_stride  <-  sum over split z's rows of dY*x^ / dY (splits slabs of N
 *   floats, rows split as sb200_linear_bwd_dw_f32 does; reduce with sb200_grad_reduce_norm_f32).
 * dg_slabs = db_slabs = NULL: no parameter gradient (the slabs are not touched). */
int sb200_layernorm_bwd_f32(const float* dY, int64_t ldy, const float* h, int64_t ldh, const float* stats,
                            const float* g, int M, int N, int relu, float* dX, int64_t lddx, float* dg_slabs,
                            float* db_slabs, int64_t slab_stride, int splits, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Windowed GAE + n-step return (surreal/learner/ppo.py:372-374,387-418).
 *   rewards [B,n], values [B,n+1] (raw critic output; the (1-done) mask of ppo.py:387 is applied
 *   inside), dones [B,n].  horizon == n -> MLP branch (one output per window), horizon < n ->
 *   RNN branch (E = n-horizon+1 outputs per window).  adv/ret are [B,E].  norm_adv applies
 *   (adv-mean)/max(unbiased_std, 1e-4) over all B*E advantages.  rewards are multiplied by reward_scale
 *   (ppo.py:452) on load.
 *   workspace: sb200_gae_workspace_bytes() bytes, zero-initialised once by the caller. */
size_t sb200_gae_workspace_bytes(int B, int n, int horizon);
int sb200_gae_window_f32(const float* rewards, const float* values, const float* dones, int B, int n,
                         int horizon, double gamma, double lam, double reward_scale, int norm_adv, float* adv,
                         float* ret, void* workspace, void* stream);

/* pd[b] = [mean(A) | exp(log_var)(A) * exp(log_noise[b])]  (builders.py:127-129; per-actor noise of
 * ppo_agent.py:139 when log_noise != NULL). */
int sb200_make_pd_f32(const float* mean, int64_t ldm, const float* log_var, const float* log_noise, int B,
                      int A, float* pd, int64_t ldp, void* stream);
/* ZFilter.z_update (z_filter.py:44-57): stats = running_sum[D] | running_sumsq[D] | count[1], updated in place. */
int sb200_zfilter_update_f32(const float* x, int64_t ldx, int64_t rows, int D, float* stats, void* stream);

/* Global-batch statistics helpers for the data-parallel learner: moments3 = {sum, sum of squares, count} (fp64,
 * summed over ranks by the caller); normalize applies (x-mean)/max(unbiased std, floor) (ppo.py:413-416). */
int sb200_moments_f32(const float* x, int64_t n, double* moments3, void* stream);
int sb200_normalize_f32(float* x, int64_t n, const double* moments3, double floor_value, void* stream);
int sb200_add_f32(float* dst, const float* src, int64_t n, void* stream);
/* RewardFilter as called from ppo.py:452-456: out = forward(rewards*reward_scale) with the current statistics,
 * then update (running_sumsq is OVERWRITTEN, reward_filter.py:42).  stats = count | running_sum | running_sumsq. */
int sb200_reward_filter_f32(const float* rewards, int64_t n, double reward_scale, double eps, float* stats,
                            float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * PPO losses: forward + gradient in one pass (replaces surreal/learner/ppo.py:194-225, 250-285,
 * 311-332, 553-557, 568-575 and DiagGauss of surreal/model/ppo_net.py:29-72 with torch autograd).
 * stats[] is a device float array of SB200_STAT_COUNT slots. */
#define SB200_STAT_SURR 0            /* _surr_loss */
#define SB200_STAT_LOSS 1            /* _clip_surr_loss (clip) / _kl_loss_adapt (adapt) */
#define SB200_STAT_ENTROPY 2         /* _entropy */
#define SB200_STAT_KL_PRE 3          /* adapt: _pol_kl inside the loss (before the step) */
#define SB200_STAT_KL_POST 4         /* _pol_kl after the step (early-stop test, ppo.py:553-556) */
#define SB200_STAT_GRAD_NORM_ACTOR 5
#define SB200_STAT_VAL_LOSS 6
#define SB200_STAT_EXPLAINED_VAR 7
#define SB200_STAT_GRAD_NORM_CRITIC 8
#define SB200_STAT_RETURN_MEAN 9     /* _avg_return_targ */
#define SB200_STAT_LOG_SIG 10        /* _avg_log_sig */
#define SB200_STAT_BEHAVE_LIK 11     /* _avg_behave_likelihood */
#define SB200_STAT_IS_WEIGHT 12      /* _avg_is_weight */
#define SB200_STAT_REF_BEHAVE_KL 13  /* _ref_behave_diff */
#define SB200_STAT_EPOCHS 14         /* number of policy epochs executed this learn() */
#define SB200_STAT_VAL_MOMENTS 16    /* 8 slots: mean(ret-v), mean((ret-v)^2), mean(ret), mean(ret^2) as (hi, lo) float pairs */
#define SB200_STAT_COUNT 32

size_t sb200_ppo_loss_workspace_bytes(int B, int A);   /* zero-initialise once */
/* mode 0 = clip (hyper[0] = clip_epsilon), mode 1 = adapt (hyper[1] = beta; needs sb200_ppo_kl_f32(ref, learn)
 * to have run on the same workspace first).  mean: actor output after tanh [B,ldm]; dpre: gradient w.r.t.
 * the pre-tanh output [B,ldd] (padding columns zeroed); dlog_var [A].  hyper is a DEVICE array of doubles so
 * that publish-time adaptation (ppo.py:648-661) does not invalidate captured graphs.
 * stop_flag (may be NULL): when *stop_flag != 0 the kernel is a no-op (device-side KL early stop). */
int sb200_ppo_policy_loss_f32(int mode, const float* mean, int64_t ldm, const float* log_var,
                              const float* actions, int64_t lda, const float* adv, const float* behave_pd,
                              int64_t ldb, const float* ref_pd, int64_t ldr, int B, int A,
                              const double* hyper, double eta, double kl_target, float* dpre, int64_t ldd,
                              float* dlog_var, float* stats, void* workspace, const int* stop_flag, void* stream);
/* mean KL(p0 || (mean, exp(log_var))) -> stats[stat_slot] (slot < 0: none) and the workspace; raises *stop_flag
 * when the mean exceeds stop_threshold (> 0). */
int sb200_ppo_kl_f32(const float* p0, int64_t ld0, const float* mean, int64_t ldm, const float* log_var,
                     int B, int A, float* stats, int stat_slot, double stop_threshold, int* stop_flag,
                     int defer, void* workspace, void* stream);
/* Data-parallel split of the above: with defer != 0 sb200_ppo_kl_f32 only leaves the LOCAL mean KL as a double at
 * byte offset sb200_ppo_loss_kl_offset() of the workspace; the caller averages it over ranks (NCCL) and then
 * sb200_ppo_kl_apply publishes it to stats / raises the stop flag identically on every rank. */
int sb200_ppo_kl_apply(void* workspace, float* stats, int stat_slot, double stop_threshold, int* stop_flag,
                       void* stream);
size_t sb200_ppo_loss_kl_offset(void);
int sb200_value_loss_f32(const float* values, int64_t ldv, const float* returns, int B, float* dpre,
                         int64_t ldd, float* stats, void* workspace, void* stream);
int sb200_ppo_final_stats_f32(const float* mean, int64_t ldm, const float* log_var, const float* actions,
                              int64_t lda, const float* behave_pd, int64_t ldb, const float* ref_pd,
                              int64_t ldr, int B, int A, float* stats, void* workspace, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Optimiser over one flat parameter buffer (replaces clip_grad_norm_/clip_grad_value_ + torch.optim.Adam:
 * ppo.py:159-168,244-247,349-352; ddpg.py:145-165,309-310,332-333).
 *   grad_reduce_norm: grad[i] = scale * sum_z slabs[z*slab_stride + i] (fixed order); global L2 norm (and
 *                     step += 1 when bump_step) into the workspace.  Data-parallel learners call it twice around
 *                     the NCCL all-reduce: (slabs -> grad, scale 1, no bump), (grad -> grad, 1/world, bump).
 *   clip_adam: clip_mode 0 none / 1 global norm (clip_value = max_norm) / 2 by value; lr is a DEVICE double.
 *   workspace: sb200_optim_workspace_bytes(), zero-initialised once (it holds the Adam step count). */
size_t sb200_optim_workspace_bytes(void);
int sb200_grad_reduce_norm_f32(const float* slabs, int64_t slab_stride, int splits, float* grad, int64_t n,
                               double scale, int bump_step, void* workspace, const int* stop_flag, void* stream);
int sb200_clip_adam_f32(float* params, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                        const double* lr, double beta1, double beta2, double eps, double weight_decay,
                        int clip_mode, double clip_value, void* workspace, float* norm_out,
                        const int* stop_flag, void* stream);
/* target = target*(1-tau) + tau*src (soft target update, ddpg.py:410-418); a no-op when *stop_flag != 0. */
int sb200_soft_update_f32(float* target, const float* src, int64_t n, double tau, const int* stop_flag, void* stream);
/* Hard target update with PeriodicTracker(period).track_increment(incr) semantics on a device counter, so that several
 * learner updates and the copies among them fit in one CUDA graph: DDPG counts updates (ddpg.py:419-428, incr = 1),
 * DQN counts samples (dqn.py:84-86, incr = batch size).  tick != 0: *counter += incr first (pass it for the first
 * buffer of an update, 0 for the others sharing the counter); then target = src when the count crossed a multiple of
 * period in that increment.  Neither happens when *stop_flag != 0. */
int sb200_hard_update_f32(float* target, const float* src, int64_t n, int64_t* counter, int64_t period, int64_t incr,
                          int tick, const int* stop_flag, void* stream);

/* ---------------------------------------------------------------------------------------------
 * DDPG element-wise pieces (surreal/learner/ddpg.py:261-262,279,305,324-331,335-341); the networks run through
 * sb200_mlp_forward_f32 (critic: aux_layer = 1 for cat(h, action)) and the backward / optimiser entries above. */
#define SB200_DSTAT_ACTOR_LOSS 0
#define SB200_DSTAT_CRITIC_LOSS 1
#define SB200_DSTAT_ACTION_NORM 2
#define SB200_DSTAT_REWARDS 3
#define SB200_DSTAT_Q_TARGET 4
#define SB200_DSTAT_Q_POLICY 5
#define SB200_DSTAT_ACTION_ABSMAX 6   /* for the deferred `assert |a| <= 1` of ddpg.py:261-262 */
#define SB200_DSTAT_TD_ERROR 7        /* weighted critic loss only: mean |q - y| (the reference DQN's td_error) */
#define SB200_DSTAT_IS_WEIGHT 8       /* weighted critic loss only: mean importance weight */
/* byte offset inside the DDPG workspace of the int32 "bad action" flag: sb200_ddpg_target*_f32 set it to 1 unless
 * max|a| <= 1, so a NaN action raises it too (the reference asserts this BEFORE any update, ddpg.py:261-262); pass its
 * address as stop_flag to the optimiser / soft-update calls of the same learn() so an out-of-range batch leaves every
 * parameter untouched. */
size_t sb200_ddpg_bad_action_offset(void);
size_t sb200_ddpg_workspace_bytes(int B);
/* y = rewards + discount * q_next * (1 - dones), discount = gamma ** n_step. */
int sb200_ddpg_target_f32(const float* rewards, const float* q_next, int64_t ldq, const float* dones,
                          const float* actions, int64_t lda, int B, int A, double discount, float* y,
                          float* stats, void* workspace, void* stream);
/* MSE(q, y): dq = 2 (q - y) / B. */
int sb200_ddpg_critic_loss_f32(const float* q, int64_t ldq, const float* y, int B, float* dq, int64_t ldd,
                               float* stats, void* workspace, void* stream);
/* The critic loss of prioritized replay (dqn.py:148-168): mean(w (q - y)^2), dq = 2 w (q - y) / B, with importance
 * weights w [B]; stats also get TD_ERROR and IS_WEIGHT.  priorities [B] (or NULL): |q - y| + eps per row, the new
 * priorities of the sampled records.  With every w == 1 dq and the loss equal sb200_ddpg_critic_loss_f32's bit for bit. */
int sb200_ddpg_critic_loss_weighted_f32(const float* q, int64_t ldq, const float* y, int B, const float* weights,
                                        float* dq, int64_t ldd, float* priorities, double eps, float* stats,
                                        void* workspace, void* stream);
/* TD3 options (ddpg.py:267-283): target2 = ddpg_target with y = min(y, y2) over two target critics; smooth_action =
 * clamp(pi + clip(policy_noise * N(0,1), -noise_clip, noise_clip), -1, 1) (unit_noise [B][A] injected draws, or NULL
 * for Philox keyed by (seed, *step_counter, row)). */
int sb200_ddpg_target2_f32(const float* rewards, const float* q_next, int64_t ldq, const float* q_next2, int64_t ldq2,
                           const float* dones, const float* actions, int64_t lda, int B, int A, double discount,
                           float* y, float* stats, void* workspace, void* stream);
int sb200_ddpg_smooth_action_f32(const float* pi, int64_t ldp, const float* unit_noise, int B, int A,
                                 double policy_noise, double noise_clip, uint64_t seed, const uint64_t* step_counter,
                                 float* out, int64_t ldo, void* stream);
/* actor loss -mean(q_pi): seeds dq = -1/B for the backward pass through the critic. */
int sb200_ddpg_actor_seed_f32(const float* q_pi, int64_t ldq, int B, float* dq, int64_t ldd, float* stats,
                              void* workspace, void* stream);
/* dpre = dout * (1 - out^2). */
int sb200_tanh_bwd_f32(const float* dout, int64_t ldo, const float* out, int64_t ldy, int B, int A,
                       float* dpre, int64_t ldd, void* stream);

/* ---------------------------------------------------------------------------------------------
 * DQN (surreal/learner/dqn.py, agent/q_agent.py, model/q_net.py).  The Q towers run through sb200_mlp_forward_f32 /
 * the packed forward (one call per tower: the action tower [rows][n_actions], with dueling also the state tower
 * [rows][1]); these entries combine them, Q = (A - mean_j A) + V, or Q = A without a state tower.
 *
 * act: one warp per actor, argmax_j Q_j (first index among ties), then epsilon-greedy.  epsilon is
 *   schedule(*act_counter) when `schedule` is given -- the device array [t_0..t_{P-1} | v_0..v_{P-1} | outside] of a
 *   PiecewiseSchedule with P = n_points (utils/schedule.py:34-73; LinearSchedule is [(0, 1), (T, final)] with outside
 *   value final) -- else fixed_eps.  Philox4x32-10 keyed (seed, *act_counter, actor): u = x / 2^32 < epsilon explores
 *   with action floor(y * n_actions / 2^32).  Writes the action index as a float (the record's action field),
 *   optionally a one-hot row [N][ldo] (ldo >= n_actions, the tail zero) and the index as int64.  The caller advances
 *   *act_counter after the call (q_agent.py:45: T += 1 per act).
 * agent_act: QAgent.act in one call, for host and device observations: [H2D obs_host -> obs unless obs_host is NULL] ->
 *   the tower forwards (on the packed weights when adv_packed is given: both towers' packs, the per-step copy a rollout
 *   chunk packs once; else the fused forward) -> act -> [when action_host is not NULL: D2H of the int64 actions and ONE
 *   stream synchronisation].  With the host pointers NULL no copy to or from the host and no synchronisation is
 *   issued: the call is graph-capturable.  value_net / value_packed / value: the state tower, all NULL without dueling. */
#define SB200_DQN_MAX_ACTIONS 1024
int sb200_dqn_act_f32(const float* adv, int64_t lda, const float* value, int64_t ldv, int N, int n_actions,
                      const double* schedule, int n_points, double fixed_eps, uint64_t seed, const int64_t* act_counter,
                      float* action, float* one_hot, int64_t ldo, int64_t* action_i64, void* stream);
typedef struct {
    const sb200_mlp* adv_net;           /* action tower: D -> ... -> n_actions */
    const sb200_mlp* value_net;         /* state tower: D -> ... -> 1, or NULL */
    const float* adv_packed;            /* packed weights of both towers, or NULL: the fused forward */
    const float* value_packed;
    int N;
    const float* obs_host;              /* [N][D] pinned, or NULL: obs already holds this step's observations */
    float* obs;                         /* [N][ld_obs] */
    int64_t ld_obs;
    float* adv;                         /* [N][n_actions] */
    float* value;                       /* [N][1] or NULL */
    const double* schedule;             /* as in sb200_dqn_act_f32 */
    int n_points;
    double fixed_eps;
    uint64_t seed;
    const int64_t* act_counter;
    float* action;                      /* [N] action indices as floats */
    float* one_hot;                     /* [N][ldo] or NULL */
    int64_t ldo;
    int64_t* action_i64;                /* [N] or NULL; required with action_host */
    int64_t* action_host;               /* [N] pinned; NULL: no D2H and no synchronisation */
} sb200_dqn_agent_act;
int sb200_dqn_agent_act_f32(const sb200_dqn_agent_act* args, void* stream);
/* TD step of one update (dqn.py:44-69), one thread per row: q = Q(s)[a] from the online towers (q_a, q_v), the target
 * towers at s' (t_a, t_v) and, for double Q, the online towers at s' (o_a, o_v; NULL for max over the target row).
 * y = r + gamma (1 - done) q', td = q - y, loss = mean(w huber(td)) with the Huber of delta 1 (w = 1 when weights is
 * NULL).  Writes d_a / d_v, the gradients w.r.t. the towers' outputs (dQ_a = w clamp(td, -1, 1) / B; dueling:
 * dA_j = dQ_j - mean_k dQ_k, dV = sum_k dQ_k; padding columns zero), priorities[b] = |td| + priority_eps when given, the
 * SB200_QSTAT_* statistics as fixed-order sums, and the workspace's bad-action flag: 1 when some action is not an
 * integer in [0, n_actions) (such rows compute with action 0).  Pass the flag as stop_flag to the optimiser calls of the
 * update.  workspace: sb200_dqn_workspace_bytes(B), zero-initialised once. */
#define SB200_QSTAT_LOSS 0
#define SB200_QSTAT_TD_ERROR 1        /* mean |td| (dqn.py:87-90) */
#define SB200_QSTAT_Q 2               /* mean Q(s, a) */
#define SB200_QSTAT_IS_WEIGHT 3       /* mean importance weight (1 without weights) */
#define SB200_QSTAT_BAD_ROWS 4        /* rows whose action is out of range */
size_t sb200_dqn_workspace_bytes(int B);
size_t sb200_dqn_bad_action_offset(void);
int sb200_dqn_td_f32(const float* q_a, int64_t ld_qa, const float* q_v, int64_t ld_qv, const float* t_a, int64_t ld_ta,
                     const float* t_v, int64_t ld_tv, const float* o_a, int64_t ld_oa, const float* o_v, int64_t ld_ov,
                     const float* actions, const float* rewards, const float* dones, const float* weights, int B,
                     int n_actions, double gamma, double priority_eps, float* d_a, int64_t ld_da, float* d_v,
                     int64_t ld_dv, float* priorities, float* stats, void* workspace, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Experience staging of PPO: ExpSenderWrapperMultiStepMovingWindowWithInfo._step (exp_sender_wrapper.py:209-228) for N
 * actors + FIFOReplay.insert (fifo_replay.py:27,34-35).  Every entry that stages a step takes this one descriptor of the
 * buffers involved (all device memory, allocated once by the caller).
 *   Per actor a window deque in HBM: stage_pos [N] = items it holds, stage_obs [N][n+1][D], stage_act [N][n][A],
 *   stage_pd [N][n][2A], stage_rew / stage_done [N][n].  A window is complete at n items; completed windows are copied
 *   into FIFO slots in (step, actor) order, drop-oldest at capacity; then `stride` items are popped; done clears the deque.
 *   Record layout, in the deques and in the ring alike (n = n_step; r_*: C records, one array per field):
 *     obs [n+1][D] (row n = obs_next) | act [n][A] | pd [n][2A] (mean | std) | rew [n] | done [n]
 *   D = floats per observation row of a record (an RNN policy's rows also carry its cells, see sb200_window_rows).
 *   dest [N]: the current step's slot of each actor's window (slot | -1 not complete | -2 complete but dropped).
 *   fifo_state: sb200_fifo_state_bytes() bytes {int head,count,capacity,dropped; int64 total_in,total_out}.
 *   step_counter: the Philox step counter; the step's slot assignment advances it by one. */
typedef struct {
    int N, n_step, stride, D, A;
    int* stage_pos;
    float *stage_obs, *stage_act, *stage_pd, *stage_rew, *stage_done;
    int* dest;
    void* fifo_state;
    float *r_obs, *r_act, *r_pd, *r_rew, *r_done;
    uint64_t* step_counter;
} sb200_windows;
/* The rows one env step hands the window staging.  obs_next: each actor's true successor; obs_reset: what it observes
 * next (the reset observation where done); [N][obs_dim] each; reward / done [N].
 *   *_host: pinned host copies, all four or none.  With them the call first uploads them into the device rows
 *     (obs_next_host == obs_reset_host: one upload, into obs_reset, which then serves as both).
 *   layers > 0: an RNN policy, whose record rows are [obs (obs_dim) | h_0 .. h_{layers-1} | c_0 .. c_{layers-1}]
 *     (D = obs_dim + 2 * layers * H).  The successor row and the reset row are assembled from the env's rows and the
 *     agent's [layers][N][H] cells h / c as they are now, i.e. the cells it acts from on the next observation.  Rows whose
 *     two copies exceed 48 KB of shared memory (a pixel frame's words plus the cells) are committed by a kernel that reads
 *     the row words straight from the rows and cells instead of staging them; force_wide = 1 takes that kernel for any
 *     row width (same bytes written).  layers = 0: D = obs_dim, no cells.
 *   slots_assigned: sb200_ppo_sample_f32 (assign_slots = 1) has already assigned this step's slots. */
typedef struct {
    float *obs_next, *obs_reset, *reward, *done;
    const float *obs_next_host, *obs_reset_host, *reward_host, *done_host;
    int obs_dim;
    int layers, H;
    const float *h, *c;
    int slots_assigned, force_wide;
} sb200_window_rows;
/* ppo_window_step: [H2D of the host rows] -> slot assignment of the windows this step completes (unless slots_assigned;
 * advances fifo_state and *step_counter) -> commit of the step into the deques and of the completed windows into the
 * ring.  1 or 2 kernels. */
int sb200_ppo_window_step_f32(const sb200_windows* windows, const sb200_window_rows* rows, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Batched actors (one call serves all N co-located actors of a step).
 *   ppo_sample: PPOAgent.act after the network (surreal/agent/ppo_agent.py:138-149): pd = [mean | exp(log_var)*
 *     exp(log_noise_i)], action = clip(eps*std+mean, -1, 1).  eps [N,A] injected N(0,1) draws or NULL for
 *     Philox4x32-10 keyed by (seed, *step_counter, actor).  With `stage` (sb200_windows; NULL: not staged) the step's
 *     action / pd rows are also written to each actor's window deque.  assign_slots = 1 (needs `stage`, and
 *     step_counter == stage->step_counter) fuses the slot assignment of the windows this step completes (it depends only
 *     on the deque lengths, so it can precede the env step): the same launch writes stage->dest, advances fifo_state and
 *     *step_counter (+1, after every block has drawn with the old value).  Follow with ppo_window_step
 *     (slots_assigned = 1) or env_step with `windows`.
 *   ddpg_noise: DDPGAgent.act after the network (ddpg_agent.py:176-183): clip -> + sigma_i*N(0,1) -> clip. */
int sb200_ppo_sample_f32(const float* mean, int64_t ldm, const float* log_var, const float* log_noise,
                         const float* eps, int N, int A, int deterministic, uint64_t seed, uint64_t* step_counter,
                         float* action, float* pd, const sb200_windows* stage, int assign_slots, void* stream);

/* Categorical policy of PPO for discrete action spaces (csrc/ppo_cat.cu; semantics: tests/cat_ref.py).  The actor head
 * outputs K logits (no tanh, no log_var).  pd row = [p_0..p_{K-1} | log p_0..log p_{K-1}] (2K floats) from a
 * max-subtracted log-softmax; actions are one-hot rows [K]: the window records keep their [A] / [2A] layout with A = K.
 * likelihood(a) = max(p_a, 1e-5), KL(p0 || p1) = sum p0 (log p0 - log p1), entropy = -sum p log p.  One warp per row.
 * K: 2 .. SB200_PPO_CAT_MAX_K, the widest layer the fused forward accepts (sb200_mlp_forward_f32).
 *   cat_sample: logits [N][ldl] -> pd [N][2K], one-hot action [N][K], index [N] int64 (or NULL).  Inverse CDF of one
 *     uniform per actor, u = (x >> 8) * 2^-24 with x the first word of Philox4x32-10 keyed (seed, *step_counter,
 *     actor << 16) as ppo_sample keys its normals: the action is the first j with u < c_j, c_j the fp32 running sum of
 *     p_0..p_j, or K - 1 if none.  deterministic: the argmax of the logits (lowest index among ties).  stage /
 *     assign_slots exactly as sb200_ppo_sample_f32 (stage->A == K).
 *   cat_make_pd: logits [B][ldl] -> pd [B][ldp].
 *   cat_policy_loss: the clip (mode 0) or adapt (mode 1) loss of sb200_ppo_policy_loss_f32 with the categorical
 *     likelihoods; dlogits [B][ldd] = gradient w.r.t. the logits (padding columns zeroed); the same stats slots
 *     (ENTROPY = mean entropy of the current policy) and stop_flag no-op.  Adapt needs sb200_ppo_cat_kl_f32(ref, learn)
 *     on the same workspace first.
 *   cat_kl: mean KL(p0 || softmax(logits)) -> stats[stat_slot] and the workspace; raises *stop_flag above stop_threshold.
 *   cat_final_stats: BEHAVE_LIK, IS_WEIGHT and REF_BEHAVE_KL of sb200_ppo_final_stats_f32 (no LOG_SIG).
 * workspace: sb200_ppo_loss_workspace_bytes(B, K). */
#define SB200_PPO_CAT_MAX_K 4096
int sb200_ppo_cat_sample_f32(const float* logits, int64_t ldl, int N, int K, int deterministic, uint64_t seed,
                             uint64_t* step_counter, float* action, float* pd, int64_t* index, const sb200_windows* stage,
                             int assign_slots, void* stream);
int sb200_ppo_cat_make_pd_f32(const float* logits, int64_t ldl, int B, int K, float* pd, int64_t ldp, void* stream);
int sb200_ppo_cat_policy_loss_f32(int mode, const float* logits, int64_t ldl, const float* actions, int64_t lda,
                                  const float* adv, const float* behave_pd, int64_t ldb, const float* ref_pd, int64_t ldr,
                                  int B, int K, const double* hyper, double eta, double kl_target, float* dlogits,
                                  int64_t ldd, float* stats, void* workspace, const int* stop_flag, void* stream);
int sb200_ppo_cat_kl_f32(const float* p0, int64_t ld0, const float* logits, int64_t ldl, int B, int K, float* stats,
                         int stat_slot, double stop_threshold, int* stop_flag, void* workspace, void* stream);
int sb200_ppo_cat_final_stats_f32(const float* logits, int64_t ldl, const float* actions, int64_t lda,
                                  const float* behave_pd, int64_t ldb, const float* ref_pd, int64_t ldr, int B, int K,
                                  float* stats, void* workspace, void* stream);
int sb200_ddpg_noise_f32(const float* mean, int64_t ldm, const float* sigma, const float* unit_noise, int N,
                         int A, int deterministic, uint64_t seed, const uint64_t* step_counter,
                         float* action, void* stream);
/*   ddpg_ou_noise: the same with Ornstein-Uhlenbeck exploration (surreal/agent/action_noise.py:22-39): ou_state [N][A]
 *     float64 is advanced in place, x <- x + theta*(0 - x)*dt + sigma_i*sqrt(dt)*N(0,1); sigma [N] float64.  The caller
 *     zeroes ou_state at episode start (DDPGAgent.pre_episode, ddpg_agent.py:205-208). */
int sb200_ddpg_ou_noise_f32(const float* mean, int64_t ldm, const double* sigma, const float* unit_noise, int N, int A,
                            int deterministic, uint64_t seed, const uint64_t* step_counter, double theta, double dt,
                            double* ou_state, float* action, void* stream);
/* ---------------------------------------------------------------------------------------------
 * Device-resident envs (csrc/env.cu): all N actors advance in one step call at fixed addresses (CUDA-graph capturable),
 * and done actors auto-reset inside it.  One descriptor per env, filled once by its owner; `kind` selects the task:
 *   SB200_ENV_SYNTH: the synthetic env of the benchmark configs (SURVEY §8d): s' = tanh(Ws s + Wa a) + 0.01 xi,
 *     r = -|s|^2/D + 0.1 xi', done at max_steps (MaxStepWrapper, env/wrapper.py:142-163); a done actor's state is
 *     re-drawn ~ N(0,1).  state [N][D] = what the agent observes next (obs NULL).  WsT [D][D] / WaT [A][D]: Ws / Wa
 *     transposed (k-major, WsT[k][d] = Ws[d][k]).  Noise keyed by (seed, *step_counter, actor).
 *   SB200_ENV_SYNTH_PIXEL: the synthetic PIXEL env (SURVEY §8d cfg 4): every step each actor observes a fresh uint8 frame
 *     of uniform random bytes; reward -mean(a^2) + 0.1 N(0,1); done at max_steps.  D = the frame's 32-bit words (frame
 *     bytes / 4, a multiple of 4); state / obs_next [N][D] words hold the frames (obs NULL).  Keyed like SYNTH.
 *   SB200_ENV_CARTPOLE, SB200_ENV_PENDULUM: classic-control tasks (semantics: tests/classic_ref.py; no counterpart in the
 *     reference, which reaches them through gym), one thread per actor.  obs [N][D] = what each actor observes next;
 *     episode [N] = its episode index; done = terminal or ep_step reaching max_steps (<= 0: no cap).  A done actor starts
 *     episode index + 1 in the same launch, its state drawn from Philox4x32-10 keyed (seed ^ const, episode index, actor).
 *     step_counter is not read.
 *     CARTPOLE: CartPole-v1.  state = obs = (x, x_dot, theta, theta_dot) [N][4]; action one-hot rows [N][2] (index 1,
 *       i.e. a[1] > a[0], pushes right); reward 1; terminal when |x| > 2.4 or |theta| > 12 deg (strict, against the fp32
 *       thresholds).  Registered episode limit 500.
 *     PENDULUM: Pendulum-v1.  state (theta, theta_dot) [N][2], obs (cos, sin, theta_dot) [N][3]; action [N][1] clipped
 *       to [-1, 1] and scaled to the torque 2a; never terminal.  Registered episode limit 200.
 * Every kind: action [N][A]; ep_step [N] = steps of each actor's episode; obs_next = the true successor (terminal where
 * done); reward [N]; done [N] (0 / 1).
 *   env_step: one step.  With `windows` (NULL: none) the step is fused with the commit half of ppo_window_step (`windows`,
 *     whose dest ppo_sample has assigned; its N / D / A must be the env's): the successor rows are staged straight from
 *     shared memory.  1 launch; the pixel env: 2, and no fused commit (SB200_ERR_UNSUPPORTED with `windows`).
 *   env_reset: the classic kinds only: every actor to episode 0, ep_step 0; state and obs drawn.  (The synthetic envs
 *     reset from the host.) */
#define SB200_ENV_SYNTH 0
#define SB200_ENV_SYNTH_PIXEL 1
#define SB200_ENV_CARTPOLE 2
#define SB200_ENV_PENDULUM 3
typedef struct {
    int kind;                           /* SB200_ENV_* */
    int N, D, A;
    int max_steps;
    uint64_t seed;                      /* the key the kernels draw with */
    void* state;                        /* fp32 rows, or the pixel env's frames */
    float* obs;                         /* classic kinds; NULL where the observation is the state */
    const float* WsT;                   /* SB200_ENV_SYNTH only */
    const float* WaT;
    int* ep_step;
    int* episode;                       /* classic kinds only */
    const uint64_t* step_counter;       /* the agents' Philox step counter */
    void* obs_next;
    float* reward;
    float* done;
} sb200_env;
int sb200_env_step_f32(const sb200_env* env, const float* action, const sb200_windows* windows, void* stream);
int sb200_env_reset_f32(const sb200_env* env, void* stream);

/* ---------------------------------------------------------------------------------------------
 * DDPG parameter-space exploration noise (surreal/agent/param_noise.py:9-74, ddpg_agent.py:136-153,174-175): every
 * actor acts with its own perturbed copy of the policy.  Images are [N][actor_stride] floats, each in the layout of
 * the actor's flat buffer (FlatNet), actor_stride = flat size rounded up to 32 floats (128 B); padding stays zero.
 * Adaptive mode keeps a device act counter (AdaptiveNormalParameterNoise.i) and per-actor distances dist[N]. */
typedef struct {
    uint64_t acts;          /* acts since the last apply (param_noise.py:38,47,60) */
    uint32_t ticket;        /* last-CTA ticket of the launches below; 0 between launches */
    uint32_t pad;
} sb200_param_noise_state;
/* param_noise_apply: NormalParameterNoise.apply / AdaptiveNormalParameterNoise.apply (param_noise.py:14-24,49-71) on the
 *   unperturbed flat actor `net`: image_k = fl32((double)W + sigma[k] * z), z ~ N(0,1) in float64, from `unit_noise`
 *   ([N][actor_stride] float64, tests) or Philox4x32-10 + double Box-Muller keyed by (seed, fetch_index, actor, offset).
 *   When `state` != NULL (adaptive) the same launch first updates sigma[k] in float64 from dist[k] / state->acts (float32)
 *   against target_stddev, skipped when acts == 0, then resets acts to 0.  No host synchronisation. */
int sb200_ddpg_param_noise_apply_f32(const sb200_mlp* net, int N, float* images, int64_t actor_stride, double* sigma,
                                     const double* unit_noise, uint64_t seed, uint64_t fetch_index, const float* dist,
                                     sb200_param_noise_state* state, double alpha, double target_stddev, void* stream);
/* Per-actor forward (ddpg_agent.py:173, csrc/mlp_fwd_per_actor.cu): out[k] = net_k(x[k]) where net_k is `net` (the
 *   descriptor of image 0) shifted by k * actor_stride floats (0: every row uses the same weights).  fp32, fixed-order
 *   sums: bit-identical from run to run.  When `state` != NULL the launch counts one act (state->acts += 1), and when also
 *   `shared` != NULL (the unperturbed actor, same layout) and state->acts % dist_interval == 0 on entry it writes
 *   dist[k] = |pi_shared(x[k]) - pi_k(x[k])|_2 (compute_action_distance, param_noise.py:42-47).  The counter is read on
 *   the device, so the call can be captured in a graph.  No aux input; SB200_ERR_UNSUPPORTED above 48 KB of shared memory. */
int sb200_mlp_forward_per_actor_f32(const sb200_mlp* net, int64_t actor_stride, const float* x, int64_t ldx, int N,
                                    float* out, int64_t ld_out, const sb200_mlp* shared, float* dist, int dist_interval,
                                    sb200_param_noise_state* state, void* stream);
/* DDPGAgent.act (ddpg_agent.py:155-184) in one call, for host and device observations: [H2D obs_host -> obs unless
 *   obs_host is NULL] -> actor forward -> ddpg_ou_noise (when ou_state != NULL, with sigma64) or ddpg_noise (with sigma)
 *   -> [when action_host is not NULL: D2H action and ONE stream synchronisation].  With the host pointers NULL no copy to
 *   or from the host and no synchronisation is issued: the call is graph-capturable.  The forward is chosen explicitly,
 *   because a per-actor forward with actor_stride 0 and no state (normal parameter noise before the first fetch) has the
 *   same arguments as the fused one:
 *     SB200_DDPG_FWD_FUSED: sb200_mlp_forward_f32 of `net`;
 *     SB200_DDPG_FWD_PACKED: sb200_mlp_forward_packed_f32 of `net` on `packed` (the per-step copy a rollout chunk packs);
 *     SB200_DDPG_FWD_PER_ACTOR: sb200_mlp_forward_per_actor_f32 with `net` the descriptor of image 0, actor_stride,
 *       shared, dist, dist_interval and pn_state.
 *   unit_noise: injected N(0,1) draws [N][A] or NULL (Philox).  2 kernels below 2048 actors. */
#define SB200_DDPG_FWD_FUSED 0
#define SB200_DDPG_FWD_PACKED 1
#define SB200_DDPG_FWD_PER_ACTOR 2
typedef struct {
    int forward;                        /* SB200_DDPG_FWD_* */
    const sb200_mlp* net;               /* actor: D -> ... -> A */
    const float* packed;                /* SB200_DDPG_FWD_PACKED only */
    int64_t actor_stride;               /* SB200_DDPG_FWD_PER_ACTOR only, as in sb200_mlp_forward_per_actor_f32 */
    const sb200_mlp* shared;
    float* dist;
    int dist_interval;
    sb200_param_noise_state* pn_state;
    int N;
    const float* obs_host;              /* [N][D] pinned, or NULL: obs already holds this step's observations */
    float* obs;                         /* [N][ld_obs] */
    int64_t ld_obs;
    float* mean;                        /* [N][A] actor output */
    const float* sigma;                 /* [N] float32: normal noise */
    const double* sigma64;              /* [N] float64: OU noise */
    const float* unit_noise;
    int deterministic;
    uint64_t seed;
    const uint64_t* step_counter;
    double theta, dt;                   /* OU noise only */
    double* ou_state;                   /* [N][A] float64, or NULL: normal noise */
    float* action;                      /* [N][A] */
    float* action_host;                 /* pinned; NULL: no D2H and no synchronisation */
} sb200_ddpg_act;
int sb200_ddpg_act_f32(const sb200_ddpg_act* args, void* stream);

/* PPOAgent.act (ppo_net.py:268-279,317-351,368-375, ppo_agent.py:133-149) in one call, for host and device observations
 * and every policy form:
 *   layers = 0, no frames: the MLP policy.  The head reads the observation rows with the z-filter fused into its forward
 *     (on head_packed, the per-step copy a rollout chunk packs once, when given).
 *   layers = 0, frames: the CNN policy: the CNN stem stage below into xf, then the head on xf.
 *   layers >= 1: the LSTM policy: h, c copied to h_before, c_before (the step's onetime_infos) -> rows_zfilter of the
 *     observations into xf (or the CNN stem stage with frames) -> per layer k: input projection (mlp_forward of ih[k] into
 *     pre_x) and lstm_forward from layer k's cells, updated in place -> head on the last layer's output.
 *   Every form: [H2D obs_host -> obs or frames_host -> frames first, unless NULL] -> ... -> ppo_sample (with `stage` and
 *   assign_slots) -> [when action_host is not NULL: D2H action / pd, and h_before / c_before when h_before_host is not
 *   NULL, then ONE stream synchronisation].  Cells are [layers][N][H] (h_before_host / c_before_host receive that layout).
 *   Layer k writes h_out[(layers-1-k) % 2].  Kernels while every forward stays below 2048 rows (one kernel each): 2 for
 *   the MLP policy, 5 for the CNN policy, 2 * layers + 3 for the LSTM policy, 2 more with frames (the stem's 3 in place
 *   of the z-filter).  With the host pointers NULL no copy to or from the host and no synchronisation is issued: the
 *   call is graph-capturable. */
#define SB200_MAX_RNN_LAYERS 8
typedef struct {
    const sb200_mlp* head;              /* actor head: D (layers = 0) or H -> ... -> A */
    const float* head_packed;           /* packed head weights (MLP policy only), or NULL: the fused forward */
    sb200_zfilter zf;                   /* z-filter of the observation rows */
    const sb200_mlp* ih[SB200_MAX_RNN_LAYERS];  /* input projection of layer k: in -> 4H (W_ih^T, b_ih) */
    const float* whh[SB200_MAX_RNN_LAYERS];     /* W_hh^T [H][4H] of layer k */
    const float* bhh[SB200_MAX_RNN_LAYERS];     /* b_hh [4H] of layer k */
    int layers, N, D, H;
    const float* obs_host;              /* [N][D] pinned, or NULL: obs already holds this step's observations */
    float* obs;                         /* [N][ld_obs] */
    int64_t ld_obs;
    float* xf;                          /* [N][ld_xf] z-filtered rows or stem features (not read by the MLP policy) */
    int64_t ld_xf;
    float* pre_x;                       /* [N][4H] */
    float* h_out[2];                    /* [N][ldh] each; h_out[1] only for layers > 1 */
    int ldh;
    float* h;                           /* [layers][N][H] cells, updated in place */
    float* c;
    float* h_before;                    /* [layers][N][H] cells before the step */
    float* c_before;
    float* mean;                        /* [N][A] head output */
    const float* log_var;
    const float* log_noise;
    const float* eps;                   /* injected N(0,1) draws [N][A] or NULL (Philox) */
    int deterministic;
    uint64_t seed;
    uint64_t* step_counter;
    float* action;
    float* pd;
    const sb200_windows* stage;         /* window staging of this step (NULL: not staged), see ppo_sample */
    int assign_slots;
    float* action_host;                 /* pinned; NULL: no D2H and no synchronisation */
    float* pd_host;
    float* h_before_host;               /* pinned; NULL: the cells stay on the device */
    float* c_before_host;
    /* Optional CNN stem stage (pixel input, ppo_net.py:268-279): with frames != NULL the first layer (or the head) reads
     * the stem's features instead of the observations (obs and zf are not read):  [H2D frames_host -> frames unless
     * NULL] -> conv_forward(1) of frames / 255 -> conv_forward(2) -> fc (Linear + ReLU) into xf [N][ld_xf], D = fc's
     * output width. */
    const uint8_t* frames_host;         /* [N][frame_c][frame_h][frame_w] pinned, or NULL: frames already hold this step's */
    uint8_t* frames;                    /* [N][frame_c][frame_h][frame_w] uint8 on the device, or NULL */
    int frame_c, frame_h, frame_w;
    const float* conv_w1;               /* conv1 k8 s4 -> 16 channels, kernel layout (csrc/stem.cu) */
    const float* conv_b1;
    const float* conv_w2;               /* conv2 k4 s2 -> 32 channels */
    const float* conv_b2;
    const sb200_mlp* fc;                /* the stem's Linear + ReLU: 32 * H2 * W2 -> D */
    float* a1;                          /* [N][16][H1][W1] */
    float* a2;                          /* [N][32 * H2 * W2] */
    /* SB200_PD_GAUSSIAN (0): ppo_sample.  SB200_PD_CATEGORICAL: the head outputs K logits into mean [N][K] and the last
     * stage is sb200_ppo_cat_sample_f32 (action: one-hot rows [N][K], pd [N][2K]; log_var, log_noise and eps are not
     * read). */
    int pd_type;
} sb200_ppo_act;
#define SB200_PD_GAUSSIAN 0
#define SB200_PD_CATEGORICAL 1
int sb200_ppo_act_f32(const sb200_ppo_act* args, void* stream);

/* Persistent rollout: T steps of policy forward -> sample -> synthetic env step -> window staging for ALL N
 * actors in ONE launch (a 4-CTA cluster owns 32 actors for the whole chunk; the policy weights stay resident in
 * shared memory, layer outputs cross CTAs through distributed shared memory).  Replaces T x (ppo_sample with
 * assign_slots + env_step with `windows` + the policy forward), i.e. the actor main loop of surreal/agent/base.py:224-271
 * for the synthetic env (`env`).  Same sampling / env arithmetic and Philox keys as the per-step entries.
 *   The kernel stages into the window deques of `windows` (whose N / D / A must match) and reads its step counter.
 *   Completed windows are written to a per-actor OUTBOX (o_*: [N*W] records in the record layout of sb200_windows,
 *   ev_step [N*W] = chunk-relative completion step, ev_count [N]); W >= T / stride + 2.
 *   rollout_commit then assigns FIFO slots in the reference's (step, actor) arrival order, copies the windows into
 *   the ring of `windows`, advances its fifo_state and *step_counter (+T).  scratch: sb200_ppo_rollout_scratch_ints()
 *   ints.
 *   rollout_supported: 1 when `net` (2 hidden layers whose widths are multiples of 16, head <= 32, D % 4 == 0,
 *   D <= 128) fits the shared-memory plan; otherwise use the per-step entries. */
typedef struct {
    const sb200_mlp* net;               /* policy: D -> H1 -> H2 -> A */
    const float* zf_stats;              /* NULL: no z-filter */
    float zf_eps;
    const float* log_var;               /* [A] */
    const float* log_noise;             /* [N] or NULL */
    uint64_t agent_seed;
    int deterministic;
    const sb200_env* env;               /* SB200_ENV_SYNTH, with the rollout's N / D / A; stepped in place */
    float* action;                      /* outputs of the LAST step, like the per-step entries leave them */
    float* pd;
    const sb200_windows* windows;       /* window staging and FIFO ring (not read by rollout_footprint) */
    float* o_obs;                       /* outbox */
    float* o_act;
    float* o_pd;
    float* o_rew;
    float* o_done;
    int* ev_step;
    int* ev_count;
    int W;
    int N, D, A, T;
} sb200_ppo_rollout;
int sb200_ppo_rollout_supported(const sb200_mlp* net, int D, int A);
size_t sb200_ppo_rollout_scratch_ints(int N, int W, int T);
int sb200_ppo_rollout_f32(const sb200_ppo_rollout* args, void* stream);
/* SMs that sb200_ppo_rollout_f32 with these net / N / D / A holds for the whole chunk when all its CTAs are resident at
 * once (one wave, one CTA per SM) -> *sms; 0 when the chunk runs in several waves or residency is not known. */
int sb200_ppo_rollout_footprint(const sb200_ppo_rollout* args, int* sms);
int sb200_ppo_rollout_commit_f32(const sb200_ppo_rollout* args, int* scratch, void* stream);

/* Persistent rollout of the recurrent policy (csrc/rollout_rnn.cu): T steps of z-filter -> LSTM layers -> actor head ->
 * sampling -> synthetic env step -> window staging for ALL N actors in ONE launch.  Replaces T x (sb200_ppo_act_f32
 * with `stage` and assign_slots + sb200_env_step_f32 + sb200_ppo_window_step_f32 with the cells), i.e. the actor
 * main loop of surreal/agent/base.py:224-271 with the LSTM policy of ppo_net.py:317-351 and ppo_agent.py:84-93,133-154,
 * for the synthetic env.  A CTA owns 8 actors; their
 * env state and [L][H] cells stay in shared memory for the whole chunk.  Same records, Philox keys and FIFO order as
 * that chain: the action noise of step t is keyed by *step_counter + t, the env noise by *step_counter + t + 1.
 *   base: a filled sb200_ppo_rollout for the env, sampling, outbox and windows; base->net is the actor head
 *     (H -> ... -> A), base->D the env's observation width; the window records are base->D + 2 * layers * H wide
 *     ([obs | h_0 .. h_{L-1} | c_0 .. c_{L-1}], utils.rnn_cell_layout).  Commit with sb200_ppo_rollout_commit_f32 on a
 *     copy of `base` whose D is the record width.
 *   ih / whh / bhh / layers / H / h / c / h_before / c_before: as in sb200_ppo_act.  The cells are read at entry and
 *     written back at exit; h_before / c_before receive the cells before the chunk's last step.
 *   Each staged row carries the cells the actor acts from on that row's observation (the successor row and, after done,
 *   the reset row alike: the cells carry over across episodes).
 *   rollout_rnn_supported: 1 when the shapes fit the kernel, from the shapes alone (no device needed): 1 ..
 *     SB200_MAX_RNN_LAYERS layers, H <= 128, D <= 256, a head of 1 .. SB200_MAX_LAYERS layers each <= 512 wide,
 *     A <= 32, each ih[k] one Linear (in -> 4H, no activation), no LayerNorm, no aux input; else 0, and rollout_rnn_f32 /
 *     rollout_rnn_footprint return SB200_ERR_UNSUPPORTED: use the per-step entries.
 *   rollout_rnn_footprint: SMs the chunk holds from start to end when its grid is at most one CTA per SM (one wave);
 *     0 otherwise. */
typedef struct sb200_ppo_rollout_rnn {
    const sb200_ppo_rollout* base;
    const sb200_mlp* ih[SB200_MAX_RNN_LAYERS];  /* input projection of layer k: in -> 4H (W_ih^T, b_ih) */
    const float* whh[SB200_MAX_RNN_LAYERS];     /* W_hh^T [H][4H] of layer k */
    const float* bhh[SB200_MAX_RNN_LAYERS];     /* b_hh [4H] of layer k */
    int layers, H;
    float* h;                           /* [layers][N][H] cells, updated in place */
    float* c;
    float* h_before;                    /* [layers][N][H] cells before the last step */
    float* c_before;
} sb200_ppo_rollout_rnn;
int sb200_ppo_rollout_rnn_supported(const sb200_ppo_rollout_rnn* args);
int sb200_ppo_rollout_rnn_f32(const sb200_ppo_rollout_rnn* args, void* stream);
int sb200_ppo_rollout_rnn_footprint(const sb200_ppo_rollout_rnn* args, int* sms);

/* ---------------------------------------------------------------------------------------------
 * HBM replay (the PPO window staging that fills the FIFO ring is sb200_windows above).
 *   fifo_pop: FIFOReplay.sample (fifo_replay.py:37-39): slot ids of the `batch` oldest windows; *status = 1
 *     if fewer are queued.   fifo_push: host-side Replay.insert() of k windows -> their slot ids.
 *   replay_gather: out[b] = src[idx[b]] for records of record_floats floats (idx32 or idx64 non-NULL). */
size_t sb200_fifo_state_bytes(void);
int sb200_fifo_pop(void* fifo_state, int batch, int* idx, int* status, void* stream);
int sb200_fifo_push(void* fifo_state, int k, int* slots, void* stream);
int sb200_replay_gather_f32(const float* src, int64_t record_floats, const int* idx32, const int64_t* idx64,
                            int batch, float* out, void* stream);
/* Every field of the sampled records in ONE launch (srcs / outs / record_floats are HOST arrays of nfields <= 8 entries):
 * outs[f][b] = srcs[f][idx[b]].  Replaces the per-key np.stack loops of aggregator.py:52-103,151-205. */
int sb200_replay_gather_multi_f32(const float* const* srcs, float* const* outs, const int64_t* record_floats,
                                  int nfields, const int* idx32, const int64_t* idx64, int batch, void* stream);
/* UniformReplay.sample (uniform_replay.py:43-47) on the device: `batch` i.i.d. draws WITH replacement over a sampling
 * view and the gather of every field of the drawn records (field arrays as in replay_gather_multi), in ONE launch with
 * no host input that depends on the ring's fill level -- so sample -> learn can be one CUDA graph.
 *   view (device): {int64 start, count, capacity}; draw r in [0, count) is ring slot (start + r) % capacity.
 *   sampler (device): sb200_uniform_sampler_bytes() bytes {uint64 draw_counter; int32 status; uint32 ticket}, zeroed
 *     once.  The launch advances draw_counter itself: replaying a captured graph draws fresh indices.
 *   Index stream: Philox4x32-10 call p, keyed (seed, draw_counter, p), serves draws 2p (words x:y) and 2p+1 (z:w); a
 *     draw is floor(u * count / 2^64) of its 64 bits u.  No rejection loop; bias <= count / 2^64 per index (< 2^-43 for
 *     a 2^20-slot ring).  NOT the reference's random.randint stream (that one is sb200_mt19937_randint_fill_h below).
 *   indices [batch]: the drawn ring slots.  count == 0: no ring access, outputs untouched, status = 1, counter kept.
 * uniform_view: the view between two chunks of inserts that excludes every slot the next `reserve` inserts can write:
 *   size + reserve <= capacity: {0, size}; else {(next_idx + reserve) % capacity, capacity - reserve}. */
size_t sb200_uniform_sampler_bytes(void);
int sb200_uniform_view(const void* uniform_state, int64_t reserve, int64_t* view, void* stream);
int sb200_uniform_sample_gather_f32(const float* const* srcs, float* const* outs, const int64_t* record_floats,
                                    int nfields, const int64_t* view, uint64_t seed, void* sampler, int batch,
                                    int64_t* indices, void* stream);
/* Prioritized replay (Schaul et al. 2016; the reference's prioritized_replay.py + segment_tree.py) over the uniform
 * ring: a sum tree and a min tree of p^alpha over the ring's slots, in device memory, and the entries that admit new
 * records, sample with importance weights and write new priorities, all capturable (no host read, fixed grids).
 *   Trees: `leaves` = capacity rounded up to a power of two (>= 2), heap order (node 1 is the root, node i has children
 *   2i and 2i+1, leaf j is node leaves + j).  leaf [leaves] fp32 p^alpha, 0 for a slot never inserted (and for slots
 *   >= capacity); sum [leaves] fp64 internal nodes, parent = left + right; mn [leaves] fp32 internal min nodes, where a 0
 *   leaf counts as +inf.  Internal nodes are rebuilt from their children, one CTA per `subtree` leaves (only subtrees
 *   flagged in dirty [leaves / subtree]), then the levels above, so tree values never depend on thread scheduling.
 *   owner [capacity]: int32 scratch of the priority update, all -1 at construction and after every update.
 *   ctrl: sb200_per_ctrl_bytes() bytes {int64 admitted; int64 updates; float max_priority; uint32 ticket}, zeroed with
 *   max_priority = 1.0 at construction.
 * per_tree_layout: `leaves` and `subtree` of a ring of `capacity` slots.
 * per_admit: every slot inserted since the last admit (total_in of the uniform state against ctrl.admitted, with wrap;
 *   all slots once the gap reaches capacity) gets max_priority^alpha, then the tree is rebuilt.  Call it before
 *   sb200_uniform_view.
 * per_rebuild: rebuild dirty subtrees (every subtree when full != 0) and the levels above.
 * per_sample_gather: as uniform_sample_gather (same view, Philox call/counter convention and empty-view rule), but draw
 *   k takes u = (64-bit word >> 11) * 2^-53 and mass = u * S, S the leaf sum over the view (split in two segments when it
 *   wraps), and descends the sum tree by prefix sum from the view's first slot (find_prefixsum_idx), clamped into the
 *   view.  weights [batch]: (leaf / min over the view)^(-beta), in fp64, with beta = beta_override when >= 0, else
 *   beta0 + min(updates / beta_anneal_iters, 1) (1 - beta0) (beta0 alone when beta_anneal_iters <= 0).  The launch
 *   advances the sampler's draw_counter and ctrl.updates.
 * per_update: leaf[indices[b]] = priorities[b]^alpha, the last b winning among equal indices, max_priority = max(it,
 *   priorities); then the rebuild.  Nothing happens while *stop_flag != 0 (stop_flag may be NULL). */
typedef struct sb200_per_tree {
    int64_t capacity;
    int64_t leaves;
    int64_t subtree;
    float* leaf;
    double* sum;
    float* mn;
    uint32_t* dirty;
    int32_t* owner;
    void* ctrl;
} sb200_per_tree;
size_t sb200_per_ctrl_bytes(void);
int sb200_per_tree_layout(int64_t capacity, int64_t* leaves, int64_t* subtree);
int sb200_per_admit(const sb200_per_tree* tree, const void* uniform_state, double alpha, void* stream);
int sb200_per_rebuild(const sb200_per_tree* tree, int full, void* stream);
int sb200_per_sample_gather_f32(const sb200_per_tree* tree, const float* const* srcs, float* const* outs,
                                const int64_t* record_floats, int nfields, const int64_t* view, uint64_t seed,
                                void* sampler, int batch, double beta0, double beta_anneal_iters, double beta_override,
                                int64_t* indices, float* weights, void* stream);
int sb200_per_update_f32(const sb200_per_tree* tree, const int64_t* indices, const float* priorities, int batch,
                         double alpha, const int* stop_flag, void* stream);
/* Experience staging of DDPG: ExpSenderWrapperSSARNStepBootstrap._step (exp_sender_wrapper.py:96-112) for N actors +
 * UniformReplay.insert (uniform_replay.py:36-41): k-th insert -> slot k % capacity, actor order.  One descriptor of the
 * buffers involved (device memory, allocated once by the caller), taken whole by both ssar_step entries.
 *   Per actor a deque of < n_step pending transitions: dq_len [N], dq_obs [N][n][D], dq_act [N][n][A], dq_rew [N][n]
 *   (float64 running n-step sums).  dest / emit [N]: the current step's ring slot and float32 reward of each actor's
 *   emitted record.  Ring r_*: obs / obs_next [C][D], act [C][A], rew / done [C].
 *   uniform_state: sb200_uniform_state_bytes() bytes {int64 next_idx,size,capacity,total_in}.
 *   step_counter: the Philox step counter, advanced by one per step.
 *   Rounding, as the reference's `e += pow(gamma, n_step - i - 1) * r` on Python floats: gamma^k is libm pow on the
 *   host, each step's product is rounded to float64, then the sum (no fused multiply-add); the record's reward is the
 *   sum rounded to float32 once, at emission.  1 <= n_step <= SB200_SSAR_MAX_NSTEP (the gamma^k table is a kernel
 *   argument); both ssar_step entries refuse a larger n_step with SB200_ERR_ARG before any launch. */
#define SB200_SSAR_MAX_NSTEP 64
typedef struct {
    int N, n_step;
    double gamma;
    int D, A;
    int* dq_len;
    float *dq_obs, *dq_act;
    double* dq_rew;
    int* dest;
    float* emit;
    void* uniform_state;
    float *r_obs, *r_obs_next, *r_act, *r_rew, *r_done;
    uint64_t* step_counter;
} sb200_ssar;
size_t sb200_uniform_state_bytes(void);
/*   ssar_step: one step of a device env: s_t = obs [N][D], a_t = action [N][A], obs_next / reward / done. */
int sb200_ssar_step_f32(const sb200_ssar* ssar, const float* obs, const float* action, const float* obs_next,
                        const float* reward, const float* done, void* stream);
/*   ssar_step_host: ssar_step for a host env, one call: H2D of obs_next, action, done and the rewards AS FLOAT64 (the
 *     reference sums Python floats, with the rounding above), then the ssar_step
 *     kernels, then obs <- the reset observation (obs_reset_host, or obs_next when obs_reset_host == obs_next_host).
 *     obs [N][D] holds s_t on entry and the next s_t on return.  Host pointers must be pinned. */
int sb200_ssar_step_host_f32(const sb200_ssar* ssar, const float* obs_next_host, const float* obs_reset_host,
                             const float* action_host, const double* reward_host, const float* done_host, float* obs,
                             float* obs_next_dev, float* action_dev, double* reward_dev, float* done_dev, void* stream);
/* CPython random.Random-compatible MT19937 on the HOST (uniform_replay.py:43-45 draws
 * random.randint(0, len-1) per sample; SURVEY Appendix A.6).  state_h: sb200_mt19937_state_bytes() bytes. */
size_t sb200_mt19937_state_bytes(void);
int sb200_mt19937_seed_h(void* state_h, const uint32_t* key_h, int key_len);     /* random.seed(int): 32-bit limbs */
int sb200_mt19937_set_state_h(void* state_h, const uint32_t* words624_h, int index);   /* random.getstate()[1] */
int sb200_mt19937_get_state_h(const void* state_h, uint32_t* words624_h, int* index);
int sb200_mt19937_randint_fill_h(void* state_h, int64_t population, int64_t count, int64_t* out_h);

#ifdef __cplusplus
}
#endif
#endif /* SURREAL_B200_H */
