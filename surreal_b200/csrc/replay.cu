// HBM-resident replay: FIFO queue control, gather of sampled records into the learner's batch buffers,
// the DDPG n-step SSAR staging + UniformReplay ring insert, a host-side MT19937 that reproduces
// CPython's random.randint index stream bit for bit, and the on-device uniform sampler (Philox indices + gather in one
// launch) that lets sample -> learn live inside one CUDA graph.
//
// Replaces surreal/replay/fifo_replay.py:6-48, uniform_replay.py:6-74, the aggregators' np.stack loops
// (aggregator.py:52-103,151-262) and ExpSenderWrapperSSARNStepBootstrap (exp_sender_wrapper.py:72-112).
// Records are stored SoA (one array per field, record-major) so that every field of a record is one
// contiguous, 16-byte aligned run: gathers move whole sectors.
#include "replay_dev.cuh"
#include <string.h>

namespace {

struct FifoState {          // must match rollout.cu
    int head;
    int count;
    int capacity;
    int dropped;
    long long total_in;
    long long total_out;
    unsigned int ticket;     // used by the fused sampling kernel (rollout.cu)
    int pad_;
};

// pop `batch` oldest windows: idx[k] = physical slot of the k-th oldest (fifo_replay.py:37-39).
__global__ void fifo_pop_kernel(FifoState* fifo, int batch, int* __restrict__ idx, int* __restrict__ status) {
    const int tid = threadIdx.x;
    const int head = fifo->head, count = fifo->count, cap = fifo->capacity;
    const bool ok = count >= batch;
    for (int k = tid; k < batch; k += blockDim.x) idx[k] = ok ? (int)(((long long)head + k) % cap) : 0;
    __syncthreads();
    if (tid == 0) {
        if (ok) {
            fifo->head = (int)(((long long)head + batch) % cap);
            fifo->count = count - batch;
            fifo->total_out += batch;
            *status = 0;
        } else {
            *status = 1;               // popleft from a too-short deque would raise IndexError in the reference
        }
    }
}

// host-driven push of `k` windows that already sit in slots chosen by this kernel (used by Replay.insert()).
__global__ void fifo_push_kernel(FifoState* fifo, int k, int* __restrict__ slots) {
    if (threadIdx.x != 0) return;
    int head = fifo->head, count = fifo->count;
    const int cap = fifo->capacity;
    for (int j = 0; j < k; ++j) {
        slots[j] = (int)(((long long)head + count) % cap);
        if (count == cap) {            // deque(maxlen) drops the oldest
            head = (head + 1) % cap;
            fifo->dropped += 1;
        } else {
            count += 1;
        }
    }
    fifo->head = head;
    fifo->count = count;
    fifo->total_in += k;
}

// out[b] = src[idx[b]] for records of `rec` floats (rec*4 bytes contiguous per record).
// One warp per record, float4 lanes when aligned: full 32-byte sectors on both sides.
__global__ void __launch_bounds__(256) gather_kernel(const float* __restrict__ src, long long rec,
                                                     const int* __restrict__ idx, const long long* __restrict__ idx64,
                                                     int batch, float* __restrict__ out, int vec) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int b = warp; b < batch; b += nwarps) {
        const long long s = (idx64 != nullptr) ? idx64[b] : (long long)idx[b];
        const float* sp = src + s * rec;
        float* dp = out + (long long)b * rec;
        if (vec) {
            const float4* s4 = reinterpret_cast<const float4*>(sp);
            float4* d4 = reinterpret_cast<float4*>(dp);
            for (long long k = lane; k < rec / 4; k += 32) d4[k] = s4[k];
        } else {
            for (long long k = lane; k < rec; k += 32) dp[k] = sp[k];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// ExpSenderWrapperSSARNStepBootstrap._step (exp_sender_wrapper.py:96-112), batched, + UniformReplay.insert.
// Per actor a deque of < n_step pending transitions [obs, action, reward(fp64), done]; every step each
// pending entry gets obs_next/done overwritten and reward += gamma^(n_step-i-1) * r (exponent by deque
// POSITION, the reference's warm-up quirk); the new transition is appended; when the deque holds n_step
// entries the oldest is emitted.  Emitted records go to ring slot (next_idx + rank) % capacity in actor
// order (uniform_replay.py:36-41).
// (UniformState {next_idx, size, capacity, total_in}: replay_dev.cuh)

// gamma^k for k < n_step, from the host's libm pow: the function CPython's float.__pow__ calls.
struct GammaPow {
    double p[SB200_SSAR_MAX_NSTEP];
};

// Rew: float for device envs, double for host envs, whose float64 rewards the reference sums as Python floats.
// Each step's product and sum are rounded separately, as `e += pow(gamma, k) * r` rounds them in Python: no FMA.
template <typename Rew>
__global__ void __launch_bounds__(1024) ssar_flags_kernel(const Rew* __restrict__ reward,
                                                          const float* __restrict__ done, int N, int n_step,
                                                          const GammaPow gp, int* __restrict__ dq_len,
                                                          double* __restrict__ dq_rew, int* __restrict__ dest,
                                                          float* __restrict__ emit_rew, UniformState* us,
                                                          unsigned long long* step_ctr) {
    __shared__ int warp_tot[32];
    __shared__ int warp_excl[32];
    __shared__ int chunk_total;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int base = 0;
    for (int i0 = 0; i0 < N; i0 += 1024) {
        const int i = i0 + tid;
        int flag = 0;
        if (i < N) {
            const int len = dq_len[i];
            const double r = (double)reward[i];
            double* q = dq_rew + (long long)i * n_step;
            for (int e = 0; e < len; ++e) q[e] = __dadd_rn(q[e], __dmul_rn(gp.p[n_step - e - 1], r));
            q[len] = r;                                   // append (position len)
            flag = (len + 1 == n_step) ? 1 : 0;
            if (flag) emit_rew[i] = (float)q[0];          // popleft's accumulated reward -> fp32 at the learner
        }
        int incl = flag;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const int w = warp_tot[lane];
            int wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += t;
            }
            warp_excl[lane] = wi - w;
            if (lane == 31) chunk_total = wi;
        }
        __syncthreads();
        if (i < N) dest[i] = flag ? (base + warp_excl[warp] + incl - flag) : -1;
        base += chunk_total;
        __syncthreads();
    }
    const long long K = base, cap = us->capacity, nxt = us->next_idx;
    for (int i = tid; i < N; i += 1024) {
        const int r = dest[i];
        if (r >= 0) dest[i] = (K > cap && r < K - cap) ? -1 : (int)((nxt + r) % cap);
    }
    __syncthreads();
    if (tid == 0) {
        us->next_idx = (nxt + K) % cap;
        us->size = (us->size + K > cap) ? cap : us->size + K;
        us->total_in += K;
        if (step_ctr != nullptr) *step_ctr += 1ull;
    }
}

// one block per actor: maintain the obs/action deque, write the emitted record into its replay slot.
__global__ void __launch_bounds__(128) ssar_commit_kernel(const float* __restrict__ obs, const float* __restrict__ action,
                                                          const float* __restrict__ obs_next,
                                                          const float* __restrict__ done, int N, int n_step, int D, int A,
                                                          int* __restrict__ dq_len, float* __restrict__ dq_obs,
                                                          float* __restrict__ dq_act, double* __restrict__ dq_rew,
                                                          const int* __restrict__ dest, const float* __restrict__ emit_rew,
                                                          float* __restrict__ r_obs, float* __restrict__ r_obs_next,
                                                          float* __restrict__ r_act, float* __restrict__ r_rew,
                                                          float* __restrict__ r_done) {
    const int i = blockIdx.x, tid = threadIdx.x;
    const int len = dq_len[i];
    float* qo = dq_obs + (long long)i * n_step * D;
    float* qa = dq_act + (long long)i * n_step * A;
    double* qr = dq_rew + (long long)i * n_step;
    // append the new transition's obs/action at position len
    for (int d = tid; d < D; d += blockDim.x) qo[(long long)len * D + d] = obs[(long long)i * D + d];
    for (int j = tid; j < A; j += blockDim.x) qa[(long long)len * A + j] = action[(long long)i * A + j];
    __syncthreads();
    int nlen = len + 1;
    const int slot = dest[i];
    const bool emit = (nlen == n_step);
    if (emit) {
        if (slot >= 0) {
            for (int d = tid; d < D; d += blockDim.x) {
                r_obs[(long long)slot * D + d] = qo[d];
                r_obs_next[(long long)slot * D + d] = obs_next[(long long)i * D + d];
            }
            for (int j = tid; j < A; j += blockDim.x) r_act[(long long)slot * A + j] = qa[j];
            if (tid == 0) {
                r_rew[slot] = emit_rew[i];
                r_done[slot] = done[i];
            }
        }
        __syncthreads();
        // popleft: shift the remaining n_step-1 entries down by one
        for (int e = 0; e + 1 < nlen; ++e) {
            for (int d = tid; d < D; d += blockDim.x) qo[(long long)e * D + d] = qo[(long long)(e + 1) * D + d];
            for (int j = tid; j < A; j += blockDim.x) qa[(long long)e * A + j] = qa[(long long)(e + 1) * A + j];
            __syncthreads();
        }
        if (tid == 0)
            for (int e = 0; e + 1 < nlen; ++e) qr[e] = qr[e + 1];
        nlen -= 1;
    }
    __syncthreads();
    if (done[i] > 0.5f) nlen = 0;                          // _reset clears the deque (exp_sender_wrapper.py:91-94)
    if (tid == 0) dq_len[i] = nlen;
}

// ---- host: CPython-compatible MT19937 ----------------------------------------------------------
struct MT {
    uint32_t mt[624];
    int idx;
};

void mt_init_genrand(MT* g, uint32_t s) {
    g->mt[0] = s;
    for (int i = 1; i < 624; ++i) g->mt[i] = 1812433253u * (g->mt[i - 1] ^ (g->mt[i - 1] >> 30)) + (uint32_t)i;
    g->idx = 624;
}

void mt_init_by_array(MT* g, const uint32_t* key, int klen) {
    mt_init_genrand(g, 19650218u);
    int i = 1, j = 0;
    uint32_t* mt = g->mt;
    for (int k = (624 > klen ? 624 : klen); k; --k) {
        mt[i] = (mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1664525u)) + key[j] + (uint32_t)j;
        ++i; ++j;
        if (i >= 624) { mt[0] = mt[623]; i = 1; }
        if (j >= klen) j = 0;
    }
    for (int k = 623; k; --k) {
        mt[i] = (mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1566083941u)) - (uint32_t)i;
        ++i;
        if (i >= 624) { mt[0] = mt[623]; i = 1; }
    }
    mt[0] = 0x80000000u;
    g->idx = 624;
}

inline uint32_t mt_next(MT* g) {
    uint32_t* mt = g->mt;
    if (g->idx >= 624) {
        for (int k = 0; k < 624; ++k) {
            const uint32_t y = (mt[k] & 0x80000000u) | (mt[(k + 1) % 624] & 0x7fffffffu);
            mt[k] = mt[(k + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        }
        g->idx = 0;
    }
    uint32_t y = mt[g->idx++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
}

// GatherFields / gather_record: replay_dev.cuh
__global__ void __launch_bounds__(256) gather_multi_kernel(const __grid_constant__ GatherFields f, const int* __restrict__ idx,
                                                           const long long* __restrict__ idx64, int batch) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int b = warp; b < batch; b += nwarps) {
        const long long s = (idx64 != nullptr) ? idx64[b] : (long long)idx[b];
        gather_record(f, s, b, lane);
    }
}

// ------------------------------------------------------------------------------------------------
// UniformReplay.sample (uniform_replay.py:43-47) without the host: `batch` i.i.d. draws WITH replacement, uniform over
// the `count` records of a sampling view {start, count, capacity} that lives in device memory, and the gather of the
// drawn records, in one launch.  Draw r of the view is ring slot (start + r) % capacity.
//
// Index stream: Philox call p = philox4x32_10(seed, draw_counter, p) serves draws 2p (words x:y) and 2p + 1 (words z:w);
// a draw takes its 64 random bits u = hi:lo and r = floor(u * count / 2^64) (__umul64hi).  No rejection loop: every
// thread does the same work, at a bias of at most count / 2^64 per index (< 2^-43 for a 2^20-slot ring).  The launch
// advances draw_counter itself (the last block to finish, after every block has read it), so a captured graph draws
// fresh indices at every replay.  Not the reference's stream: random.randint parity is sb200_mt19937_randint_fill_h.
// UniformView / UniformSampler: replay_dev.cuh

// One warp per Philox call = two records: lane 0 draws, the warp copies.
__global__ void __launch_bounds__(256) uniform_sample_gather_kernel(const __grid_constant__ GatherFields f,
                                                                    const UniformView* __restrict__ view,
                                                                    unsigned long long seed, UniformSampler* sm, int batch,
                                                                    long long* __restrict__ indices) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    const long long start = view->start, count = view->count, cap = view->capacity;
    const unsigned long long ctr = *(volatile unsigned long long*)&sm->draw_counter;
    if (count >= 1) {
        for (int p = warp; 2 * p < batch; p += nwarps) {
            unsigned long long r0 = 0, r1 = 0;
            if (lane == 0) {
                const Philox4 z = philox4x32_10(seed, ctr, (unsigned long long)p);
                r0 = __umul64hi(((unsigned long long)z.x << 32) | z.y, (unsigned long long)count);
                r1 = __umul64hi(((unsigned long long)z.z << 32) | z.w, (unsigned long long)count);
            }
            r0 = __shfl_sync(0xffffffffu, r0, 0);
            r1 = __shfl_sync(0xffffffffu, r1, 0);
            const long long s0 = (start + (long long)r0) % cap, s1 = (start + (long long)r1) % cap;
            const bool two = 2 * p + 1 < batch;
            if (lane == 0) {
                indices[2 * p] = s0;
                if (two) indices[2 * p + 1] = s1;
            }
            gather_record(f, s0, 2 * p, lane);
            if (two) gather_record(f, s1, 2 * p + 1, lane);
        }
    }
    if (last_block_ticket(&sm->ticket, gridDim.x) && threadIdx.x == 0) {
        sm->status = (count >= 1) ? 0 : 1;
        if (count >= 1) sm->draw_counter = ctr + 1ull;
    }
}

// The sampling view of the ring between two chunks of inserts: every filled slot that the next `reserve` inserts cannot
// overwrite.  While those inserts still land beyond the filled part the view is [0, size); once they wrap into live
// records it starts behind them, start = (next_idx + reserve) % capacity, and offers capacity - reserve records (the
// `reserve` oldest, about to be overwritten, are left out).
__global__ void uniform_view_kernel(const UniformState* __restrict__ us, long long reserve, UniformView* view) {
    const long long cap = us->capacity, size = us->size;
    const bool fits = size + reserve <= cap;
    view->start = fits ? 0 : (us->next_idx + reserve) % cap;
    view->count = fits ? size : cap - reserve;
    view->capacity = cap;
}

}  // namespace

extern "C" int sb200_fifo_pop(void* fifo_state, int batch, int* idx, int* status, void* stream) {
    SB200_REQUIRE(fifo_state && idx && status && batch >= 1);
    fifo_pop_kernel<<<1, 256, 0, (cudaStream_t)stream>>>((FifoState*)fifo_state, batch, idx, status);
    return sb200_launch_status();
}

extern "C" int sb200_fifo_push(void* fifo_state, int k, int* slots, void* stream) {
    SB200_REQUIRE(fifo_state && slots && k >= 1);
    fifo_push_kernel<<<1, 32, 0, (cudaStream_t)stream>>>((FifoState*)fifo_state, k, slots);
    return sb200_launch_status();
}

extern "C" int sb200_replay_gather_f32(const float* src, int64_t record_floats, const int* idx32, const int64_t* idx64,
                                       int batch, float* out, void* stream) {
    SB200_REQUIRE(src && out && (idx32 || idx64) && batch >= 1 && record_floats >= 1);
    const int vec = (record_floats % 4 == 0) && ((((uintptr_t)src) | ((uintptr_t)out)) & 15) == 0;
    int blocks = (batch + 7) / 8;
    if (blocks > 132 * 8) blocks = 132 * 8;
    gather_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(src, record_floats, idx32, (const long long*)idx64, batch, out,
                                                            vec);
    return sb200_launch_status();
}

extern "C" int sb200_replay_gather_multi_f32(const float* const* srcs, float* const* outs, const int64_t* record_floats,
                                             int nfields, const int* idx32, const int64_t* idx64, int batch, void* stream) {
    SB200_REQUIRE((idx32 || idx64) && batch >= 1);
    GatherFields f;
    SB200_REQUIRE(gather_fields_ok(srcs, outs, record_floats, nfields, &f));
    int blocks = (batch + 7) / 8;
    if (blocks > 132 * 8) blocks = 132 * 8;
    gather_multi_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(f, idx32, (const long long*)idx64, batch);
    return sb200_launch_status();
}

extern "C" size_t sb200_uniform_sampler_bytes(void) { return sizeof(UniformSampler); }

extern "C" int sb200_uniform_view(const void* uniform_state, int64_t reserve, int64_t* view, void* stream) {
    SB200_REQUIRE(uniform_state && view && reserve >= 0);
    uniform_view_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((const UniformState*)uniform_state, reserve, (UniformView*)view);
    return sb200_launch_status();
}

extern "C" int sb200_uniform_sample_gather_f32(const float* const* srcs, float* const* outs, const int64_t* record_floats,
                                               int nfields, const int64_t* view, uint64_t seed, void* sampler, int batch,
                                               int64_t* indices, void* stream) {
    SB200_REQUIRE(view && sampler && indices && batch >= 1);
    GatherFields f;
    SB200_REQUIRE(gather_fields_ok(srcs, outs, record_floats, nfields, &f));
    int blocks = ((batch + 1) / 2 + 7) / 8;
    if (blocks > 132 * 8) blocks = 132 * 8;
    uniform_sample_gather_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(f, (const UniformView*)view, seed,
                                                                          (UniformSampler*)sampler, batch,
                                                                          (long long*)indices);
    return sb200_launch_status();
}

extern "C" size_t sb200_uniform_state_bytes(void) { return sizeof(UniformState); }

// Host check of an SSAR staging descriptor: every buffer present and the shape sane (step_counter may be NULL).
static bool ssar_ok(const sb200_ssar* s) {
    return s != nullptr && s->N >= 1 && s->n_step >= 1 && s->n_step <= SB200_SSAR_MAX_NSTEP && s->D >= 1 && s->A >= 1 &&
           s->dq_len && s->dq_obs && s->dq_act &&
           s->dq_rew && s->dest && s->emit && s->uniform_state && s->r_obs && s->r_obs_next && s->r_act && s->r_rew &&
           s->r_done;
}

// The two kernels of one SSAR step; Rew: float for device envs, double for host envs.
template <typename Rew>
static int ssar_launch(const sb200_ssar* s, const float* obs, const float* action, const float* obs_next, const Rew* reward,
                       const float* done, cudaStream_t st) {
    GammaPow gp = {};
    for (int k = 0; k < s->n_step; ++k) gp.p[k] = pow(s->gamma, (double)k);
    ssar_flags_kernel<Rew><<<1, 1024, 0, st>>>(reward, done, s->N, s->n_step, gp, s->dq_len, s->dq_rew, s->dest,
                                               s->emit, (UniformState*)s->uniform_state,
                                               (unsigned long long*)s->step_counter);
    ssar_commit_kernel<<<s->N, 128, 0, st>>>(obs, action, obs_next, done, s->N, s->n_step, s->D, s->A, s->dq_len, s->dq_obs,
                                             s->dq_act, s->dq_rew, s->dest, s->emit, s->r_obs, s->r_obs_next, s->r_act,
                                             s->r_rew, s->r_done);
    return sb200_launch_status(2);
}

extern "C" int sb200_ssar_step_f32(const sb200_ssar* s, const float* obs, const float* action, const float* obs_next,
                                   const float* reward, const float* done, void* stream) {
    SB200_REQUIRE(ssar_ok(s) && obs && action && obs_next && reward && done);
    return ssar_launch(s, obs, action, obs_next, reward, done, (cudaStream_t)stream);
}

extern "C" int sb200_ssar_step_host_f32(const sb200_ssar* s, const float* obs_next_host, const float* obs_reset_host,
                                        const float* action_host, const double* reward_host, const float* done_host,
                                        float* obs, float* obs_next_dev, float* action_dev, double* reward_dev,
                                        float* done_dev, void* stream) {
    SB200_REQUIRE(ssar_ok(s) && obs_next_host && obs_reset_host && action_host && reward_host && done_host);
    SB200_REQUIRE(obs && obs_next_dev && action_dev && reward_dev && done_dev);
    const int N = s->N;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t row_bytes = (size_t)N * s->D * sizeof(float);
    SB200_CUDA(cudaMemcpyAsync(obs_next_dev, obs_next_host, row_bytes, cudaMemcpyHostToDevice, st));
    SB200_CUDA(cudaMemcpyAsync(action_dev, action_host, (size_t)N * s->A * sizeof(float), cudaMemcpyHostToDevice, st));
    SB200_CUDA(cudaMemcpyAsync(reward_dev, reward_host, (size_t)N * sizeof(double), cudaMemcpyHostToDevice, st));
    SB200_CUDA(cudaMemcpyAsync(done_dev, done_host, (size_t)N * sizeof(float), cudaMemcpyHostToDevice, st));
    const int rc = ssar_launch(s, obs, action_dev, obs_next_dev, reward_dev, done_dev, st);
    if (rc != SB200_OK) return rc;
    // s_t of the next transition, after the commit has appended this one's
    if (obs_reset_host != obs_next_host)
        SB200_CUDA(cudaMemcpyAsync(obs, obs_reset_host, row_bytes, cudaMemcpyHostToDevice, st));
    else
        SB200_CUDA(cudaMemcpyAsync(obs, obs_next_dev, row_bytes, cudaMemcpyDeviceToDevice, st));
    return SB200_OK;
}

// ---- CPython random.Random index stream (host) -------------------------------------------------
extern "C" size_t sb200_mt19937_state_bytes(void) { return sizeof(MT); }

extern "C" int sb200_mt19937_seed_h(void* state_h, const uint32_t* key_h, int key_len) {
    SB200_REQUIRE(state_h && key_h && key_len >= 1);
    mt_init_by_array((MT*)state_h, key_h, key_len);
    return SB200_OK;
}

extern "C" int sb200_mt19937_set_state_h(void* state_h, const uint32_t* words624_h, int index) {
    SB200_REQUIRE(state_h && words624_h && index >= 0 && index <= 624);
    memcpy(((MT*)state_h)->mt, words624_h, 624 * sizeof(uint32_t));
    ((MT*)state_h)->idx = index;
    return SB200_OK;
}

extern "C" int sb200_mt19937_get_state_h(const void* state_h, uint32_t* words624_h, int* index) {
    SB200_REQUIRE(state_h && words624_h && index);
    memcpy(words624_h, ((const MT*)state_h)->mt, 624 * sizeof(uint32_t));
    *index = ((const MT*)state_h)->idx;
    return SB200_OK;
}

extern "C" int sb200_mt19937_randint_fill_h(void* state_h, int64_t population, int64_t count, int64_t* out_h) {
    // random.randint(0, population-1) == _randbelow_with_getrandbits(population), population < 2^32:
    // k = population.bit_length(); r = getrandbits(k) = genrand_uint32() >> (32-k); repeat until r < population.
    SB200_REQUIRE(state_h && out_h && population >= 1 && population <= 0xffffffffLL && count >= 0);
    MT* g = (MT*)state_h;
    int k = 0;
    for (uint64_t v = (uint64_t)population; v; v >>= 1) ++k;
    for (int64_t c = 0; c < count; ++c) {
        uint32_t r;
        do { r = mt_next(g) >> (32 - k); } while ((int64_t)r >= population);
        out_h[c] = (int64_t)r;
    }
    return SB200_OK;
}
