// Prioritized experience replay on the device (Schaul et al. 2016, in the form of the reference's
// surreal/replay/prioritized_replay.py + segment_tree.py): a sum tree and a min tree of p^alpha over the slots of the
// uniform ring, the admission of new records at max_priority^alpha, proportional sampling with importance weights and
// the gather of the drawn records in one launch, and the write-back of new priorities.
//
// Two bugs of the reference are fixed here: its insert writes the new priority into the slot AFTER the record
// (prioritized_replay.py:62-66), and its sampler takes the mass from sum(0, len - 1), whose end is exclusive, so the
// newest record could never be drawn (prioritized_replay.py:119).  Here a record's own slot gets the priority, and the
// mass is taken over the whole view.
//
// Layout (include/surreal_b200.h, sb200_per_tree): heap order over P = leaves slots, fp32 leaves, fp64 internal sums,
// fp32 internal mins (a min is exact in any precision).  Every internal node is recomputed from its two children, by the
// CTA that owns its subtree or by the one CTA of the top levels: no float atomics, so a tree depends only on its leaves.
#include "replay_dev.cuh"

namespace {

constexpr int PER_SUBTREE = 2048;          // leaves per subtree CTA (1024 threads, two leaves each)
constexpr int PER_THREADS = 256;

struct PerCtrl {
    long long admitted;          // total_in of the uniform ring at the last admit
    long long updates;           // sample launches that drew: the step of the beta schedule
    float max_priority;          // running max of every raw priority set (prioritized_replay.py:41,143)
    unsigned int ticket;
};

struct PerTree {                 // the kernels' copy of sb200_per_tree
    long long cap, P, sub;
    float* leaf;
    double* sum;
    float* mn;
    unsigned int* dirty;
    int* owner;
    PerCtrl* ctrl;
};

__device__ __forceinline__ double node_sum(const PerTree& t, long long i) {
    return i >= t.P ? (double)t.leaf[i - t.P] : t.sum[i];
}
__device__ __forceinline__ float node_min(const PerTree& t, long long i) {
    if (i >= t.P) {
        const float v = t.leaf[i - t.P];
        return v > 0.0f ? v : INFINITY;
    }
    return t.mn[i];
}

// p^alpha as the leaf holds it: in fp64, rounded once
__device__ __forceinline__ float leaf_value(float p, double alpha) { return (float)pow((double)p, alpha); }

// One CTA per subtree of `sub` leaves: its internal nodes, level by level in shared memory, each written through to
// the tree.  Subtrees whose dirty flag is clear are skipped (unless `all`).
__global__ void __launch_bounds__(PER_SUBTREE / 2) per_subtree_kernel(const PerTree t, int all) {
    __shared__ double s_sum[PER_SUBTREE / 2];
    __shared__ float s_min[PER_SUBTREE / 2];
    const long long s = blockIdx.x;
    if (!all && t.dirty[s] == 0u) return;
    const long long nsub = t.P / t.sub, root = nsub + s;
    const int half = (int)(t.sub / 2), tid = threadIdx.x;
    // the level just above the leaves: node root * half + tid has leaves 2 tid, 2 tid + 1 of the subtree
    if (tid < half) {
        const long long l = s * t.sub + 2 * tid;
        const float a = t.leaf[l], b = t.leaf[l + 1];
        const double v = (double)a + (double)b;
        const float m = fminf(a > 0.0f ? a : INFINITY, b > 0.0f ? b : INFINITY);
        s_sum[tid] = v;
        s_min[tid] = m;
        t.sum[root * half + tid] = v;
        t.mn[root * half + tid] = m;
    }
    for (int w = half / 2; w >= 1; w >>= 1) {
        __syncthreads();
        double v = 0.0;
        float m = 0.0f;
        if (tid < w) {
            v = s_sum[2 * tid] + s_sum[2 * tid + 1];
            m = fminf(s_min[2 * tid], s_min[2 * tid + 1]);
        }
        __syncthreads();
        if (tid < w) {
            s_sum[tid] = v;
            s_min[tid] = m;
            t.sum[root * w + tid] = v;
            t.mn[root * w + tid] = m;
        }
    }
    if (tid == 0) t.dirty[s] = 0u;
}

// The levels above the subtree roots (nodes 1 .. nsub - 1), by one CTA, level by level through global memory.
__global__ void __launch_bounds__(1024) per_top_kernel(const PerTree t) {
    const long long nsub = t.P / t.sub;
    for (long long w = nsub / 2; w >= 1; w >>= 1) {
        for (long long i = w + threadIdx.x; i < 2 * w; i += blockDim.x) {
            t.sum[i] = t.sum[2 * i] + t.sum[2 * i + 1];
            t.mn[i] = fminf(t.mn[2 * i], t.mn[2 * i + 1]);
        }
        __syncthreads();
    }
}

// Admit: the slots of inserts [admitted, total_in) get max_priority^alpha (all slots once the gap reaches capacity).
__global__ void __launch_bounds__(PER_THREADS) per_admit_kernel(const PerTree t, const UniformState* __restrict__ us,
                                                                double alpha) {
    const long long total = us->total_in, admitted = t.ctrl->admitted, cap = t.cap;
    const long long gap = total - admitted;
    const long long n = gap >= cap ? cap : gap;
    const long long first = gap >= cap ? 0 : admitted % cap;
    const float v = leaf_value(t.ctrl->max_priority, alpha);
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const long long slot = (first + k) % cap;
        t.leaf[slot] = v;
        t.dirty[slot / t.sub] = 1u;
    }
    if (last_block_ticket(&t.ctrl->ticket, gridDim.x) && threadIdx.x == 0) t.ctrl->admitted = total;
}

// sum / min of leaves [l, r), bottom-up (left and right partial results, joined at the end)
__device__ double range_sum(const PerTree& t, long long l, long long r) {
    double left = 0.0, right = 0.0;
    for (l += t.P, r += t.P; l < r; l >>= 1, r >>= 1) {
        if (l & 1) left = left + node_sum(t, l++);
        if (r & 1) right = node_sum(t, --r) + right;
    }
    return left + right;
}
__device__ float range_min(const PerTree& t, long long l, long long r) {
    float m = INFINITY;
    for (l += t.P, r += t.P; l < r; l >>= 1, r >>= 1) {
        if (l & 1) m = fminf(m, node_min(t, l++));
        if (r & 1) m = fminf(m, node_min(t, --r));
    }
    return m;
}

// find_prefixsum_idx (segment_tree.py:101-124): the leaf where the running prefix passes x
__device__ long long descend(const PerTree& t, double x) {
    long long i = 1;
    while (i < t.P) {
        const double l = node_sum(t, 2 * i);
        if (l > x) {
            i = 2 * i;
        } else {
            x = x - l;
            i = 2 * i + 1;
        }
    }
    return i - t.P;
}

struct ViewSums {
    double s1, s;                // leaf sum of the first segment [start, end1), and of the whole view
    double base;                 // leaf sum of [0, start): the prefix in front of the view
    long long end1, end2;        // segments [start, end1) and [0, end2) (end2 = 0: the view does not wrap)
    float min_leaf;
    double beta;
};

// One warp per Philox call = two draws: lanes 0 and 1 each descend for one, the warp gathers both records.
__global__ void __launch_bounds__(256) per_sample_gather_kernel(const __grid_constant__ GatherFields f, const PerTree t,
                                                                const UniformView* __restrict__ view,
                                                                unsigned long long seed, UniformSampler* sm, int batch,
                                                                double beta0, double anneal, double beta_override,
                                                                long long* __restrict__ indices,
                                                                float* __restrict__ weights) {
    __shared__ ViewSums vs;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    const long long start = view->start, count = view->count;
    const unsigned long long ctr = *(volatile unsigned long long*)&sm->draw_counter;
    const long long upd = *(volatile long long*)&t.ctrl->updates;
    if (count >= 1) {
        if (threadIdx.x == 0) {
            const long long end = start + count;
            vs.end1 = end <= t.cap ? end : t.cap;
            vs.end2 = end <= t.cap ? 0 : end - t.cap;
            vs.base = range_sum(t, 0, start);
            vs.s1 = range_sum(t, start, vs.end1);
            vs.s = vs.end2 > 0 ? vs.s1 + range_sum(t, 0, vs.end2) : vs.s1;
            float m = range_min(t, start, vs.end1);
            if (vs.end2 > 0) m = fminf(m, range_min(t, 0, vs.end2));
            vs.min_leaf = m;
            double beta = beta0;
            if (beta_override >= 0.0) {
                beta = beta_override;
            } else if (anneal > 0.0) {                 // LinearSchedule (utils/schedule.py:96-99)
                const double frac = fmin((double)upd / anneal, 1.0);
                beta = beta0 + frac * (1.0 - beta0);
            }
            vs.beta = beta;
        }
        __syncthreads();
        for (int p = warp; 2 * p < batch; p += nwarps) {
            long long slot = 0;
            if (lane < 2) {
                const Philox4 z = philox4x32_10(seed, ctr, (unsigned long long)p);
                const unsigned long long word = lane == 0 ? (((unsigned long long)z.x << 32) | z.y)
                                                          : (((unsigned long long)z.z << 32) | z.w);
                const double u = (double)(word >> 11) * 0x1.0p-53;
                const double mass = __dmul_rn(u, vs.s);
                long long lo, hi;
                double x;
                if (vs.end2 == 0 || mass < vs.s1) {
                    x = vs.base + mass;
                    lo = start;
                    hi = vs.end1;
                } else {
                    x = mass - vs.s1;
                    lo = 0;
                    hi = vs.end2;
                }
                slot = descend(t, x);
                slot = slot < lo ? lo : (slot >= hi ? hi - 1 : slot);     // fp rounding at a segment's edge
                const int b = 2 * p + lane;
                if (b < batch) {
                    indices[b] = slot;
                    weights[b] = (float)pow((double)t.leaf[slot] / (double)vs.min_leaf, -vs.beta);
                }
            }
            const long long s0 = __shfl_sync(0xffffffffu, slot, 0), s1 = __shfl_sync(0xffffffffu, slot, 1);
            gather_record(f, s0, 2 * p, lane);
            if (2 * p + 1 < batch) gather_record(f, s1, 2 * p + 1, lane);
        }
    }
    if (last_block_ticket(&sm->ticket, gridDim.x) && threadIdx.x == 0) {
        sm->status = (count >= 1) ? 0 : 1;
        if (count >= 1) {
            sm->draw_counter = ctr + 1ull;
            t.ctrl->updates = upd + 1;
        }
    }
}

// Priority write-back, step 1: owner[slot] = the last batch position that names the slot.
__global__ void __launch_bounds__(PER_THREADS) per_owner_kernel(const PerTree t, const long long* __restrict__ idx,
                                                                int batch, const int* __restrict__ stop) {
    if (stop != nullptr && *stop != 0) return;
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    const long long s = idx[b];
    if (s >= 0 && s < t.cap) atomicMax(t.owner + s, b);
}

// Step 2: the owner writes the leaf, flags its subtree and hands the slot back (-1).  A non-owner reads either the
// owner's position or -1, never its own, so the reset needs no second launch.  max_priority takes every priority of the
// batch, overwritten ones included, as the reference's sequential loop does (prioritized_replay.py:137-143); atomicMax
// on the bits of a positive float is the float max, exactly.
__global__ void __launch_bounds__(PER_THREADS) per_write_kernel(const PerTree t, const long long* __restrict__ idx,
                                                                const float* __restrict__ prio, int batch, double alpha,
                                                                const int* __restrict__ stop) {
    if (stop != nullptr && *stop != 0) return;
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    const long long s = idx[b];
    if (s < 0 || s >= t.cap) return;
    const float p = prio[b];
    if (p > 0.0f) atomicMax(reinterpret_cast<int*>(&t.ctrl->max_priority), __float_as_int(p));   // every priority set
    if (t.owner[s] != b) return;
    t.leaf[s] = leaf_value(p, alpha);
    t.dirty[s / t.sub] = 1u;
    t.owner[s] = -1;
}

}  // namespace

static long long per_leaves(long long cap) {
    long long P = 2;
    while (P < cap) P <<= 1;
    return P;
}

static bool per_tree_ok(const sb200_per_tree* h, PerTree* t) {
    if (h == nullptr || h->capacity < 1 || !h->leaf || !h->sum || !h->mn || !h->dirty || !h->owner || !h->ctrl)
        return false;
    const long long P = per_leaves(h->capacity);
    const long long sub = P < PER_SUBTREE ? P : PER_SUBTREE;
    if (h->leaves != P || h->subtree != sub) return false;
    *t = PerTree{h->capacity, P, sub, h->leaf, h->sum, h->mn, (unsigned int*)h->dirty, (int*)h->owner,
                 (PerCtrl*)h->ctrl};
    return true;
}

static int per_rebuild(const PerTree& t, int all, cudaStream_t st) {
    const long long nsub = t.P / t.sub;
    per_subtree_kernel<<<(unsigned)nsub, (unsigned)(t.sub / 2), 0, st>>>(t, all);
    if (nsub > 1) {
        per_top_kernel<<<1, 1024, 0, st>>>(t);
        return sb200_launch_status(2);
    }
    return sb200_launch_status();
}

extern "C" size_t sb200_per_ctrl_bytes(void) { return sizeof(PerCtrl); }

extern "C" int sb200_per_tree_layout(int64_t capacity, int64_t* leaves, int64_t* subtree) {
    SB200_REQUIRE(capacity >= 1 && capacity <= (1ll << 30) && leaves && subtree);
    *leaves = per_leaves(capacity);
    *subtree = *leaves < PER_SUBTREE ? *leaves : PER_SUBTREE;
    return SB200_OK;
}

extern "C" int sb200_per_rebuild(const sb200_per_tree* tree, int full, void* stream) {
    PerTree t;
    SB200_REQUIRE(per_tree_ok(tree, &t));
    return per_rebuild(t, full != 0, (cudaStream_t)stream);
}

extern "C" int sb200_per_admit(const sb200_per_tree* tree, const void* uniform_state, double alpha, void* stream) {
    PerTree t;
    SB200_REQUIRE(per_tree_ok(tree, &t) && uniform_state && alpha >= 0.0);
    cudaStream_t st = (cudaStream_t)stream;
    long long blocks = (t.cap + PER_THREADS - 1) / PER_THREADS;
    if (blocks > 132 * 4) blocks = 132 * 4;
    per_admit_kernel<<<(unsigned)blocks, PER_THREADS, 0, st>>>(t, (const UniformState*)uniform_state, alpha);
    const int rc = sb200_launch_status();
    if (rc != SB200_OK) return rc;
    return per_rebuild(t, 0, st);
}

extern "C" int sb200_per_sample_gather_f32(const sb200_per_tree* tree, const float* const* srcs, float* const* outs,
                                           const int64_t* record_floats, int nfields, const int64_t* view, uint64_t seed,
                                           void* sampler, int batch, double beta0, double beta_anneal_iters,
                                           double beta_override, int64_t* indices, float* weights, void* stream) {
    PerTree t;
    SB200_REQUIRE(per_tree_ok(tree, &t) && view && sampler && indices && weights && batch >= 1);
    GatherFields f;
    SB200_REQUIRE(gather_fields_ok(srcs, outs, record_floats, nfields, &f));
    int blocks = ((batch + 1) / 2 + 7) / 8;
    if (blocks > 132 * 8) blocks = 132 * 8;
    per_sample_gather_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(f, t, (const UniformView*)view, seed,
                                                                       (UniformSampler*)sampler, batch, beta0,
                                                                       beta_anneal_iters, beta_override,
                                                                       (long long*)indices, weights);
    return sb200_launch_status();
}

extern "C" int sb200_per_update_f32(const sb200_per_tree* tree, const int64_t* indices, const float* priorities,
                                    int batch, double alpha, const int* stop_flag, void* stream) {
    PerTree t;
    SB200_REQUIRE(per_tree_ok(tree, &t) && indices && priorities && batch >= 1 && alpha >= 0.0);
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)((batch + PER_THREADS - 1) / PER_THREADS);
    per_owner_kernel<<<blocks, PER_THREADS, 0, st>>>(t, (const long long*)indices, batch, stop_flag);
    per_write_kernel<<<blocks, PER_THREADS, 0, st>>>(t, (const long long*)indices, priorities, batch, alpha, stop_flag);
    const int rc = sb200_launch_status(2);
    if (rc != SB200_OK) return rc;
    return per_rebuild(t, 0, st);
}
