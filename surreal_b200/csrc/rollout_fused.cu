// Persistent rollout kernel: T env steps of ALL co-located actors in ONE launch.
//
// The per-step launch sequence (policy forward -> sample -> env step -> window staging) is bound by fixed costs:
// every launch re-fetches the policy weights from L2 (a chain of dependent round trips) and pays
// launch + drain, 128 steps x 3 launches per rollout for a fraction of that in arithmetic.  Actors are
// independent of one another, so the loop over time can move INSIDE the kernel:
//   * a thread-block cluster of 4 CTAs owns a group of 32 actors (G = 2: two groups) for the whole chunk;
//   * each CTA keeps a QUARTER of every hidden layer's weights resident in shared memory for all T steps (fetched
//     once with cp.async); its 8 layer warps compute that quarter of the layer's columns for the group's 32 rows
//     (fp32 FFMA in register tiles) and push the result into the peers' shared memory with st.async, which counts
//     the bytes on the receiver's mbarrier: no cluster barrier inside the loop over steps;
//   * each CTA then finishes ITS 8 actors of the group: head, sampling, environment step, window staging -- one warp
//     per actor, observations / env state never leave shared memory between steps; the other 8 warps do the
//     action-independent half of the env step while the layers run;
//   * finished windows go to a per-actor outbox with their completion step; sb200_ppo_rollout_commit_f32 assigns
//     FIFO slots in the reference's (step, actor) arrival order afterwards and copies them into the replay ring.
// Sampling and environment arithmetic are those of rollout.cu, and both paths draw their noise from common.cuh
// (action_noise1, env_noise), so they draw the same noise; the policy forward is fp32 FFMA (the per-step path uses
// 3xTF32 tensor-core products; both are fp32-accurate, they differ by rounding order only).
#include <cooperative_groups.h>

#include <algorithm>
#include <mutex>

#include "common.cuh"
#include "rollout_dev.cuh"

namespace {

namespace cg = cooperative_groups;

constexpr int RF_CS = 4;            // CTAs per cluster
constexpr int RF_ROWS = 32;         // actors per cluster
constexpr int RF_OWN = RF_ROWS / RF_CS;
constexpr int RF_THREADS = 512;     // 16 warps: thread (ty = row 0..31, tx = column quad 0..15)

// -DRF_TRACE (tools/rollout_trace.py builds that variant; never the shipped library): clock64 stamps of cluster 0's
// first steps, one row per (CTA, step), read back through sb200_debug_rf_trace().
// RF_TID: the thread index the stamps and the layer functions go by
#define RF_TID threadIdx.x
#ifdef RF_TRACE
constexpr int RF_TR_STEPS = 8, RF_TR_IDS = 32;
__device__ long long g_rf_trace[RF_CS][RF_TR_STEPS][RF_TR_IDS];
#define RF_STAMP(id, who)                                                                           \
    do {                                                                                            \
        if (blockIdx.x < RF_CS && RF_TID == (who) && rf_t >= 2 && rf_t < 2 + RF_TR_STEPS)           \
            g_rf_trace[blockIdx.x][rf_t - 2][id] = clock64();                                       \
    } while (0)
// per CTA of the last launch: %smid, %globaltimer at entry, %globaltimer at exit (shows how many waves the grid ran in)
constexpr int RF_TR_CTAS = 4096;
__device__ long long g_rf_cta[RF_TR_CTAS][3];
__device__ __forceinline__ void rf_cta_stamp(int slot) {
    if (threadIdx.x != 0 || blockIdx.x >= RF_TR_CTAS) return;
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    if (slot == 1) {
        unsigned sm;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
        g_rf_cta[blockIdx.x][0] = sm;
    }
    g_rf_cta[blockIdx.x][slot] = (long long)t;
}
#define RF_CTA_STAMP(slot) rf_cta_stamp(slot)
#else
#define RF_STAMP(id, who) do { } while (0)
#define RF_CTA_STAMP(slot) do { } while (0)
#endif

struct RfParams {
    const float* W[3];
    const float* b[3];
    int ldw[3];
    int act[3];
    int D, H1, H2, A;
    const float* zf;
    float zf_eps;
    const float* log_var;
    const float* log_noise;
    unsigned long long agent_seed;
    int deterministic;
    float* state;
    const float* WsT;
    const float* WaT;
    int* ep_step;
    int max_steps;
    unsigned long long env_seed;
    float* action;
    float* pd;
    float* obs_next;
    float* reward;
    float* done;
    int* stage_pos;
    float* stage_obs;
    float* stage_act;
    float* stage_pd;
    float* stage_rew;
    float* stage_done;
    float* o_obs;
    float* o_act;
    float* o_pd;
    float* o_rew;
    float* o_done;
    int* ev_step;
    int* ev_count;
    int Wout;                       // outbox entries per actor
    int N, n_step, stride, T;
    const unsigned long long* step_ctr;
    // shared-memory plan (float offsets)
    int oW1, oW2, oWh, oB, oX0, oH1, oH2, oPart, oZf, oEnv, oS, oNext, oAct, oPre;
    int oHs;                        // two groups per cluster: head slice sums [16][8][ldw[2]]
    int gstride;                    // two groups per cluster: floats between group 0's and group 1's X0 .. Pre
    int ldx0, ldh1, ldh2;
    int head_mode;                  // G = 1: 1 = k-sliced head over all owned actors, 0 = two warps per actor
};

// Schedule of a step.  Warps 0..7 run the hidden layers; warps 8..15 meanwhile do the part of the env step that does
// not depend on the action (Philox + Box-Muller draws, Ws.s, |s|^2): it needs only the state at the top of the step, so
// it stays off the serial chain behind the layers.  Where a layer's k split goes through shared memory its register
// tiles are 8 rows x 4 columns: 12 LDS.128 per 128 FMA instead of 8 per 64 with 4 x 4 tiles -- the layer loop is bound
// by shared-memory loads, not by FFMA issue.  A warp = 16 column quads x 2 k-halves over ONE 8-row group, so the
// activation loads are warp-wide broadcasts.  Named barrier 1 joins the 256 threads of the layer warps.
__device__ __forceinline__ void rf_bar_math() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// ---- mbarrier-signalled DSMEM hand-offs.  A cluster barrier would cost more: barrier.cluster.arrive.release compiles
// to MEMBAR.ALL.GPU + ERRBAR + CGAERRBAR in front of the barrier (the kernel's global stores of the step must drain to
// L2 first) and the wait to a CCTL.IVALL.  st.async carries the data AND the completion count to the consumer's
// mbarrier, so the producer needs no fence and the consumer polls its own shared memory.
// Spin until the phase with this parity has completed; a transaction count that can never be met would hang the GPU, so
// the spin is bounded (~1 s) and traps instead.
__device__ __forceinline__ void rf_mbar_wait(uint64_t* bar, unsigned parity) {
    const unsigned a = smem_u32(bar);
    for (unsigned spin = 0;; ++spin) {
        unsigned ok;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(a), "r"(parity) : "memory");
        if (ok) return;
        if (spin > (1u << 26)) __trap();
    }
}
__device__ __forceinline__ void rf_st_async_v4(unsigned dst_cluster_addr, const float4& v, unsigned mbar_cluster_addr) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];"
                 ::"r"(dst_cluster_addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "r"(mbar_cluster_addr) : "memory");
}

// sum over the 32 lanes of s[j], returned in the lanes with j == 4*bit4 + 2*bit3 + bit2 of the lane index (9 shuffles)
__device__ __forceinline__ float rf_reduce8(const float (&s)[8], int lane) {
    const bool u4 = (lane & 16) != 0, u3 = (lane & 8) != 0, u2 = (lane & 4) != 0;
    float t[4], u[2];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float recv = __shfl_xor_sync(0xffffffffu, u4 ? s[i] : s[i + 4], 16);
        t[i] = (u4 ? s[i + 4] : s[i]) + recv;
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const float recv = __shfl_xor_sync(0xffffffffu, u3 ? t[i] : t[i + 2], 8);
        u[i] = (u3 ? t[i + 2] : t[i]) + recv;
    }
    float v = (u2 ? u[1] : u[0]) + __shfl_xor_sync(0xffffffffu, u2 ? u[0] : u[1], 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}

// First hidden layer on the 8 math warps WITHOUT a shared-memory reduction: K = D is short (64), so a 4-way k split
// reduced through shared memory spent more on partial tiles, the barrier and the second pass (1.5 K cycles) than on its
// 4 k quads of FMAs.
// Here warp w owns rows 4w..4w+3, lane = (column quad, k half); the two k halves of a lane pair are summed by shuffle
// (each lane keeps two of the four rows) and the epilogue stores / pushes straight from registers.
__device__ __forceinline__ void rf2_layer1(const float* __restrict__ Xin, int ldin, int K, const float* __restrict__ Ws, int Nc,
                                           const float* __restrict__ bias_s, int act, float* __restrict__ Hout, int ldout,
                                           int col0, unsigned smem_base, unsigned crank, unsigned bar_off) {
    const int tid = (int)RF_TID, warp = tid >> 5, lane = tid & 31;
    const int cg0 = lane & 15, kh = lane >> 4;
    const bool up = kh != 0;
    const int kq = (((K >> 2) + 1) >> 1) << 2;               // k span of one half (multiple of 4)
    const int k_lo = kh * kq, k_hi = min(K, k_lo + kq);
    const int nq = Nc >> 2;
    const float* xr = Xin + (warp * 4) * ldin;
    unsigned pb[RF_CS - 1];
#pragma unroll
    for (int c = 1; c < RF_CS; ++c) pb[c - 1] = mapa_u32(smem_base, (crank + (unsigned)c) % RF_CS);
    for (int c4 = cg0; c4 < ((nq + 15) & ~15); c4 += 16) {    // uniform trip count: the shuffles need the whole warp
        const bool on = c4 < nq;
        const float* wp = Ws + (on ? c4 : 0) * 4;
        float2 acc[4][2];
#pragma unroll
        for (int r = 0; r < 4; ++r) acc[r][0] = acc[r][1] = make_float2(0.0f, 0.0f);
#pragma unroll 2
        for (int k = k_lo; k < k_hi; k += 4) {
            const float4 w0 = *reinterpret_cast<const float4*>(wp + (k + 0) * Nc);
            const float4 w1 = *reinterpret_cast<const float4*>(wp + (k + 1) * Nc);
            const float4 w2 = *reinterpret_cast<const float4*>(wp + (k + 2) * Nc);
            const float4 w3 = *reinterpret_cast<const float4*>(wp + (k + 3) * Nc);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const float4 a = *reinterpret_cast<const float4*>(xr + r * ldin + k);
                float2 aa = make_float2(a.x, a.x);
                acc[r][0] = fma2(aa, make_float2(w0.x, w0.y), acc[r][0]);
                acc[r][1] = fma2(aa, make_float2(w0.z, w0.w), acc[r][1]);
                aa = make_float2(a.y, a.y);
                acc[r][0] = fma2(aa, make_float2(w1.x, w1.y), acc[r][0]);
                acc[r][1] = fma2(aa, make_float2(w1.z, w1.w), acc[r][1]);
                aa = make_float2(a.z, a.z);
                acc[r][0] = fma2(aa, make_float2(w2.x, w2.y), acc[r][0]);
                acc[r][1] = fma2(aa, make_float2(w2.z, w2.w), acc[r][1]);
                aa = make_float2(a.w, a.w);
                acc[r][0] = fma2(aa, make_float2(w3.x, w3.y), acc[r][0]);
                acc[r][1] = fma2(aa, make_float2(w3.z, w3.w), acc[r][1]);
            }
        }
        const float4 bv = *reinterpret_cast<const float4*>(bias_s + (on ? c4 : 0) * 4);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const float2 s0 = up ? acc[r][0] : acc[r + 2][0], s1 = up ? acc[r][1] : acc[r + 2][1];
            const float2 m0 = up ? acc[r + 2][0] : acc[r][0], m1 = up ? acc[r + 2][1] : acc[r][1];
            float4 o;
            o.x = apply_act((m0.x + __shfl_xor_sync(0xffffffffu, s0.x, 16)) + bv.x, act);
            o.y = apply_act((m0.y + __shfl_xor_sync(0xffffffffu, s0.y, 16)) + bv.y, act);
            o.z = apply_act((m1.x + __shfl_xor_sync(0xffffffffu, s1.x, 16)) + bv.z, act);
            o.w = apply_act((m1.y + __shfl_xor_sync(0xffffffffu, s1.y, 16)) + bv.w, act);
            if (on) {
                const int row = warp * 4 + (up ? 2 : 0) + r;
                float* qd = Hout + row * ldout + col0 + c4 * 4;
                *reinterpret_cast<float4*>(qd) = o;
                const unsigned off = smem_u32(qd) - smem_base;
#pragma unroll
                for (int c = 0; c < RF_CS - 1; ++c) rf_st_async_v4(pb[c] + off, o, pb[c] + bar_off);
            }
        }
    }
}

// Last hidden layer on the 8 math warps, for both schedules, WITHOUT a shared-memory reduction: four k quarters, each
// accumulated in k order by one lane, meet through two rounds of shuffles as ((p0 + p1) + (p2 + p3)) + bias (fp32
// addition is commutative, so which lane of a pair adds does not matter).  Warp = (row group rg = warp & 3: rows
// 8rg..8rg+7, column half ch = warp >> 2), lane = (column quad cq = lane & 7, k quarter ks = lane >> 3).  Each row goes
// only to the CTA that owns its actor, into its Hout [8][ldout] (input of the head).
__device__ __forceinline__ void rf2_layer2_direct(const float* __restrict__ Xin, int ldin, int K, const float* __restrict__ Ws,
                                                  int Nc, const float* __restrict__ bias_s, int act, float* __restrict__ Hout,
                                                  int ldout, int col0, unsigned smem_base, unsigned crank, unsigned bar_off) {
    const int tid = (int)RF_TID, warp = tid >> 5, lane = tid & 31;
    const int rg = warp & 3, ch = warp >> 2, cq = lane & 7, ks = lane >> 3;
    const bool u3 = (lane & 8) != 0, u4 = (lane & 16) != 0;
    const int kq = (((K >> 2) + 3) >> 2) << 2;               // k span of one quarter (multiple of 4)
    const int k_lo = ks * kq, k_hi = min(K, k_lo + kq);
    const int nq = Nc >> 2;
    const float* xr = Xin + (rg * 8) * ldin;
    for (int cb = ch * 8; cb < nq; cb += 16) {               // uniform trip count: the shuffles need the whole warp
        const int c4 = cb + cq;
        const bool on = c4 < nq;
        const float* wp = Ws + (on ? c4 : 0) * 4;
        float2 acc[8][2];
#pragma unroll
        for (int r = 0; r < 8; ++r) acc[r][0] = acc[r][1] = make_float2(0.0f, 0.0f);
#pragma unroll 2
        for (int k = k_lo; k < k_hi; k += 4) {
            const float4 w0 = *reinterpret_cast<const float4*>(wp + (k + 0) * Nc);
            const float4 w1 = *reinterpret_cast<const float4*>(wp + (k + 1) * Nc);
            const float4 w2 = *reinterpret_cast<const float4*>(wp + (k + 2) * Nc);
            const float4 w3 = *reinterpret_cast<const float4*>(wp + (k + 3) * Nc);
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const float4 a = *reinterpret_cast<const float4*>(xr + r * ldin + k);
                float2 aa = make_float2(a.x, a.x);
                acc[r][0] = fma2(aa, make_float2(w0.x, w0.y), acc[r][0]);
                acc[r][1] = fma2(aa, make_float2(w0.z, w0.w), acc[r][1]);
                aa = make_float2(a.y, a.y);
                acc[r][0] = fma2(aa, make_float2(w1.x, w1.y), acc[r][0]);
                acc[r][1] = fma2(aa, make_float2(w1.z, w1.w), acc[r][1]);
                aa = make_float2(a.z, a.z);
                acc[r][0] = fma2(aa, make_float2(w2.x, w2.y), acc[r][0]);
                acc[r][1] = fma2(aa, make_float2(w2.z, w2.w), acc[r][1]);
                aa = make_float2(a.w, a.w);
                acc[r][0] = fma2(aa, make_float2(w3.x, w3.y), acc[r][0]);
                acc[r][1] = fma2(aa, make_float2(w3.z, w3.w), acc[r][1]);
            }
        }
        // round 1, quarters 0 <-> 1 and 2 <-> 3: lanes with bit 3 clear keep rows 0..3, the others rows 4..7
        float2 s[4][2];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float2 snd = u3 ? acc[r][h] : acc[r + 4][h], kp = u3 ? acc[r + 4][h] : acc[r][h];
                s[r][h].x = kp.x + __shfl_xor_sync(0xffffffffu, snd.x, 8);
                s[r][h].y = kp.y + __shfl_xor_sync(0xffffffffu, snd.y, 8);
            }
        // round 2, (p0 + p1) <-> (p2 + p3): lanes with bit 4 clear keep the first two of their four rows
        const float4 bv = *reinterpret_cast<const float4*>(bias_s + (on ? c4 : 0) * 4);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const float2 snd0 = u4 ? s[r][0] : s[r + 2][0], kp0 = u4 ? s[r + 2][0] : s[r][0];
            const float2 snd1 = u4 ? s[r][1] : s[r + 2][1], kp1 = u4 ? s[r + 2][1] : s[r][1];
            float4 o;
            o.x = apply_act((kp0.x + __shfl_xor_sync(0xffffffffu, snd0.x, 16)) + bv.x, act);
            o.y = apply_act((kp0.y + __shfl_xor_sync(0xffffffffu, snd0.y, 16)) + bv.y, act);
            o.z = apply_act((kp1.x + __shfl_xor_sync(0xffffffffu, snd1.x, 16)) + bv.z, act);
            o.w = apply_act((kp1.y + __shfl_xor_sync(0xffffffffu, snd1.y, 16)) + bv.w, act);
            if (on) {
                const int row = rg * 8 + (u3 ? 4 : 0) + (u4 ? 2 : 0) + r;
                const unsigned owner = (unsigned)(row / RF_OWN);
                float* qd = Hout + (row - (int)owner * RF_OWN) * ldout + col0 + c4 * 4;
                if (owner == crank) *reinterpret_cast<float4*>(qd) = o;
                else {
                    const unsigned pb = mapa_u32(smem_base, owner);
                    rf_st_async_v4(pb + (smem_u32(qd) - smem_base), o, pb + bar_off);
                }
            }
        }
    }
}

__device__ __forceinline__ void rf_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void rf_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// The env matrices: G = 1 keeps them in shared memory, G = 2 reads them from global memory through L1.
template <int G>
__device__ __forceinline__ float rf_env_w(const float* w) {
    if constexpr (G == 2) return __ldg(w);
    else return *w;
}

// Group g's tiles and its owned actors' rows in shared memory (G = 2: group 1's lie gstride floats after group 0's).
struct RfGroup {
    float *X0, *H1, *H2, *S, *Nx;
    float *Ac, *Sd, *Zn, *Hp;             // [8][A] each: actions | std | N(0,1) draws | head_mode 0 halves [2][8][A]
    float *Eacc, *Egx, *Erz, *Eq;         // action-independent env step: [8][D] Ws.s, successor noise, reset draw | [8][2]
    // G = 2 keeps the action draws of a step in the buffer of its parity (rf2_action_noise): Zn | Act slot 1
    __device__ __forceinline__ float* zn2(int par, int A) const { return par ? Ac + RF_OWN * A : Zn; }
    __device__ __forceinline__ RfGroup(const RfParams& p, float* smem, int g) {
        float* b = smem + g * p.gstride;
        X0 = b + p.oX0; H1 = b + p.oH1; H2 = b + p.oH2; S = b + p.oS; Nx = b + p.oNext;
        Ac = b + p.oAct; Sd = Ac + 2 * RF_OWN * p.A; Zn = Sd + RF_OWN * p.A; Hp = Zn + RF_OWN * p.A;  // (slot 1: zn2, see rf_plan)
        Eacc = b + p.oPre; Egx = Eacc + RF_OWN * p.D; Erz = Egx + RF_OWN * p.D; Eq = Erz + RF_OWN * p.D;
    }
};

// One-time loads of a chunk: this CTA's column quarters of the hidden layers' weights and the whole head by cp.async (G = 1:
// the env matrices too), biases, z-filter columns, the owned actors' deque length and episode step, every group's owned
// state rows and input tile, the std rows; the mbarriers are initialised.  Ends with the cluster barrier and returns the
// step counter the chunk starts at.
template <int G>
__device__ __forceinline__ unsigned long long rf_setup(const RfParams& p, unsigned crank, int (&s_pos)[G][RF_OWN],
                                                       int (&s_ep)[G][RF_OWN], int (&s_cnt)[G][RF_OWN],
                                                       uint64_t (&s_bar)[G][3]) {
    extern __shared__ __align__(16) float smem[];
    const int tid = (int)RF_TID, lane = tid & 31, warp = tid >> 5;
    const int D = p.D, H1 = p.H1, H2 = p.H2, A = p.A;
    const int Nc1 = H1 / RF_CS, Nc2 = H2 / RF_CS;
    const int ldwh = p.ldw[2];
    float* B1s = smem + p.oB;
    float* B2s = B1s + Nc1;
    float* Bhs = B2s + Nc2;
    float* Zm = smem + p.oZf;
    float* Zs = Zm + D;
    const long long row0 = (long long)(blockIdx.x / RF_CS) * (G * RF_ROWS);
    for (int f = tid; f < D * (Nc1 >> 2); f += RF_THREADS) {
        const int k = f / (Nc1 >> 2), q = f - k * (Nc1 >> 2);
        cp_async16(smem + p.oW1 + k * Nc1 + q * 4, p.W[0] + (long long)k * p.ldw[0] + crank * Nc1 + q * 4, 16);
    }
    for (int f = tid; f < H1 * (Nc2 >> 2); f += RF_THREADS) {
        const int k = f / (Nc2 >> 2), q = f - k * (Nc2 >> 2);
        cp_async16(smem + p.oW2 + k * Nc2 + q * 4, p.W[1] + (long long)k * p.ldw[1] + crank * Nc2 + q * 4, 16);
    }
    for (int f = tid; f < (H2 * ldwh) >> 2; f += RF_THREADS) cp_async16(smem + p.oWh + f * 4, p.W[2] + f * 4, 16);
    if constexpr (G == 1) {
        float* EWs = smem + p.oEnv;
        for (int f = tid; f < (D * D) >> 2; f += RF_THREADS) cp_async16(EWs + f * 4, p.WsT + f * 4, 16);
        for (int f = tid; f < (A * D) >> 2; f += RF_THREADS) cp_async16(EWs + D * D + f * 4, p.WaT + f * 4, 16);
    }
    cp_async_commit();
    for (int n = tid; n < Nc1; n += RF_THREADS) B1s[n] = p.b[0][crank * Nc1 + n];
    for (int n = tid; n < Nc2; n += RF_THREADS) B2s[n] = p.b[1][crank * Nc2 + n];
    for (int n = tid; n < ldwh; n += RF_THREADS) Bhs[n] = (n < A) ? p.b[2][n] : 0.0f;
    if (p.zf != nullptr) {
        const float cnt = p.zf[2 * D];
        for (int k = tid; k < D; k += RF_THREADS) {
            const float mean = p.zf[k] / cnt;
            const float var = p.zf[D + k] / cnt - mean * mean;
            Zm[k] = mean;
            Zs[k] = fmaxf(sqrtf(var), p.zf_eps);
        }
    }
    if (tid < G * RF_OWN) {
        const int g = tid / RF_OWN, a = tid - g * RF_OWN;
        const long long i = row0 + g * RF_ROWS + crank * RF_OWN + a;
        s_pos[g][a] = (i < p.N) ? p.stage_pos[i] : 0;
        s_ep[g][a] = (i < p.N) ? p.ep_step[i] : 0;
        s_cnt[g][a] = 0;
    }
    __syncthreads();
    for (int idx = tid; idx < G * RF_ROWS * D; idx += RF_THREADS) {
        const int gm = idx / D, k = idx - gm * D;
        const int g = gm / RF_ROWS, m = gm - g * RF_ROWS;
        const long long i = row0 + g * RF_ROWS + m;
        float v = (i < p.N) ? p.state[i * D + k] : 0.0f;
        const int own = m - (int)crank * RF_OWN;
        if (own >= 0 && own < RF_OWN) smem[p.oS + g * p.gstride + own * D + k] = v;
        if (p.zf != nullptr) v = fminf(fmaxf((v - Zm[k]) / Zs[k], -5.0f), 5.0f);
        smem[p.oX0 + g * p.gstride + m * p.ldx0 + k] = (i < p.N) ? v : 0.0f;
    }
    if (tid == 0) {
        for (int g = 0; g < G; ++g)
            for (int i = 0; i < 3; ++i) mbar_init(&s_bar[g][i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // the warps that finish the owned actors (G = 1: warps 0..7, G = 2: warps 8..15) keep their std rows
    const int own = warp & (RF_OWN - 1);
    if ((warp < RF_OWN) == (G == 1) && lane < A) {
        for (int g = 0; g < G; ++g) {
            const long long i = row0 + g * RF_ROWS + crank * RF_OWN + own;
            const float sc = (i < p.N && p.log_noise != nullptr) ? expf(p.log_noise[i]) : 1.0f;
            RfGroup(p, smem, g).Sd[own * A + lane] = ppo_std(p.log_var[lane], sc);
        }
    }
    const unsigned long long ctr0 = (p.step_ctr != nullptr) ? *p.step_ctr : 0ull;
    cp_async_wait<0>();
    cg::this_cluster().sync();
    return ctr0;
}

// Head, head_mode 1: k slice sl = [sl H2/16, (sl+1) H2/16) for ALL 8 owned actors (lane = actor x 4 k sub-lanes), so the
// head weights are read from shared memory once per step instead of once per actor (the 2 x 8 KB per actor were 1 K
// cycles of the shared-memory pipe).  The slice sums go to Hsum [16][8][ldw[2]].
__device__ __forceinline__ void rf_head_slice(const RfParams& p, const float* __restrict__ H2rows,
                                              const float* __restrict__ Whs, int sl, int lane, float* __restrict__ Hsum) {
    const int ks = p.H2 >> 4;                             // H2 % 16 == 0 (rf_plan)
    const int ldwh = p.ldw[2];
    const int a8 = lane >> 2, ksub = lane & 3;
    const bool u1 = (lane & 2) != 0, u0 = (lane & 1) != 0;
    const float* hrow = H2rows + a8 * p.ldh2 + sl * ks;
    const float* wbase = Whs + (sl * ks) * ldwh;
    for (int n8 = 0; n8 < p.A; n8 += 8) {
        float s8[8];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) s8[jj] = 0.0f;
        const bool second = (n8 + 4 < ldwh);
        for (int k = ksub; k < ks; k += 4) {
            const float hv = hrow[k];
            const float* wr = wbase + k * ldwh + n8;
            const float4 w0 = *reinterpret_cast<const float4*>(wr);
            s8[0] = fmaf(hv, w0.x, s8[0]); s8[1] = fmaf(hv, w0.y, s8[1]);
            s8[2] = fmaf(hv, w0.z, s8[2]); s8[3] = fmaf(hv, w0.w, s8[3]);
            if (second) {
                const float4 w1 = *reinterpret_cast<const float4*>(wr + 4);
                s8[4] = fmaf(hv, w1.x, s8[4]); s8[5] = fmaf(hv, w1.y, s8[5]);
                s8[6] = fmaf(hv, w1.z, s8[6]); s8[7] = fmaf(hv, w1.w, s8[7]);
            }
        }
        // sum over the 4 k sub-lanes: after two exchange rounds lane ksub holds outputs 2 ksub', 2 ksub' + 1
        float t4[4], t2[2];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float recv = __shfl_xor_sync(0xffffffffu, u1 ? s8[i] : s8[i + 4], 2);
            t4[i] = (u1 ? s8[i + 4] : s8[i]) + recv;
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const float recv = __shfl_xor_sync(0xffffffffu, u0 ? t4[i] : t4[i + 2], 1);
            t2[i] = (u0 ? t4[i + 2] : t4[i]) + recv;
        }
        const int j0 = n8 + (u1 ? 4 : 0) + (u0 ? 2 : 0);
        float* dst = Hsum + ((sl * RF_OWN + a8) * ldwh);
        if (j0 < p.A) dst[j0] = t2[0];
        if (j0 + 1 < p.A) dst[j0 + 1] = t2[1];
    }
}

// Step t of owned actor `own` of a group, by the warp that finishes it, from the head's sums on: action and its staging,
// the chunk's final outputs, the action-dependent half of the env step, reward and done, the episode step, and the
// outbox entry of a window that completes.  Hsum: the head_mode 1 slice sums (rf_head_slice).  Returns the slot for
// commit_actor; rew / dn are set in every lane.
template <int G>
__device__ __forceinline__ int rf_act_env(const RfParams& p, const RfGroup& gr, int t, int own, int lane, long long i_own,
                                          const float* __restrict__ Hsum, const float* __restrict__ Bhs,
                                          const float* __restrict__ EWa, int pos, int& ep_s, int& cnt_s, float& rew,
                                          float& dn) {
    [[maybe_unused]] const int rf_t = t;              // read by RF_STAMP only
    const int D = p.D, A = p.A, ldwh = p.ldw[2];
    const bool valid = i_own < p.N, final_step = (t == p.T - 1);
    const float* zn = (G == 2) ? gr.zn2(t & 1, A) : gr.Zn;
    int slot = SLOT_NONE;
    if (lane < A) {
        const int j = lane;
        float pre;
        if (G == 2 || p.head_mode == 1) {             // G = 2 runs head_mode 1 only (rf_shape)
            pre = 0.0f;
#pragma unroll 4
            for (int w = 0; w < RF_THREADS / 32; ++w) pre += Hsum[(w * RF_OWN + own) * ldwh + j];    // fixed order
        } else {
            pre = gr.Hp[own * A + j] + gr.Hp[(RF_OWN + own) * A + j];
        }
        RF_STAMP(19, 0);
        const float mu = apply_act(pre + Bhs[j], p.act[2]);
        const float sd = gr.Sd[own * A + j];
        const float a = ppo_action(mu, sd, zn[own * A + j], p.deterministic);
        gr.Ac[own * A + j] = a;
        if (valid) {
            p.stage_act[((long long)i_own * p.n_step + pos) * A + j] = a;
            p.stage_pd[((long long)i_own * p.n_step + pos) * 2 * A + j] = mu;
            p.stage_pd[((long long)i_own * p.n_step + pos) * 2 * A + A + j] = sd;
            if (final_step) {
                p.action[i_own * A + j] = a;
                p.pd[i_own * 2 * A + j] = mu;
                p.pd[i_own * 2 * A + A + j] = sd;
            }
        }
    }
    __syncwarp();
    RF_STAMP(20, 0);
    float* sown = gr.S + own * D;
    const int ep = ep_s + 1;
    const bool is_done = env_done(ep, p.max_steps);
    dn = is_done ? 1.0f : 0.0f;
    rew = env_reward(gr.Eq[2 * own], D, gr.Eq[2 * own + 1]);
    for (int d = lane; d < D; d += 32) {
        float acc = gr.Eacc[own * D + d];
#pragma unroll 4
        for (int k = 0; k < A; ++k) acc = fmaf(rf_env_w<G>(EWa + k * D + d), gr.Ac[own * A + k], acc);
        const float nxt = env_successor(acc, gr.Egx[own * D + d]);
        gr.Nx[own * D + d] = nxt;
        sown[d] = is_done ? gr.Erz[own * D + d] : nxt;
        if (valid && final_step) p.obs_next[i_own * D + d] = nxt;
    }
    RF_STAMP(21, 0);
    if (lane == 0) {
        ep_s = is_done ? 0 : ep;
        if (valid && final_step) {
            p.reward[i_own] = rew;
            p.done[i_own] = dn;
        }
        if (valid && pos + 1 == p.n_step) {
            const int w = cnt_s;
            if (w < p.Wout) {
                slot = (int)(i_own * p.Wout + w);
                p.ev_step[slot] = t;
                cnt_s = w + 1;
            } else {
                slot = SLOT_DROPPED;
            }
        }
    }
    slot = __shfl_sync(0xffffffffu, slot, 0);
    __syncwarp();
    return slot;
}

// Next observation of owned actor `own` (tile row m) -> z-filter -> its row of this CTA's input tile and, by st.async
// counted on the peers' mbarrier at bar_off, of the three peers' tiles.  Not after a chunk's last step: nobody reads it.
__device__ __forceinline__ void rf_push_input(const RfParams& p, const RfGroup& gr, int own, int m, long long i_own,
                                              int lane, unsigned smem_base, const unsigned (&peer_base)[RF_CS - 1],
                                              unsigned bar_off) {
    extern __shared__ __align__(16) float smem[];
    const float* Zm = smem + p.oZf;
    const float* Zs = Zm + p.D;
    const int q4 = lane;
    if (q4 < (p.D >> 2)) {
        float4 v = *reinterpret_cast<const float4*>(gr.S + own * p.D + q4 * 4);
        if (i_own >= p.N) v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p.zf != nullptr) {
            const float4 zm = *reinterpret_cast<const float4*>(Zm + q4 * 4);
            const float4 zs = *reinterpret_cast<const float4*>(Zs + q4 * 4);
            v.x = fminf(fmaxf((v.x - zm.x) / zs.x, -5.0f), 5.0f);
            v.y = fminf(fmaxf((v.y - zm.y) / zs.y, -5.0f), 5.0f);
            v.z = fminf(fmaxf((v.z - zm.z) / zs.z, -5.0f), 5.0f);
            v.w = fminf(fmaxf((v.w - zm.w) / zs.w, -5.0f), 5.0f);
            if (i_own >= p.N) v = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float* qx = gr.X0 + m * p.ldx0 + q4 * 4;
        *reinterpret_cast<float4*>(qx) = v;
        const unsigned off = smem_u32(qx) - smem_base;
#pragma unroll
        for (int c = 0; c < RF_CS - 1; ++c) rf_st_async_v4(peer_base[c] + off, v, peer_base[c] + bar_off);
    }
}

// Two groups: the action draws N(0, 1) of step t of group g (owned actors i0 .. i0 + 7) by the layer warps, into the
// buffer of parity t & 1 (RfGroup::zn2).  They depend on neither state nor action, so the layer warps take them while
// they would otherwise wait for the other group's input rows, and the tail warps, whose chain sets the step, no longer
// run a Philox round and two Box-Muller draws per actor for them.  The values are those of action_noise1 at the same
// counter.  A called function: inlined, its registers pushed the layer code into spills.
__device__ __noinline__ void rf2_action_noise(const RfParams& p, const RfGroup& gr, long long i0, unsigned long long ctr,
                                              int par, int tid) {
    const int A = p.A, nq = (A + 3) >> 2;
    float* zn = gr.zn2(par, A);
    for (int idx = tid; idx < RF_OWN * nq; idx += RF_THREADS / 2) {
        const int a = idx / nq, q = idx - a * nq;
        const float4 z = action_noise4(p.agent_seed, ctr, i0 + a, q);
        const float zv[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
        for (int c = 0; c < 4; ++c)
            if (4 * q + c < A) zn[a * A + 4 * q + c] = zv[c];
    }
}

// Two groups of 32 actors per cluster (G = 2), software-pipelined, so that a chunk of N actors needs half as many
// clusters.  Warps 0..7 ("layer warps") run hidden layers 1 and 2 for group 0, then for group 1, step after step.
// Warps 8..15 ("tail warps", warp 8 + a for owned actor a of each group) take the whole tail of a group -- the
// action-independent env precompute, head, sampling, env step, window staging, the push of the next input rows -- while
// the layer warps compute the other group.  Arithmetic, operand order and Philox keys are those of the G = 1 schedule
// (head_mode 1, the same layer, head slice and tail functions), so both give the same results.
//
// Hand-offs, per group g (each group has its own tiles, state and three mbarriers):
//   layer -> peers: H1 rows (all 32) and H2 rows (owners' only) by st.async, counted on the receiver's h1[g] / h2[g];
//   layer -> tail:  own H2 rows, named barrier 2 + g (layer warps bar.arrive, tail warps bar.sync; 512 threads);
//   tail  -> peers: next X0 rows by st.async, counted on x0[g];
//   tail  -> layer: own next X0 rows, named barrier 4 + g (tail warps bar.arrive, layer warps bar.sync).
// No reverse "buffer free" signal is needed: every buffer of group g is rewritten only behind a chain of hand-offs that
// starts after its last reader is done.
//   * X0[g], step t+1: a peer pushes it after its head of step t, which needs this CTA's H2 rows of step t, which the
//     layer warps push only after all of them passed layer 1 (rf_bar_math), the last reader of X0[g].  The tail warps
//     rewrite their own rows after their head, i.e. after named barrier 2 + g, which every layer warp reaches after layer 2.
//   * H1[g], step t+1: a peer pushes it after its layer 1 of step t+1, which needs this CTA's X0 rows of step t+1, which
//     the tail warps push after named barrier 2 + g: after every layer warp has finished layer 2, the reader of H1[g].
//   * H2[g], step t+1: written by layer 2 of step t+1 (peers' and own), behind layer 1 of step t+1, behind the X0 rows of
//     step t+1 of every CTA of the cluster, which this CTA's tail pushes after its head of step t, the reader of H2[g].
//   * the same chains order every st.async of step t+1 after the mbarrier wait of step t, so no phase receives bytes of
//     the next one.  Each phase is armed once (expect_tx; arrival count 1) by thread 0 after the previous phase is known
//     complete: h1[g] and h2[g] after the layer warps' wait on named barrier 4 + g (the tail waited h2[g] of the step
//     before), x0[g] after the layer warps' own wait on x0[g].
//   * named barriers 2 + g and 4 + g never see two generations of arrivals at once: each arrival of step t+1 sits behind
//     the other side's arrival of step t on the other barrier.
//   * the head slice buffer is used by the tail warps only, between named barrier 6 (tail warps, 256 threads) and the
//     next group's named barrier 2 + g', which all 256 tail threads must reach.
__device__ __forceinline__ void rf2_two_groups(const RfParams& p, unsigned crank, unsigned long long ctr0,
                                               int (&s_pos)[2][RF_OWN], int (&s_ep)[2][RF_OWN], int (&s_cnt)[2][RF_OWN],
                                               uint64_t (&s_bar)[2][3]) {
    constexpr int G = 2;
    extern __shared__ __align__(16) float smem[];
    const unsigned smem_base = smem_u32(smem);
    unsigned peer_base[RF_CS - 1];
#pragma unroll
    for (int c = 1; c < RF_CS; ++c) peer_base[c - 1] = mapa_u32(smem_base, (crank + (unsigned)c) % RF_CS);
    const int tid = (int)RF_TID, lane = tid & 31, warp = tid >> 5;
    const int D = p.D, H1 = p.H1, H2 = p.H2, A = p.A;
    const int Nc1 = H1 / RF_CS, Nc2 = H2 / RF_CS;
    float* B1s = smem + p.oB;
    float* B2s = B1s + Nc1;
    float* Bhs = B2s + Nc2;
    float* Hs = smem + p.oHs;
    const float* __restrict__ EWs = p.WsT;   // env matrices: global memory, through L1
    const long long row0 = (long long)(blockIdx.x / RF_CS) * (G * RF_ROWS);
    // bytes a CTA receives from its three peers per step and group (as G = 1)
    const unsigned tx_h1 = 3u * RF_ROWS * Nc1 * 4u, tx_h2 = 3u * RF_OWN * Nc2 * 4u, tx_x0 = 3u * RF_OWN * D * 4u;
    const bool layer = warp < RF_OWN;
    const int own = warp & (RF_OWN - 1);              // tail warp 8 + own: owned actor `own` of each group

    if (layer) {
        for (int t = 0; t < p.T; ++t) {
            const bool final_step = (t == p.T - 1);
            [[maybe_unused]] const int rf_t = t;      // read by RF_STAMP only
            RF_STAMP(0, 0);
            for (int g = 0; g < G; ++g) {
                const RfGroup gr(p, smem, g);
                const long long i0 = row0 + g * RF_ROWS + (int)crank * RF_OWN;
                if (t == 0 && !p.deterministic) rf2_action_noise(p, gr, i0, ctr0, 0, tid);
                if (t > 0) {                                   // own rows from the tail warps, the peers' rows by st.async
                    rf_bar_sync(4 + g, 2 * 256);
                    rf_mbar_wait(&s_bar[g][2], (unsigned)(t - 1) & 1u);
                }
                if (tid == 0) {
                    mbar_arrive_expect_tx(&s_bar[g][0], tx_h1);
                    mbar_arrive_expect_tx(&s_bar[g][1], tx_h2);
                    if (!final_step) mbar_arrive_expect_tx(&s_bar[g][2], tx_x0);
                }
                rf2_layer1(gr.X0, p.ldx0, D, smem + p.oW1, Nc1, B1s, p.act[0], gr.H1, p.ldh1, (int)crank * Nc1, smem_base,
                           crank, smem_u32(&s_bar[g][0]) - smem_base);
                rf_bar_math();
                rf_mbar_wait(&s_bar[g][0], (unsigned)t & 1u);
                RF_STAMP(3 + 2 * g, 0);
                rf2_layer2_direct(gr.H1, p.ldh1, H1, smem + p.oW2, Nc2, B2s, p.act[1], gr.H2, p.ldh2, (int)crank * Nc2,
                                  smem_base, crank, smem_u32(&s_bar[g][1]) - smem_base);
                RF_STAMP(4 + 2 * g, 0);
                rf_bar_arrive(2 + g, 2 * 256);
                // the next step's action draws: their buffer's last reader, the tail's env step of step t - 1, is behind
                // named barrier 4 + g above; the tail reads them behind barrier 2 + g of step t + 1
                if (!final_step && !p.deterministic)
                    rf2_action_noise(p, gr, i0, ctr0 + (unsigned long long)(t + 1), (t + 1) & 1, tid);
            }
        }
        return;
    }
    for (int t = 0; t < p.T; ++t) {
        const unsigned long long ctr = ctr0 + (unsigned long long)t;
        [[maybe_unused]] const int rf_t = t;          // read by RF_STAMP only
        for (int g = 0; g < G; ++g) {
            const RfGroup gr(p, smem, g);
            const int m_own = (int)crank * RF_OWN + own;
            const long long i_own = row0 + g * RF_ROWS + m_own;
            RF_STAMP(8 + 4 * g, 256);
            // ---- everything of the step that does not depend on the action: the env warps' arithmetic of G = 1.  Here
            // this work is on the step's critical path, next to layer warps that keep the shared-memory pipe busy, so
            // what it puts through L1 counts.  Ws.s for the group's 8 owned actors is one register-tiled product on
            // tail warps 8..11 (tt < 128): a thread takes column d of 4 actors, so each weight is read through L1 twice
            // per group and step instead of once per actor, and the state rows are warp-wide float4 broadcasts.  Each
            // output is one fmaf chain over k in ascending order, as in the G = 1 env warps, so both give the same bits.
            // Eacc is read by the actors' warps behind named barrier 6 (the head), and rewritten only after every tail
            // warp passed barrier 6 of the other group, behind its last reader; the state rows read here were last
            // written before that same barrier.
            {
                const int tt = tid - RF_THREADS / 2;
                if (tt < 128) {
                    const int a0 = (tt >> 6) * 4;
                    const float* s0 = gr.S + a0 * D;
                    for (int d = tt & 63; d < D; d += 64) {
                        float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll 4
                        for (int k = 0; k < D; k += 4) {
                            const float w0 = __ldg(EWs + (k + 0) * D + d), w1 = __ldg(EWs + (k + 1) * D + d);
                            const float w2 = __ldg(EWs + (k + 2) * D + d), w3 = __ldg(EWs + (k + 3) * D + d);
#pragma unroll
                            for (int a = 0; a < 4; ++a) {
                                const float4 s4 = *reinterpret_cast<const float4*>(s0 + a * D + k);
                                acc[a] = fmaf(w0, s4.x, acc[a]);
                                acc[a] = fmaf(w1, s4.y, acc[a]);
                                acc[a] = fmaf(w2, s4.z, acc[a]);
                                acc[a] = fmaf(w3, s4.w, acc[a]);
                            }
                        }
#pragma unroll
                        for (int a = 0; a < 4; ++a) gr.Eacc[(a0 + a) * D + d] = acc[a];
                    }
                }
                const float* sh = gr.S + own * D;
                float q = 0.0f;
                for (int d = lane; d < D; d += 32) q += sh[d] * sh[d];
                q = warp_sum(q);
                const bool h_done = env_done(s_ep[g][own] + 1, p.max_steps);
                for (int d = 2 * lane; d < D; d += 64) {          // D % 4 == 0: d + 1 < D
                    const Philox4 r0 = env_noise(p.env_seed, ctr, i_own, d);
                    const Philox4 r1 = env_noise(p.env_seed, ctr, i_own, d + 1);
                    const float2 gz0 = box_muller(r0.x, r0.y), gz1 = box_muller(r1.x, r1.y);
                    *reinterpret_cast<float2*>(gr.Egx + own * D + d) = make_float2(gz0.x, gz1.x);
                    *reinterpret_cast<float2*>(gr.Erz + own * D + d) =
                        h_done ? make_float2(env_reset_draw(r0), env_reset_draw(r1)) : make_float2(0.0f, 0.0f);
                    if (d == 0) {
                        gr.Eq[2 * own] = q;
                        gr.Eq[2 * own + 1] = gz0.y;
                    }
                }                                             // the action draws come from the layer warps
            }
            rf_bar_sync(2 + g, 2 * 256);                   // own rows of the last hidden layer, then the peers' rows
            rf_mbar_wait(&s_bar[g][1], (unsigned)t & 1u);
            RF_STAMP(9 + 4 * g, 256);
            // ---- head: the 16 k slices of G = 1, two per tail warp; their sums meet in the head slice buffer
            for (int sl = own; sl < 16; sl += RF_OWN) rf_head_slice(p, gr.H2, smem + p.oWh, sl, lane, Hs);
            rf_bar_sync(6, 256);
            RF_STAMP(10 + 4 * g, 256);
            float rew, dn;
            const int slot = rf_act_env<G>(p, gr, t, own, lane, i_own, Hs, Bhs, p.WaT, s_pos[g][own], s_ep[g][own],
                                           s_cnt[g][own], rew, dn);
            commit_actor(i_own < p.N, (int)i_own, lane, 32, gr.Nx + own * D, gr.S + own * D, rew, dn, p.n_step, p.stride,
                         D, A, &s_pos[g][own], slot, p.stage_obs, p.stage_act, p.stage_pd, p.stage_rew, p.stage_done,
                         p.o_obs, p.o_act, p.o_pd, p.o_rew, p.o_done, WarpBarrier());
            RF_STAMP(11 + 4 * g, 256);
            if (t < p.T - 1) {
                rf_push_input(p, gr, own, m_own, i_own, lane, smem_base, peer_base, smem_u32(&s_bar[g][2]) - smem_base);
                rf_bar_arrive(4 + g, 2 * 256);
            }
        }
    }
}

// One group of 32 actors per cluster (G = 1).  Warps 0..7 run the hidden layers, then each finishes owned actor `warp`;
// warps 8..15 do the action-independent half of the env step of owned actor `warp & 7` beside the layers.  The block
// barriers of the step order every hand-off inside the CTA.
__device__ __forceinline__ void rf_one_group(const RfParams& p, unsigned crank, unsigned long long ctr0,
                                             int (&s_pos)[RF_OWN], int (&s_ep)[RF_OWN], int (&s_cnt)[RF_OWN],
                                             uint64_t (&s_bar)[3]) {
    extern __shared__ __align__(16) float smem[];
    const unsigned smem_base = smem_u32(smem);
    unsigned peer_base[RF_CS - 1];
#pragma unroll
    for (int c = 1; c < RF_CS; ++c) peer_base[c - 1] = mapa_u32(smem_base, (crank + (unsigned)c) % RF_CS);
    // (tried: the two roles on swapped warp halves, in case the scheduler's preference for one end of the warp index range
    // starved the layers -- no difference in clock64 traces)
    const int tid = (int)RF_TID, lane = tid & 31, warp = tid >> 5;
    const int D = p.D, H1 = p.H1, H2 = p.H2, A = p.A;
    const int Nc1 = H1 / RF_CS, Nc2 = H2 / RF_CS;
    const int ldwh = p.ldw[2];
    float* Whs = smem + p.oWh;
    float* B1s = smem + p.oB;
    float* B2s = B1s + Nc1;
    float* Bhs = B2s + Nc2;
    float* Part = smem + p.oPart;
    float* EWs = smem + p.oEnv;
    float* EWa = EWs + D * D;
    const RfGroup gr(p, smem, 0);
    const long long row0 = (long long)(blockIdx.x / RF_CS) * RF_ROWS;
    const unsigned bar_off_h1 = smem_u32(&s_bar[0]) - smem_base, bar_off_h2 = smem_u32(&s_bar[1]) - smem_base;
    const unsigned bar_off_x0 = smem_u32(&s_bar[2]) - smem_base;
    // bytes a CTA receives from its three peers per step: their column quarters of hidden layer 1 for all 32 rows, their
    // column quarters of the last hidden layer for the 8 owned rows, their 8 rows of the next input tile
    const unsigned tx_h1 = 3u * RF_ROWS * Nc1 * 4u, tx_h2 = 3u * RF_OWN * Nc2 * 4u, tx_x0 = 3u * RF_OWN * D * 4u;

    const bool math = warp < RF_OWN;                  // warps 0..7: layers, then owner of actor `warp`
    const int own = warp & (RF_OWN - 1);              // owned actor this warp works for (owner or env warp)
    const bool owner = math;
    const int m_own = (int)crank * RF_OWN + own;
    const long long i_own = row0 + m_own;
    const bool valid = owner && (i_own < p.N);

    for (int t = 0; t < p.T; ++t) {
        const unsigned long long ctr = ctr0 + (unsigned long long)t;
        const bool final_step = (t == p.T - 1);
        [[maybe_unused]] const int rf_t = t;          // read by RF_STAMP only
        RF_STAMP(0, 0);
        if (tid == 0) {                                       // arm this step's phases (the previous ones were consumed)
            mbar_arrive_expect_tx(&s_bar[0], tx_h1);
            mbar_arrive_expect_tx(&s_bar[1], tx_h2);
        }
        if (math) {
            if (t > 0) {                                      // the input tile: own rows (math warps wrote them) + the peers' rows
                rf_bar_math();
                rf_mbar_wait(&s_bar[2], (unsigned)(t - 1) & 1u);
            }
            RF_STAMP(18, 0);
            if (tid == 0 && !final_step) mbar_arrive_expect_tx(&s_bar[2], tx_x0);     // next tile's phase: only now is the previous one complete
            rf2_layer1(gr.X0, p.ldx0, D, smem + p.oW1, Nc1, B1s, p.act[0], gr.H1, p.ldh1, (int)crank * Nc1, smem_base, crank,
                       bar_off_h1);
            RF_STAMP(3, 0);
            rf_bar_math();
            rf_mbar_wait(&s_bar[0], (unsigned)t & 1u);
            RF_STAMP(4, 0);
            rf2_layer2_direct(gr.H1, p.ldh1, H1, smem + p.oW2, Nc2, B2s, p.act[1], gr.H2, p.ldh2, (int)crank * Nc2, smem_base,
                              crank, bar_off_h2);
            RF_STAMP(7, 0);
        } else {
            // ---- env warp h: everything of this step that does not depend on the action (the arithmetic of sample_one() /
            // synth_env_block() in rollout.cu), concurrently with the layers
            RF_STAMP(16, 256);
            const int h = own;
            const long long ih = row0 + (int)crank * RF_OWN + h;
            const float* sh = gr.S + h * D;
            float q = 0.0f;
            for (int d = lane; d < D; d += 32) q += sh[d] * sh[d];
            q = warp_sum(q);
            const bool h_done = env_done(s_ep[h] + 1, p.max_steps);
            for (int d = lane; d < D; d += 32) {
                float acc = 0.0f;
#pragma unroll 8
                for (int k = 0; k < D; ++k) acc = fmaf(EWs[k * D + d], sh[k], acc);
                const Philox4 r = env_noise(p.env_seed, ctr, ih, d);
                const float2 gz = box_muller(r.x, r.y);
                gr.Eacc[h * D + d] = acc;
                gr.Egx[h * D + d] = gz.x;
                gr.Erz[h * D + d] = h_done ? env_reset_draw(r) : 0.0f;
                if (d == 0) {
                    gr.Eq[2 * h] = q;
                    gr.Eq[2 * h + 1] = gz.y;
                }
            }
            if (!p.deterministic && lane < A) gr.Zn[h * A + lane] = action_noise1(p.agent_seed, ctr, ih, lane);
            RF_STAMP(17, 256);
        }
        __syncthreads();                                      // last hidden layer: own columns (block barrier) + the peers' columns
        rf_mbar_wait(&s_bar[1], (unsigned)t & 1u);
        // ---- head.  p.head_mode 1: warp w takes k slice w (rf_head_slice); the 16 slice sums meet in the (idle) Part buffer.
        // head_mode 0: warps w and w + 8 take the two k halves of owned actor w & 7.
        if (p.head_mode == 1) {
            rf_head_slice(p, gr.H2, Whs, warp, lane, Part);
        } else {
            const int half = warp >> 3;
            const float* hrow = gr.H2 + own * p.ldh2;
            const int kh = H2 >> 1;
            for (int n8 = 0; n8 < A; n8 += 8) {
                float s8[8];
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) s8[jj] = 0.0f;
                const bool second = (n8 + 4 < ldwh);
                for (int k = half * kh + lane; k < (half + 1) * kh; k += 32) {
                    const float hv = hrow[k];
                    const float* wr = Whs + k * ldwh + n8;
                    const float4 w0 = *reinterpret_cast<const float4*>(wr);
                    s8[0] = fmaf(hv, w0.x, s8[0]); s8[1] = fmaf(hv, w0.y, s8[1]);
                    s8[2] = fmaf(hv, w0.z, s8[2]); s8[3] = fmaf(hv, w0.w, s8[3]);
                    if (second) {
                        const float4 w1 = *reinterpret_cast<const float4*>(wr + 4);
                        s8[4] = fmaf(hv, w1.x, s8[4]); s8[5] = fmaf(hv, w1.y, s8[5]);
                        s8[6] = fmaf(hv, w1.z, s8[6]); s8[7] = fmaf(hv, w1.w, s8[7]);
                    }
                }
                const float v = rf_reduce8(s8, lane);
                const int j = n8 + (((lane >> 4) & 1) << 2) + (((lane >> 3) & 1) << 1) + ((lane >> 2) & 1);
                if ((lane & 3) == 0 && j < A) gr.Hp[(half * RF_OWN + own) * A + j] = v;
            }
        }
        RF_STAMP(9, 0);
        __syncthreads();
        RF_STAMP(10, 0);
        float rew = 0.0f, dn = 0.0f;
        int slot = SLOT_NONE;
        if (owner) slot = rf_act_env<1>(p, gr, t, own, lane, i_own, Part, Bhs, EWa, s_pos[own], s_ep[own], s_cnt[own], rew, dn);
        RF_STAMP(11, 0);
        commit_actor(valid, (int)i_own, lane, 32, gr.Nx + own * D, gr.S + own * D, rew, dn, p.n_step, p.stride, D, A,
                     s_pos + own, slot, p.stage_obs, p.stage_act, p.stage_pd, p.stage_rew, p.stage_done, p.o_obs, p.o_act,
                     p.o_pd, p.o_rew, p.o_done);
        RF_STAMP(12, 0);
        if (owner && !final_step) rf_push_input(p, gr, own, m_own, i_own, lane, smem_base, peer_base, bar_off_x0);
        RF_STAMP(13, 0);
    }
}

template <int G>
__global__ void __cluster_dims__(RF_CS, 1, 1) __launch_bounds__(RF_THREADS, 1)
    ppo_rollout2_kernel(const __grid_constant__ RfParams p) {
    RF_CTA_STAMP(1);
    __shared__ int s_pos[G][RF_OWN], s_ep[G][RF_OWN], s_cnt[G][RF_OWN];
    __shared__ __align__(8) uint64_t s_bar[G][3];   // per group: hidden layer 1 | last hidden layer rows | next input tile
    const unsigned crank = cg::this_cluster().block_rank();
    const unsigned long long ctr0 = rf_setup<G>(p, crank, s_pos, s_ep, s_cnt, s_bar);
    if constexpr (G == 2) rf2_two_groups(p, crank, ctr0, s_pos, s_ep, s_cnt, s_bar);
    else rf_one_group(p, crank, ctr0, s_pos[0], s_ep[0], s_cnt[0], s_bar[0]);
    cg::this_cluster().sync();                                // nobody leaves while a peer may still address its shared memory

    // write-back by the warps that finished the owned actors
    extern __shared__ __align__(16) float smem[];
    const int lane = (int)RF_TID & 31, warp = (int)RF_TID >> 5, own = warp & (RF_OWN - 1);
    if ((warp < RF_OWN) == (G == 1)) {
        for (int g = 0; g < G; ++g) {
            const long long i = (long long)(blockIdx.x / RF_CS) * (G * RF_ROWS) + g * RF_ROWS + (int)crank * RF_OWN + own;
            if (i >= p.N) continue;
            const float* S = smem + p.oS + g * p.gstride + own * p.D;
            for (int d = lane; d < p.D; d += 32) p.state[i * p.D + d] = S[d];
            if (lane == 0) {
                p.stage_pos[i] = s_pos[g][own];
                p.ep_step[i] = s_ep[g][own];
                p.ev_count[i] = s_cnt[g][own];
            }
        }
    }
    RF_CTA_STAMP(2);
}

// ---- post-pass 1 (one block): rank the chunk's window completions in (step, actor) order, give them FIFO slots
// with drop-oldest at capacity (fifo_replay.py:27), advance the queue and the shared step counter.
__global__ void __launch_bounds__(1024) ppo_rollout_rank_kernel(const int* __restrict__ ev_step,
                                                                const int* __restrict__ ev_count, int N, int W, int T,
                                                                int* __restrict__ bitmap, int* __restrict__ base,
                                                                int* __restrict__ ev_slot, FifoState* fifo,
                                                                unsigned long long* step_ctr) {
    const int tid = threadIdx.x, nt = blockDim.x;
    const int words = (N + 31) >> 5;
    __shared__ int s_total;
    for (int x = tid; x < T * words; x += nt) bitmap[x] = 0;
    for (int x = tid; x <= T; x += nt) base[x] = 0;
    __syncthreads();
    for (int e = tid; e < N * W; e += nt) {
        const int i = e / W, w = e - i * W;
        if (w < ev_count[i]) {
            const int t = ev_step[e];
            atomicOr(&bitmap[t * words + (i >> 5)], 1 << (i & 31));
            atomicAdd(&base[t + 1], 1);
        }
    }
    __syncthreads();
    if (tid == 0) {                                   // T is a few hundred at most: a serial prefix is negligible
        int run = 0;
        for (int t = 0; t <= T; ++t) {
            run += base[t];
            base[t] = run;
        }
        s_total = run;
    }
    __syncthreads();
    const int K = s_total;
    const int cap = fifo->capacity, head = fifo->head, count = fifo->count;
    for (int e = tid; e < N * W; e += nt) {
        const int i = e / W, w = e - i * W;
        int out = SLOT_NONE;
        if (w < ev_count[i]) {
            const int t = ev_step[e];
            int r = base[t];
            const int* bm = bitmap + t * words;
            for (int x = 0; x < (i >> 5); ++x) r += __popc(bm[x]);
            r += __popc(bm[i >> 5] & ((1u << (i & 31)) - 1u));
            out = (K > cap && r < K - cap) ? SLOT_DROPPED : (int)(((long long)head + count + r) % cap);
        }
        ev_slot[e] = out;
    }
    __syncthreads();
    if (tid == 0) {
        int nc = count + K, nh = head, dr = 0;
        if (nc > cap) {
            dr = nc - cap;
            nh = (int)(((long long)head + dr) % cap);
            nc = cap;
        }
        fifo->head = nh;
        fifo->count = nc;
        fifo->dropped += dr;
        fifo->total_in += K;
        if (step_ctr != nullptr) *step_ctr += (unsigned long long)T;
    }
}

// ---- post-pass 2: one block per outbox entry, pure copy into the replay ring
__global__ void __launch_bounds__(256) ppo_rollout_copy_kernel(const int* __restrict__ ev_slot, int n_step, int D, int A,
                                                               const float* __restrict__ o_obs,
                                                               const float* __restrict__ o_act,
                                                               const float* __restrict__ o_pd,
                                                               const float* __restrict__ o_rew,
                                                               const float* __restrict__ o_done,
                                                               float* __restrict__ r_obs, float* __restrict__ r_act,
                                                               float* __restrict__ r_pd, float* __restrict__ r_rew,
                                                               float* __restrict__ r_done) {
    const long long e = blockIdx.x;
    const int slot = ev_slot[e];
    if (slot < 0) return;
    const int g = threadIdx.x, G = blockDim.x;
    copy_floats(r_obs + (long long)slot * (n_step + 1) * D, o_obs + e * (n_step + 1) * D, (n_step + 1) * D, g, G);
    copy_floats(r_act + (long long)slot * n_step * A, o_act + e * n_step * A, n_step * A, g, G);
    copy_floats(r_pd + (long long)slot * n_step * 2 * A, o_pd + e * n_step * 2 * A, n_step * 2 * A, g, G);
    copy_floats(r_rew + (long long)slot * n_step, o_rew + e * n_step, n_step, g, G);
    copy_floats(r_done + (long long)slot * n_step, o_done + e * n_step, n_step, g, G);
}

// Shared-memory plan of ppo_rollout2_kernel<G>.  G = 1: weights, the cluster's activation tiles, Part (4 x 32 x
// max(Nc1, Nc2) floats: the head's slice sums, whose fit decides head_mode), the env matrices and the owned actors'
// state.  G = 2: no Part, the env matrices stay in global memory (read through L1 by the tail warps, off the layers'
// path), a 4 KB head slice buffer, and the per-group tiles and state twice, `gstride` floats apart.  At the configs[1]
// shape [64, 256, 256, 8]: G = 1 204 512 B, G = 2 219 552 B.
bool rf_plan(const sb200_mlp* net, int D, int A, int G, RfParams* p, size_t* smem_bytes) {
    if (net == nullptr || net->n_layers != 3 || net->aux_layer >= 0 || sb200_mlp_has_ln(net)) return false;
    const int H1 = net->dims[1], H2 = net->dims[2];
    if (net->dims[0] != D || net->dims[3] != A) return false;
    if (D % 4 != 0 || D > 128 || A < 1 || A > 32 || H1 % 16 != 0 || H2 % 16 != 0) return false;
    const int Nc1 = H1 / RF_CS, Nc2 = H2 / RF_CS, ldwh = net->ldw[2];
    long long off = 0;
    auto take = [&](long long n) { const long long o = off; off += (n + 3) / 4 * 4; return (int)o; };
    const int oW1 = take((long long)D * Nc1), oW2 = take((long long)H1 * Nc2), oWh = take((long long)H2 * ldwh);
    const int oB = take(Nc1 + Nc2 + ldwh);
    const int ldx0 = D + 4, ldh1 = H1 + 4, ldh2 = H2 + 4;
    int oX0, oH1, oH2, oPart = -1, oZf, oEnv = -1, oS, oNext, oAct, oPre, oHs = -1, gstride = 0;
    // Act: actions | N(0,1) draws of odd steps (G = 2; unused with one group) | std | N(0,1) draws | two head halves
    if (G == 1) {
        oX0 = take(RF_ROWS * ldx0); oH1 = take(RF_ROWS * ldh1); oH2 = take(RF_OWN * ldh2);
        oPart = take(4LL * RF_ROWS * (Nc1 > Nc2 ? Nc1 : Nc2));
        oZf = take(2 * D); oEnv = take((long long)D * D + A * D);
        oS = take(RF_OWN * D); oNext = take(RF_OWN * D); oAct = take(6 * RF_OWN * A);
        oPre = take(3 * RF_OWN * D + 2 * RF_OWN);
    } else {
        oZf = take(2 * D);
        oHs = take(16LL * RF_OWN * ldwh);
        const long long g0 = off;
        oX0 = take(RF_ROWS * ldx0); oH1 = take(RF_ROWS * ldh1); oH2 = take(RF_OWN * ldh2);
        oS = take(RF_OWN * D); oNext = take(RF_OWN * D); oAct = take(6 * RF_OWN * A);
        oPre = take(3 * RF_OWN * D + 2 * RF_OWN);
        gstride = (int)(off - g0);
        off += (long long)(G - 1) * gstride;
    }
    if ((size_t)off * sizeof(float) > 224 * 1024) return false;
    if (p != nullptr) {
        p->oW1 = oW1; p->oW2 = oW2; p->oWh = oWh; p->oB = oB; p->oX0 = oX0; p->oH1 = oH1; p->oH2 = oH2; p->oPart = oPart;
        p->oZf = oZf; p->oEnv = oEnv; p->oS = oS; p->oNext = oNext; p->oAct = oAct; p->oPre = oPre;
        p->oHs = oHs; p->gstride = gstride;
        p->ldx0 = ldx0; p->ldh1 = ldh1; p->ldh2 = ldh2;
        p->D = D; p->H1 = H1; p->H2 = H2; p->A = A;
    }
    if (smem_bytes != nullptr) *smem_bytes = (size_t)off * sizeof(float);
    return true;
}

template <int G>
cudaError_t rf_query_clusters(size_t smem, int* n) {
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = RF_CS;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cfg.gridDim = dim3(RF_CS);
    cfg.blockDim = dim3(RF_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    // without the opt-in to > 48 KB of dynamic shared memory the answer is 0 clusters (and it is cached): set it here too,
    // so that a query made before sb200_init() is right
    const cudaError_t e = cudaFuncSetAttribute(ppo_rollout2_kernel<G>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024);
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveClusters(n, ppo_rollout2_kernel<G>, &cfg);
}

// How many 4-CTA clusters of ppo_rollout2_kernel<G> with `smem` dynamic bytes the current device runs at once.
// A cluster must sit inside one GPC, and an H100's GPCs have uneven SM counts, so this is below SMs / 4 (30 on an H100
// SXM with 132 SMs at the configs[1] plan).  Queried once per (device, G, bytes).
int rf_max_clusters(int G, size_t smem, int* n_out) {
    struct Entry { int dev, G; size_t smem; int n; };
    static std::mutex mu;
    static Entry cache[16];
    static int n_cache = 0;
    int dev = 0;
    SB200_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(mu);
    for (int i = 0; i < n_cache; ++i)
        if (cache[i].dev == dev && cache[i].G == G && cache[i].smem == smem) {
            *n_out = cache[i].n;
            return SB200_OK;
        }
    int n = 0;
    SB200_CUDA(G == 2 ? rf_query_clusters<2>(smem, &n) : rf_query_clusters<1>(smem, &n));
    if (n_cache < 16) cache[n_cache++] = Entry{dev, G, smem, n};
    *n_out = n;
    return SB200_OK;
}

// Launch shape of a chunk: groups per cluster, CTAs, and whether they are all resident at once.
struct RfShape {
    int groups;
    long long ctas;
    bool one_wave;                    // known to run in one wave
};

// `p` / `smem` hold the G = 1 plan of rf_plan on entry; on return the plan of the chosen shape (head_mode set).
int rf_shape(const sb200_ppo_rollout* a, RfParams* p, size_t* smem, RfShape* sh) {
    const long long clusters = ((long long)a->N + RF_ROWS - 1) / RF_ROWS;
    // head_mode 1 when the slice sums fit: 16 warps x 8 actors x ldw[2] floats of the Part buffer (4 x 32 x max(Nc1, Nc2))
    p->head_mode = (16 * RF_OWN * a->net->ldw[2] <= 4 * RF_ROWS * std::max(a->net->dims[1], a->net->dims[2]) / RF_CS) ? 1 : 0;
    // Two groups of 32 actors per cluster when the device cannot hold all ceil(N / 32) one-group clusters at once (the
    // clusters that do not fit run as a whole further wave of the chunk) AND two groups at least halve the number of
    // waves: a two-group step does both groups' work, 1.74x the time of a one-group step at the configs[1] shape on an
    // H100 (38 K vs 22 K cycles), so fewer waves pay only when they are at most half as many (1024 actors: 2 -> 1
    // wave; 4096 actors: 5 -> 3 waves would be slower).  Same results as one group: same arithmetic (head_mode 1,
    // rf2_layer2_direct).
    int groups = 1, fit1 = 0, fit2 = 0;
    const int rc1 = rf_max_clusters(1, *smem, &fit1);
    if (rc1 != SB200_OK) return rc1;
    RfParams p2 = *p;
    size_t smem2 = 0;
    if (p->head_mode == 1 && rf_plan(a->net, a->D, a->A, 2, &p2, &smem2)) {
        const int rc = rf_max_clusters(2, smem2, &fit2);
        if (rc != SB200_OK) return rc;
        if (fit1 >= 1 && fit2 >= 1 && clusters > fit1) {
            const long long waves1 = (clusters + fit1 - 1) / fit1, waves2 = ((clusters + 1) / 2 + fit2 - 1) / fit2;
            if (2 * waves2 <= waves1) {
                groups = 2;
                *p = p2;
                *smem = smem2;
            }
        }
    }
    const long long launched = (clusters + groups - 1) / groups;
    sh->groups = groups;
    sh->ctas = launched * RF_CS;
    sh->one_wave = launched <= (groups == 2 ? fit2 : fit1);
    return SB200_OK;
}

}  // namespace

int sb200_rollout_fused_init() {
    SB200_CUDA(cudaFuncSetAttribute(ppo_rollout2_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
    SB200_CUDA(cudaFuncSetAttribute(ppo_rollout2_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
    return SB200_OK;
}

#ifdef RF_TRACE
static unsigned g_rf_last_grid = 0;
static size_t g_rf_last_smem = 0;
static int g_rf_last_groups = 0;

extern "C" int sb200_debug_rf_trace(long long* host_out) {
    SB200_CUDA(cudaDeviceSynchronize());
    SB200_CUDA(cudaMemcpyFromSymbol(host_out, g_rf_trace, sizeof(g_rf_trace)));
    return SB200_OK;
}

// per-CTA [smid, entry ns, exit ns] of the last persistent launch (RF_TR_CTAS rows); info = {grid CTAs, dynamic shared
// bytes, groups per cluster G, cudaOccupancyMaxActiveClusters of ppo_rollout2_kernel<G> at that configuration}
extern "C" int sb200_debug_rf_ctas(long long* host_out, long long* info) {
    SB200_CUDA(cudaDeviceSynchronize());
    SB200_CUDA(cudaMemcpyFromSymbol(host_out, g_rf_cta, sizeof(g_rf_cta)));
    int n = 0;
    const int rc = rf_max_clusters(g_rf_last_groups, g_rf_last_smem, &n);
    if (rc != SB200_OK) return rc;
    info[0] = g_rf_last_grid;
    info[1] = (long long)g_rf_last_smem;
    info[2] = g_rf_last_groups;
    info[3] = n;
    return SB200_OK;
}
#endif

// the chunk's staging descriptor is complete and describes the same N actors and record shape
static bool rollout_windows_ok(const sb200_ppo_rollout* a) {
    const sb200_windows* w = a->windows;
    return windows_ok(w) && w->N == a->N && w->D == a->D && w->A == a->A;
}

extern "C" int sb200_ppo_rollout_supported(const sb200_mlp* net, int D, int A) {
    return rf_plan(net, D, A, 1, nullptr, nullptr) ? 1 : 0;
}

extern "C" size_t sb200_ppo_rollout_scratch_ints(int N, int W, int T) {
    // bitmap [T][ceil(N/32)] | base [T+1] | ev_slot [N*W]
    return (size_t)T * ((N + 31) / 32) + (size_t)(T + 1) + (size_t)N * W;
}

extern "C" int sb200_ppo_rollout_f32(const sb200_ppo_rollout* a, void* stream) {
    SB200_REQUIRE(a != nullptr && a->net != nullptr);
    RfParams p;
    size_t smem = 0;
    if (!rf_plan(a->net, a->D, a->A, 1, &p, &smem)) return SB200_ERR_UNSUPPORTED;
    SB200_REQUIRE(a->N >= 1 && a->T >= 1 && a->W >= 1 && rollout_windows_ok(a) && rollout_env_ok(a));
    const sb200_env* e = a->env;
    SB200_REQUIRE(e->state && e->WsT && e->WaT && e->ep_step && a->action && a->pd && e->obs_next && e->reward && e->done);
    SB200_REQUIRE(a->log_var);
    SB200_REQUIRE(a->o_obs && a->o_act && a->o_pd && a->o_rew && a->o_done && a->ev_step && a->ev_count);
    for (int l = 0; l < 3; ++l) {
        p.W[l] = a->net->W[l];
        p.b[l] = a->net->b[l];
        p.ldw[l] = a->net->ldw[l];
        p.act[l] = a->net->act[l];
        SB200_REQUIRE(p.W[l] != nullptr && p.b[l] != nullptr && p.ldw[l] % 4 == 0 && (((uintptr_t)p.W[l]) & 15) == 0);
    }
    SB200_REQUIRE((((uintptr_t)e->WsT) & 15) == 0 && (((uintptr_t)e->WaT) & 15) == 0 && (((uintptr_t)e->state) & 15) == 0);
    p.zf = a->zf_stats;
    p.zf_eps = a->zf_eps;
    p.log_var = a->log_var;
    p.log_noise = a->log_noise;
    p.agent_seed = a->agent_seed;
    p.deterministic = a->deterministic;
    p.state = (float*)e->state;
    p.WsT = e->WsT;
    p.WaT = e->WaT;
    p.ep_step = e->ep_step;
    p.max_steps = e->max_steps;
    p.env_seed = e->seed;
    p.action = a->action;
    p.pd = a->pd;
    p.obs_next = (float*)e->obs_next;
    p.reward = e->reward;
    p.done = e->done;
    const sb200_windows* w = a->windows;
    p.stage_pos = w->stage_pos;
    p.stage_obs = w->stage_obs;
    p.stage_act = w->stage_act;
    p.stage_pd = w->stage_pd;
    p.stage_rew = w->stage_rew;
    p.stage_done = w->stage_done;
    p.o_obs = a->o_obs;
    p.o_act = a->o_act;
    p.o_pd = a->o_pd;
    p.o_rew = a->o_rew;
    p.o_done = a->o_done;
    p.ev_step = a->ev_step;
    p.ev_count = a->ev_count;
    p.Wout = a->W;
    p.N = a->N;
    p.n_step = w->n_step;
    p.stride = w->stride;
    p.T = a->T;
    p.step_ctr = (const unsigned long long*)w->step_counter;
    RfShape sh;
    const int rc = rf_shape(a, &p, &smem, &sh);
    if (rc != SB200_OK) return rc;
    const int groups = sh.groups;
    const long long ctas = sh.ctas;
#ifdef RF_TRACE
    g_rf_last_grid = (unsigned)ctas;
    g_rf_last_smem = smem;
    g_rf_last_groups = groups;
#endif
    if (groups == 2) ppo_rollout2_kernel<2><<<(unsigned)ctas, RF_THREADS, smem, (cudaStream_t)stream>>>(p);
    else ppo_rollout2_kernel<1><<<(unsigned)ctas, RF_THREADS, smem, (cudaStream_t)stream>>>(p);
    return sb200_launch_status();
}

extern "C" int sb200_ppo_rollout_footprint(const sb200_ppo_rollout* a, int* sms) {
    SB200_REQUIRE(a != nullptr && a->net != nullptr && sms != nullptr && a->N >= 1 && rollout_env_ok(a));
    *sms = 0;
    RfParams p;
    size_t smem = 0;
    if (!rf_plan(a->net, a->D, a->A, 1, &p, &smem)) return SB200_ERR_UNSUPPORTED;
    RfShape sh;
    const int rc = rf_shape(a, &p, &smem, &sh);
    if (rc != SB200_OK) return rc;
    if (sh.one_wave) *sms = (int)sh.ctas;             // > 200 KB of shared memory per CTA: one CTA per SM
    return SB200_OK;
}

extern "C" int sb200_ppo_rollout_commit_f32(const sb200_ppo_rollout* a, int* scratch, void* stream) {
    SB200_REQUIRE(a != nullptr && scratch != nullptr && rollout_windows_ok(a) && a->windows->step_counter);
    SB200_REQUIRE(a->N >= 1 && a->T >= 1 && a->W >= 1 && a->ev_step && a->ev_count);
    const sb200_windows* w = a->windows;
    const int words = (a->N + 31) / 32;
    int* bitmap = scratch;
    int* base = bitmap + (size_t)a->T * words;
    int* ev_slot = base + (a->T + 1);
    cudaStream_t st = (cudaStream_t)stream;
    ppo_rollout_rank_kernel<<<1, 1024, 0, st>>>(a->ev_step, a->ev_count, a->N, a->W, a->T, bitmap, base, ev_slot,
                                                (FifoState*)w->fifo_state, (unsigned long long*)w->step_counter);
    ppo_rollout_copy_kernel<<<(unsigned)((long long)a->N * a->W), 256, 0, st>>>(
        ev_slot, w->n_step, a->D, a->A, a->o_obs, a->o_act, a->o_pd, a->o_rew, a->o_done, w->r_obs, w->r_act, w->r_pd,
        w->r_rew, w->r_done);
    return sb200_launch_status(2);
}
