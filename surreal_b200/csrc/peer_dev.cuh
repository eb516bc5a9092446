// The NVLink peer-exchange protocol of the data-parallel learner, shared by the stand-alone all-reduce (peer_allreduce.cu)
// and the persistent learner kernel (epoch2.cu): the layout of every rank's symmetric buffer, the system-scope loads and
// stores, the publish-and-wait step of one slice, and the host-side check of an sb200_par.
#pragma once
#include "common.cuh"

namespace peer_dev {

constexpr int PAR_MAX_WORLD = 8;
constexpr int PAR_MAX_CTAS = 16;
static_assert(sizeof(sb200_par::peers) == PAR_MAX_WORLD * sizeof(void*), "one sb200_par.peers entry per rank");

struct ParHeader {                       // at the start of every rank's symmetric buffer
    unsigned int flags[PAR_MAX_WORLD * PAR_MAX_CTAS];   // flags[p * PAR_MAX_CTAS + b]: last call whose slice b rank p published
    unsigned int counter;                // calls completed by THIS rank
    unsigned int ticket;
    unsigned int pad[2];
    double partial[PAR_MAX_CTAS];
};

// Kernels read only peers[0, world); the entries past it are never dereferenced.
__device__ __forceinline__ ParHeader* header_of(const sb200_par& c, int p) { return reinterpret_cast<ParHeader*>(c.peers[p]); }

// rank p's slot of call parity `parity` (two slots of max_floats floats follow the header)
__device__ __forceinline__ float* slot_of(const sb200_par& c, int p, unsigned int parity) {
    return reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(c.peers[p]) + sizeof(ParHeader)) +
           (size_t)parity * (size_t)c.max_floats;
}

__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float ld_sys1(const float* p) {
    float r;
    asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(r) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ float4 ld_sys4(const float* p) {
    float4 r;
    asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ double ld_sys_f64(const double* p) {
    double r;
    asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(r) : "l"(p) : "memory");
    return r;
}

// Block-wide: once this rank's slice b of call k is in its own slot and fenced (__threadfence_system), publish
// "slice b of call k is ready" to every peer (system-scope release), then wait until every peer has published the same
// (acquire).  Afterwards the whole block may read slice b of call k from every rank's slot.  me = header_of(c, c.rank).
__device__ __forceinline__ void publish_and_wait(const sb200_par& c, ParHeader* me, int b, unsigned int k) {
    const int tid = threadIdx.x;
    __syncthreads();
    if (tid < c.world && tid != c.rank) {
        st_release_sys(&header_of(c, tid)->flags[c.rank * PAR_MAX_CTAS + b], k);
        const unsigned int* f = &me->flags[tid * PAR_MAX_CTAS + b];
        while ((int)(ld_acquire_sys(f) - k) < 0) { }
    }
    __syncthreads();
}

}  // namespace peer_dev

// Can `c` carry an exchange of `floats` floats: 1 <= world <= 8, 0 <= rank < world, a buffer for every rank, and slots of
// at least `floats` floats.
static inline int sb200_par_check(const sb200_par* c, long long floats) {
    SB200_REQUIRE(c != nullptr && c->world >= 1 && c->world <= peer_dev::PAR_MAX_WORLD && c->rank >= 0 && c->rank < c->world);
    SB200_REQUIRE(floats <= c->max_floats);
    for (int p = 0; p < c->world; ++p) SB200_REQUIRE(c->peers[p] != nullptr);
    return SB200_OK;
}
