// Device-side pieces of the HBM replay that more than one translation unit needs: the uniform ring's control block, the
// sampling view and sampler blocks, and the one-warp gather of a record's fields (replay.cu: uniform sampler;
// replay_per.cu: prioritized sampler).
#pragma once
#include "common.cuh"

struct UniformState {
    long long next_idx;
    long long size;
    long long capacity;
    long long total_in;
};

// Draw r of the view is ring slot (start + r) % capacity.
struct UniformView {
    long long start;
    long long count;
    long long capacity;
};

struct UniformSampler {
    unsigned long long draw_counter;
    int status;              // 1: the last launch found an empty view and sampled nothing
    unsigned int ticket;
};

// All fields of a record in ONE launch: out_f[b] = src_f[idx[b]] for f < nf.  A warp owns a record; its lanes walk the
// record's chunks across fields (16-byte chunks for fields whose record size / alignment allow, 4-byte otherwise), so a
// 552-byte SSAR record (obs 64, obs_next 64, action 8, reward 1, done 1 floats) is two loads + two stores per lane.
constexpr int GATHER_MAX_FIELDS = 8;
struct GatherFields {
    const float* src[GATHER_MAX_FIELDS];
    float* out[GATHER_MAX_FIELDS];
    long long rec[GATHER_MAX_FIELDS];     // floats per record
    int unit[GATHER_MAX_FIELDS];          // 4 (float4 chunks) or 1
    int chunk_end[GATHER_MAX_FIELDS];     // prefix sums of chunks per record
    int nf;
};

// record `s` of every field -> batch row `b`, by the 32 lanes of one warp
__device__ __forceinline__ void gather_record(const GatherFields& f, long long s, long long b, int lane) {
    const int total = f.chunk_end[f.nf - 1];
    for (int c = lane; c < total; c += 32) {
        int q = 0;
#pragma unroll
        for (int k = 0; k < GATHER_MAX_FIELDS - 1; ++k) q += (k < f.nf - 1 && c >= f.chunk_end[k]) ? 1 : 0;
        const int local = c - (q > 0 ? f.chunk_end[q - 1] : 0);
        if (f.unit[q] == 4) {
            reinterpret_cast<float4*>(f.out[q] + b * f.rec[q])[local] = ld_stream4(f.src[q] + s * f.rec[q] + 4 * local);
        } else {
            f.out[q][b * f.rec[q] + local] = __ldg(f.src[q] + s * f.rec[q] + local);
        }
    }
}

// Field table of the multi-field gathers from the caller's HOST arrays; false when an entry is unusable.
static inline bool gather_fields_ok(const float* const* srcs, float* const* outs, const int64_t* record_floats,
                                    int nfields, GatherFields* f) {
    if (!srcs || !outs || !record_floats || nfields < 1 || nfields > GATHER_MAX_FIELDS) return false;
    int end = 0;
    for (int k = 0; k < nfields; ++k) {
        if (!srcs[k] || !outs[k] || record_floats[k] < 1 || record_floats[k] >= (1ll << 28)) return false;
        f->src[k] = srcs[k];
        f->out[k] = outs[k];
        f->rec[k] = record_floats[k];
        const bool vec = (record_floats[k] % 4 == 0) && ((((uintptr_t)srcs[k]) | ((uintptr_t)outs[k])) & 15) == 0;
        f->unit[k] = vec ? 4 : 1;
        end += (int)(record_floats[k] / f->unit[k]);
        f->chunk_end[k] = end;
    }
    for (int k = nfields; k < GATHER_MAX_FIELDS; ++k) { f->src[k] = nullptr; f->out[k] = nullptr; f->rec[k] = 0; f->unit[k] = 1; f->chunk_end[k] = end; }
    f->nf = nfields;
    return true;
}
