// Library-level entry points of libsurreal_b200.
#include "common.cuh"

unsigned long long g_sb200_launches = 0;

extern "C" int sb200_version(void) { return 101; }

extern "C" uint64_t sb200_launch_counter(int reset) {
    const unsigned long long v = g_sb200_launches;
    if (reset) g_sb200_launches = 0;
    return (uint64_t)v;
}

extern "C" const char* sb200_status_string(int status) {
    switch (status) {
        case SB200_OK: return "ok";
        case SB200_ERR_ARG: return "invalid argument";
        case SB200_ERR_CUDA: return "CUDA error";
        case SB200_ERR_UNSUPPORTED: return "unsupported configuration";
        default: return "unknown status";
    }
}

int sb200_mlp_fwd_init();
int sb200_gae_init();
int sb200_rollout_fused_init();
int sb200_mlp_tc5_init();
int sb200_stem_init();
int sb200_epochs2_init();

extern "C" void sb200_launch_counter_add(uint64_t kernels) { g_sb200_launches += kernels; }

extern "C" int sb200_init(void) {
    int dev = 0;
    SB200_CUDA(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    SB200_CUDA(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0) {
        fprintf(stderr, "[surreal_b200] built for sm_90a (H100); found compute capability %d.%d\n", prop.major, prop.minor);
        return SB200_ERR_UNSUPPORTED;
    }
    int rc = sb200_mlp_fwd_init();
    if (rc != SB200_OK) return rc;
    rc = sb200_gae_init();
    if (rc != SB200_OK) return rc;
    rc = sb200_mlp_tc5_init();
    if (rc != SB200_OK) return rc;
    rc = sb200_stem_init();
    if (rc != SB200_OK) return rc;
    rc = sb200_epochs2_init();
    if (rc != SB200_OK) return rc;
    return sb200_rollout_fused_init();
}

extern "C" int sb200_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    SB200_CUDA(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    SB200_CUDA(cudaGetDeviceProperties(&prop, dev));
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    return SB200_OK;
}
