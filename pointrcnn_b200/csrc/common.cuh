// common.cuh -- shared helpers for libpointrcnn_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/pointrcnn_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libpointrcnn_b200 is written for sm_90a (H100) only"
#endif

namespace prb {

// error plumbing: nothing in this library exits the process (the reference's launchers do)
void set_error(const char *fmt, ...);
void count_launch(int n = 1);

inline int check_launch(const char *what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return (int)e;
    }
    count_launch();
    return 0;
}

#define PRB_REQUIRE(cond, ...)                 \
    do {                                       \
        if (!(cond)) {                         \
            prb::set_error(__VA_ARGS__);       \
            return -1;                         \
        }                                      \
    } while (0)

#define PRB_CUDA(call)                                                        \
    do {                                                                      \
        cudaError_t e__ = (call);                                             \
        if (e__ != cudaSuccess) {                                             \
            prb::set_error("%s: %s", #call, cudaGetErrorString(e__));         \
            return (int)e__;                                                  \
        }                                                                     \
    } while (0)

__host__ __device__ constexpr int ceil_div(int a, int b) { return (a + b - 1) / b; }

// The squared distance of the three reference distance kernels, in the contraction order their
// SASS shows (FMUL(dy,dy) -> FFMA(dx,dx,.) -> FFMA(dz,dz,.)).  Explicit intrinsics so the
// optimiser cannot pick another order: FPS / ball-query / three_nn indices depend on it.
__device__ __forceinline__ float dist2_ref(float dx, float dy, float dz) {
    return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
}

// counter-based random draws (kitti_io.cu's npoints draw, rcnn_sample.cu): a 32-bit hash of (seed, scene, i, salt)
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}
__device__ __forceinline__ uint32_t draw_key(uint32_t seed, uint32_t scene, uint32_t i, uint32_t salt) {
    return mix32(mix32(seed ^ (scene * 0x9e3779b9u) ^ salt) + i * 0x85ebca6bu);
}

int num_sms();   // SM count of the CURRENT device (cached per device)

// per-thread tuning block (include/pointrcnn_b200.h: prb_options).  Environment variables seed the DEFAULTS once,
// when the library is loaded; no entry point reads the environment per call, and a thread (e.g. a DataParallel
// worker) that sets its own options never disturbs another.
const prb_options &opts();

}  // namespace prb
