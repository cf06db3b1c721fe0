// common.cuh -- shared helpers for the dreammat_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/dreammat_b200.h"

#ifndef DM_NUM_SMS
#define DM_NUM_SMS 132   // H100 SXM
#endif

void dm_set_error(const char* fmt, ...);
void dm_count_launch();

// Library-owned device scratch of the deterministic reductions (GroupNorm partial rows, the hash-grid backward's fixed-point
// accumulator, the bias-gradient partial rows of the weight gradients): one buffer per device and slot, zero-filled when
// allocated.  Callers of one device must not use a slot from two streams at once (the same rule as the split-K workspace).
// A buffer is never freed, because a captured CUDA graph may hold its address; it can only grow outside stream capture (a
// warm-up call before capture sizes it).  Returns nullptr with the error set on failure.
enum { DM_SCRATCH_GN = 0, DM_SCRATCH_HASHGRID = 1, DM_SCRATCH_AA = 2, DM_SCRATCH_WGRAD = 3, DM_SCRATCH_SLOTS = 4 };
void* dm_scratch(int slot, size_t bytes, cudaStream_t st);

#define DM_CHECK_CUDA(expr)                                                          \
    do {                                                                             \
        cudaError_t _e = (expr);                                                     \
        if (_e != cudaSuccess) {                                                     \
            dm_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return (int)_e;                                                          \
        }                                                                            \
    } while (0)

// ---- programmatic dependent launch (PDL).  Kernels of the dense section call griddep_launch_dependents() first
// thing (the next kernel of the stream may then be scheduled as SM resources free up and run its prologue: barrier
// init, tensor-map prefetch) and griddep_wait() before touching global memory written by earlier
// kernels (it returns once every prerequisite grid has completed and flushed).  Both are no-ops for launches without
// the attribute, so correctness never depends on the knob (dm_tune "pdl").
extern int g_dm_pdl;
#ifdef __CUDACC__
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t dm_launch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = g_dm_pdl ? at : nullptr;
    cfg.numAttrs = g_dm_pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
#endif

#define DM_CHECK_LAUNCH()                                                            \
    do {                                                                             \
        dm_count_launch();                                                           \
        cudaError_t _e = cudaGetLastError();                                         \
        if (_e != cudaSuccess) {                                                     \
            dm_set_error("%s:%d launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
            return (int)_e;                                                          \
        }                                                                            \
    } while (0)

#define DM_REQUIRE(cond, msg)                                                        \
    do {                                                                             \
        if (!(cond)) {                                                               \
            dm_set_error("%s:%d requirement failed: %s (%s)", __FILE__, __LINE__, #cond, msg); \
            return DM_EINVAL;                                                        \
        }                                                                            \
    } while (0)

static inline int64_t dm_ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

struct f3 {
    float x, y, z;
};
__host__ __device__ __forceinline__ f3 mk3(float x, float y, float z) { f3 r; r.x = x; r.y = y; r.z = z; return r; }
__host__ __device__ __forceinline__ f3 operator+(f3 a, f3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
__host__ __device__ __forceinline__ f3 operator-(f3 a, f3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
__host__ __device__ __forceinline__ f3 operator*(f3 a, float s) { return mk3(a.x * s, a.y * s, a.z * s); }
__host__ __device__ __forceinline__ f3 operator*(float s, f3 a) { return mk3(a.x * s, a.y * s, a.z * s); }
__host__ __device__ __forceinline__ float dot3(f3 a, f3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__host__ __device__ __forceinline__ f3 cross3(f3 a, f3 b) {
    return mk3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
__device__ __forceinline__ f3 ld3(const float* p, int64_t i) { return mk3(p[3 * i], p[3 * i + 1], p[3 * i + 2]); }
__device__ __forceinline__ void st3(float* p, int64_t i, f3 v) { p[3 * i] = v.x; p[3 * i + 1] = v.y; p[3 * i + 2] = v.z; }

// F.normalize(v, dim=-1): v / max(||v||, 1e-12)
__device__ __forceinline__ f3 normalize3(f3 v) {
    float l = sqrtf(dot3(v, v));
    float inv = 1.0f / fmaxf(l, 1e-12f);
    return v * inv;
}

// get_orthogonal_directions (dreammat_material.py:542-552, raytracing_renderer.py:306-316)
__device__ __forceinline__ f3 ortho_dir(f3 d) {
    f3 o0 = mk3(d.y, -d.x, 0.0f);
    f3 o1 = mk3(-d.z, 0.0f, d.x);
    float n0 = sqrtf(dot3(o0, o0)), n1 = sqrtf(dot3(o1, o1));
    f3 o = (n0 > n1) ? o0 : o1;
    return normalize3(o);
}

__device__ __forceinline__ float lin2srgb_f(float x) {
    float r = (x > 0.0031308f) ? (powf(fmaxf(x, 0.0031308f), 1.0f / 2.4f) * 1.055f - 0.055f) : 12.92f * x;
    return fminf(fmaxf(r, 0.0f), 1.0f);
}
// derivative of lin2srgb (torch autograd semantics: where() routes grad, clamp passes at boundaries)
__device__ __forceinline__ float lin2srgb_grad(float x) {
    float r, g;
    if (x > 0.0031308f) {
        float xc = fmaxf(x, 0.0031308f);
        r = powf(xc, 1.0f / 2.4f) * 1.055f - 0.055f;
        g = 1.055f * (1.0f / 2.4f) * powf(xc, 1.0f / 2.4f - 1.0f);
    } else {
        r = 12.92f * x;
        g = 12.92f;
    }
    return (r >= 0.0f && r <= 1.0f) ? g : 0.0f;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
