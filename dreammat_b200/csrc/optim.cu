// optim.cu -- the optimizer of the ControlNet training step (controlnet_train/diffusers_train_controlnet.py:
// accelerator.clip_grad_norm_(params, max_grad_norm); torch.optim.AdamW.step()) over flat buffers:
//   dm_grad_sumsq     squared L2 norm of the flat fp32 gradient arena (deterministic two-pass reduction)
//   dm_adamw_prepare  one thread: device-resident optimizer state -> the scalars of this step (clip factor, bias corrections)
//   dm_adamw_step     AdamW on fp32 master weights, the updated weight written a second time in the 16-bit storage type
// Everything that changes from step to step (lr, the step counter, the gradient norm) is read from device memory, so a
// captured CUDA graph of the step stays valid for the whole run.  HBM-bound streaming kernels: 16-byte vector accesses,
// grid a multiple of the SM count, programmatic dependent launch.
#include <cuda_bf16.h>
#include <math.h>
#include "common.cuh"

namespace {

constexpr int OPT_THREADS = 256;

inline int opt_grid(int64_t work) {
    const int64_t b = dm_ceil_div(work, OPT_THREADS), cap = (int64_t)DM_NUM_SMS * 8;
    return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

// threads of a block added in a fixed order: lanes by the shuffle tree, then warps 0..7 by thread 0
__device__ __forceinline__ float block_sum_ordered(float acc) {
    __shared__ float red[OPT_THREADS / 32];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    float s = 0.f;
    if (threadIdx.x == 0)
        for (int w = 0; w < OPT_THREADS / 32; ++w) s += red[w];
    return s;      // valid in thread 0
}

// part[block] = sum of g[i]^2 over the block's share of the grid-stride loop.  The grid is a function of n alone, so the
// partition, and with it every partial sum, is the same from call to call.
__global__ void __launch_bounds__(OPT_THREADS) grad_sumsq_kernel(const float* __restrict__ g, int64_t n,
                                                                 float* __restrict__ part) {
    griddep_launch_dependents();
    griddep_wait();
    const int64_t n4 = n / 4, stride = (int64_t)gridDim.x * blockDim.x, t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    float acc = 0.f;
    for (int64_t i = t0; i < n4; i += stride) {
        const float4 v = g4[i];
        acc += v.x * v.x; acc += v.y * v.y; acc += v.z * v.z; acc += v.w * v.w;
    }
    if (t0 < n - 4 * n4) { const float v = g[4 * n4 + t0]; acc += v * v; }
    const float s = block_sum_ordered(acc);
    if (threadIdx.x == 0) part[blockIdx.x] = s;
}

// the per-block sums added in block order (each thread its strided share in order, then the fixed block order)
__global__ void __launch_bounds__(OPT_THREADS) grad_sumsq_finish_kernel(const float* __restrict__ part, int nblk,
                                                                        float* __restrict__ sumsq) {
    griddep_launch_dependents();
    griddep_wait();
    float acc = 0.f;
    for (int b = threadIdx.x; b < nblk; b += blockDim.x) acc += part[b];
    const float s = block_sum_ordered(acc);
    if (threadIdx.x == 0) *sumsq = s;
}

__global__ void adamw_prepare_kernel(const float* __restrict__ sumsq, dm_adamw_state* __restrict__ st, double beta1, double beta2,
                                     float max_grad_norm, float inv_grad_scale) {
    griddep_launch_dependents();
    griddep_wait();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const float norm = sqrtf(*sumsq) * inv_grad_scale;         // of the unscaled gradient, as clip_grad_norm_ returns it
    st->grad_norm = norm;
    if (!isfinite(norm)) {       // GradScaler semantics: an overflowed step is dropped, the moments and the counter stay
        st->skip = 1;
        st->skipped_steps += 1;
        return;
    }
    const int t = st->step + 1;
    st->step = t;
    st->skip = 0;
    st->gmul = inv_grad_scale * fminf(1.0f, max_grad_norm / (norm + 1e-6f));
    const double bc1 = 1.0 - pow(beta1, (double)t), bc2 = 1.0 - pow(beta2, (double)t);
    st->step_size = (float)((double)st->lr / bc1);
    st->inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
}

template <typename T> __device__ __forceinline__ T to_storage(float v);
template <> __device__ __forceinline__ __half to_storage<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 to_storage<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

struct AdamwK {
    float w1, b2, w2, eps, decay, gmul, step_size, inv_sqrt_bc2;      // w = 1 - beta, decay = 1 - lr * weight_decay
    // torch.optim.AdamW (single-tensor path): p *= 1 - lr*wd; m = lerp(m, g, 1-b1); v = b2 v + (1-b2) g^2;
    // p -= step_size * m / (sqrt(v) / sqrt(bc2) + eps).  A padded element (p = g = m = v = 0) stays exactly 0.
    __device__ __forceinline__ float operator()(float p, float g, float& m, float& v) const {
        g *= gmul;
        m = m + (g - m) * w1;
        v = b2 * v + w2 * g * g;
        const float denom = sqrtf(v) * inv_sqrt_bc2 + eps;
        return p * decay - step_size * (m / denom);
    }
};

// a thread owns 8 consecutive parameters per iteration: two float4 of each fp32 arena, one 16-byte store of the 16-bit copy
template <typename T>
__global__ void __launch_bounds__(OPT_THREADS) adamw_kernel(float* __restrict__ master, float* __restrict__ m, float* __restrict__ v,
                                                            const float* __restrict__ g, T* __restrict__ w16, int64_t n,
                                                            const dm_adamw_state* __restrict__ st, float w1, float beta2,
                                                            float w2, float eps, float weight_decay) {
    griddep_launch_dependents();
    griddep_wait();
    if (st->skip) return;
    AdamwK k;
    k.w1 = w1; k.b2 = beta2; k.w2 = w2; k.eps = eps; k.decay = 1.0f - st->lr * weight_decay;
    k.gmul = st->gmul; k.step_size = st->step_size; k.inv_sqrt_bc2 = st->inv_sqrt_bc2;
    const int64_t n8 = n / 8, stride = (int64_t)gridDim.x * blockDim.x, t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (int64_t i = t0; i < n8; i += stride) {
        float4 P[2], M[2], V[2], G[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            P[h] = reinterpret_cast<const float4*>(master)[2 * i + h];
            G[h] = reinterpret_cast<const float4*>(g)[2 * i + h];
            M[h] = reinterpret_cast<const float4*>(m)[2 * i + h];
            V[h] = reinterpret_cast<const float4*>(v)[2 * i + h];
        }
        uint4 o; T* oh = reinterpret_cast<T*>(&o);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            P[h].x = k(P[h].x, G[h].x, M[h].x, V[h].x); P[h].y = k(P[h].y, G[h].y, M[h].y, V[h].y);
            P[h].z = k(P[h].z, G[h].z, M[h].z, V[h].z); P[h].w = k(P[h].w, G[h].w, M[h].w, V[h].w);
            oh[4 * h + 0] = to_storage<T>(P[h].x); oh[4 * h + 1] = to_storage<T>(P[h].y);
            oh[4 * h + 2] = to_storage<T>(P[h].z); oh[4 * h + 3] = to_storage<T>(P[h].w);
            reinterpret_cast<float4*>(master)[2 * i + h] = P[h];
            reinterpret_cast<float4*>(m)[2 * i + h] = M[h];
            reinterpret_cast<float4*>(v)[2 * i + h] = V[h];
        }
        reinterpret_cast<uint4*>(w16)[i] = o;
    }
    if (t0 < n - 8 * n8) {       // up to 7 trailing parameters
        const int64_t j = 8 * n8 + t0;
        float mm = m[j], vv = v[j];
        const float p = k(master[j], g[j], mm, vv);
        master[j] = p; m[j] = mm; v[j] = vv; w16[j] = to_storage<T>(p);
    }
}

inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

extern "C" int dm_grad_sumsq(const float* g, int64_t n, float* sumsq, void* stream) {
    DM_REQUIRE(g && sumsq, "null pointer");
    DM_REQUIRE(n > 0, "n >= 1");
    DM_REQUIRE(aligned16(g) && ((uintptr_t)sumsq & 3) == 0, "g 16-byte aligned, sumsq 4-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const int nblk = opt_grid(dm_ceil_div(n, 4));
    float* part = (float*)dm_scratch(DM_SCRATCH_AFFINE, (size_t)nblk * sizeof(float), st);
    if (!part) return DM_EDRIVER;
    DM_CHECK_CUDA(dm_launch(grad_sumsq_kernel, dim3((unsigned)nblk), dim3(OPT_THREADS), 0, st, g, n, part));
    DM_CHECK_LAUNCH();
    DM_CHECK_CUDA(dm_launch(grad_sumsq_finish_kernel, dim3(1), dim3(OPT_THREADS), 0, st, (const float*)part, nblk, sumsq));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_adamw_prepare(const float* sumsq, dm_adamw_state* state, double beta1, double beta2, float max_grad_norm,
                                float inv_grad_scale, void* stream) {
    DM_REQUIRE(sumsq && state, "null pointer");
    DM_REQUIRE(((uintptr_t)sumsq & 3) == 0 && ((uintptr_t)state & 3) == 0, "4-byte aligned operands");
    DM_REQUIRE(beta1 >= 0. && beta1 < 1. && beta2 >= 0. && beta2 < 1., "betas in [0, 1)");
    DM_REQUIRE(max_grad_norm >= 0.f, "max_grad_norm >= 0 (INFINITY: no clipping)");
    DM_REQUIRE(inv_grad_scale > 0.f && inv_grad_scale <= 3.0e38f, "inv_grad_scale positive and finite");
    DM_CHECK_CUDA(dm_launch(adamw_prepare_kernel, dim3(1), dim3(32), 0, (cudaStream_t)stream, sumsq, state, beta1, beta2,
                            max_grad_norm, inv_grad_scale));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_adamw_step(int bf16, float* master, float* m, float* v, const float* g, void* w16, int64_t n,
                             const dm_adamw_state* state, double beta1, double beta2, float eps, float weight_decay,
                             void* stream) {
    DM_REQUIRE(bf16 == 0 || bf16 == 1, "dtype selector of the 16-bit copy: 0 fp16, 1 bf16");
    DM_REQUIRE(master && m && v && g && w16 && state, "null pointer");
    DM_REQUIRE(n > 0, "n >= 1");
    DM_REQUIRE(aligned16(master) && aligned16(m) && aligned16(v) && aligned16(g) && aligned16(w16) && ((uintptr_t)state & 3) == 0,
               "arenas 16-byte aligned, state 4-byte aligned");
    DM_REQUIRE(beta1 >= 0. && beta1 < 1. && beta2 >= 0. && beta2 < 1., "betas in [0, 1)");
    DM_REQUIRE(eps >= 0.f && weight_decay >= 0.f, "eps, weight_decay >= 0");
    cudaStream_t st = (cudaStream_t)stream;
    const float w1 = (float)(1.0 - beta1), w2 = (float)(1.0 - beta2);     // rounded once from double, as torch's scalars are
    const unsigned grid = (unsigned)opt_grid(dm_ceil_div(n, 8));
    if (bf16)
        DM_CHECK_CUDA(dm_launch(adamw_kernel<__nv_bfloat16>, dim3(grid), dim3(OPT_THREADS), 0, st, master, m, v, g,
                                (__nv_bfloat16*)w16, n, state, w1, (float)beta2, w2, eps, weight_decay));
    else
        DM_CHECK_CUDA(dm_launch(adamw_kernel<__half>, dim3(grid), dim3(OPT_THREADS), 0, st, master, m, v, g, (__half*)w16, n,
                                state, w1, (float)beta2, w2, eps, weight_decay));
    DM_CHECK_LAUNCH();
    return DM_OK;
}
