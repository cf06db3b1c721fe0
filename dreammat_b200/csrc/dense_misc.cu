// dense_misc.cu -- the non-GEMM kernels of the VAE-encoder / UNet / ControlNet path (rows a7, a8):
// GroupNorm(+SiLU) forward/backward, LayerNorm, GEGLU and their backward (with the norms' affine gradients), nearest 2x
// upsample, strided copies,
// transposes, row softmax forward/backward, layout / dtype conversion at the fp32 boundaries,
// posterior sampling, add_noise and the sinusoidal timestep embedding.
// NHWC activations, fp16 or bf16 storage, fp32 math.  All are HBM-bound streaming kernels:
// 16-byte vector accesses, grid sized in multiples of the SM count for the strided loops.
//
// Reference call sites (diffusers modules reached from models/guidance/dreammat_guidance.py:218-292):
// torch.nn.GroupNorm/SiLU in ResnetBlock2D, LayerNorm + GEGLU in BasicTransformerBlock,
// Upsample2D (nearest), AutoencoderKL DiagonalGaussianDistribution.sample (:291),
// DDIMScheduler.add_noise (:463), Timesteps / get_timestep_embedding.
#include <cuda_bf16.h>
#include "common.cuh"
#include "dense_hp.cuh"

namespace {

template <typename T> struct H;
template <> struct H<__half> {
    static __device__ __forceinline__ float f(__half v) { return __half2float(v); }
    static __device__ __forceinline__ __half t(float v) { return __float2half_rn(v); }
};
template <> struct H<__nv_bfloat16> {
    static __device__ __forceinline__ float f(__nv_bfloat16 v) { return __bfloat162float(v); }
    static __device__ __forceinline__ __nv_bfloat16 t(float v) { return __float2bfloat16_rn(v); }
};

template <> struct H<float> {
    static __device__ __forceinline__ float f(float v) { return v; }
    static __device__ __forceinline__ float t(float v) { return v; }
};

// storage dtype selector of every dense-path entry point: 0 fp16, 1 bf16, 2 fp32 (high-precision mode, dense_hp.cu)
#define DM_DISPATCH_T(bf16, ...)                                  \
    do {                                                          \
        if (bf16) { using T = __nv_bfloat16; __VA_ARGS__; }       \
        else { using T = __half; __VA_ARGS__; }                   \
    } while (0)
// element-wise kernels (no 16-bit vector packing) also run on fp32 storage
#define DM_DISPATCH_T3(dt, ...)                                   \
    do {                                                          \
        if ((dt) == 2) { using T = float; __VA_ARGS__; }          \
        else if (dt) { using T = __nv_bfloat16; __VA_ARGS__; }    \
        else { using T = __half; __VA_ARGS__; }                   \
    } while (0)
#define DM_DTYPE_OK(dt) DM_REQUIRE((dt) >= 0 && (dt) <= 2, "dtype selector: 0 fp16, 1 bf16, 2 fp32")

__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
__device__ __forceinline__ float silu_grad(float x) {
    float s = __fdividef(1.0f, 1.0f + __expf(-x));
    return s * (1.0f + x * (1.0f - s));
}

// ----------------------------------------------------------------------------------- GroupNorm
// Thread mapping shared by the four kernels: the channel axis is cut into slabs of `vslab` 8-channel vectors
// (vslab = largest divisor of C/8 that is <= 32, i.e. 512 contiguous bytes per pixel), grid = (pixel chunks,
// images, slabs).  A thread owns ONE vector of the slab and strides over the chunk's pixels with `lanes` =
// blockDim / vslab pixel lanes, so per-channel constants live in registers and the loop body is pure
// load / FMA / store with several 16-byte loads in flight.  Small feature maps (8x8 .. 32x32 latents) get their
// parallelism from the slab axis instead of idling most of the machine.
struct GnIdx {
    int v, q, lanes, p0, p1;
    bool active;
};
__device__ __forceinline__ GnIdx gn_index(int HW, int vslab, int chunks) {
    GnIdx m;
    m.lanes = (int)blockDim.x / vslab;
    m.q = (int)threadIdx.x / vslab;
    m.v = (int)blockIdx.z * vslab + (int)threadIdx.x % vslab;
    m.active = m.q < m.lanes;
    const int px_per_chunk = (HW + chunks - 1) / chunks;
    m.p0 = (int)blockIdx.x * px_per_chunk;
    m.p1 = min(HW, m.p0 + px_per_chunk);
    return m;
}

// Deterministic statistics: every block reduces its threads' NV per-group sums in a fixed order (no shared- or
// global-memory float atomics) and stores them in its own row of the partials (library scratch):
// partial[((img*slabs + slab)*chunks + chunk)*NV*G + NV*g + which].  gn_moments_kernel (forward, NV = 4) / gn_finish_kernel
// (backward, NV = 2) then add the rows of each group in (slab, chunk) order, so the statistics are bit-identical from run to run.
template <int NV>
__device__ __forceinline__ void gn_block_partials(const float (&a)[NV][4], bool active, int vslab, int cpg, int G, int chunks,
                                                  float* __restrict__ part) {
    __shared__ float red[256][4 * NV];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int w = 0; w < NV; ++w) red[threadIdx.x][NV * j + w] = active ? a[w][j] : 0.f;
    __syncthreads();
    const int img = blockIdx.y, slabs = gridDim.z;
    const int g0 = (8 * (int)blockIdx.z * vslab) / cpg, g1 = (8 * ((int)blockIdx.z + 1) * vslab - 1) / cpg;
    float* row = part + (((int64_t)img * slabs + blockIdx.z) * chunks + blockIdx.x) * NV * G;
    for (int i = threadIdx.x; i < NV * (g1 - g0 + 1); i += blockDim.x) {
        const int g = g0 + i / NV, which = i % NV;
        // threads t = q * vslab + (v - slab start) hold channel vector v; the group's vectors are [vlo, vhi] within this slab
        const int zb = (int)blockIdx.z * vslab;
        const int vlo = max((g * cpg) / 8, zb), vhi = min(((g + 1) * cpg - 1) / 8, zb + vslab - 1);
        float acc = 0.f;
        for (int q = 0; q < (int)blockDim.x / vslab; ++q)
            for (int v = vlo; v <= vhi; ++v) {
                const int t = q * vslab + (v - zb);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int c = 8 * v + 2 * j;         // channel pair c, c + 1 (pairs never straddle a group)
                    if (c >= g * cpg && c < (g + 1) * cpg) acc += red[t][NV * j + which];
                }
            }
        row[NV * g + which] = acc;
    }
}

// entry i = (img*G + g)*NV + which of the per-group sums: the partial rows of group g added in (slab, chunk) order
template <int NV>
__device__ __forceinline__ float gn_partial_sum(const float* __restrict__ part, int i, int C, int G, int vslab, int slabs,
                                                int chunks) {
    const int img = i / (NV * G), r = i - img * NV * G, g = r / NV, cpg = C / G;
    const int z0 = ((g * cpg) / 8) / vslab, z1 = (((g + 1) * cpg - 1) / 8) / vslab;
    float acc = 0.f;
    for (int z = z0; z <= z1; ++z)
        for (int c = 0; c < chunks; ++c) acc += part[(((int64_t)img * slabs + z) * chunks + c) * NV * G + r];
    return acc;
}

__global__ void __launch_bounds__(256) gn_finish_kernel(int n_img, int C, int G, int vslab, int slabs, int chunks,
                                                        const float* __restrict__ part, float* __restrict__ stats) {
    griddep_launch_dependents();
    griddep_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_img * G * 2) return;
    stats[i] = gn_partial_sum<2>(part, i, C, G, vslab, slabs, chunks);
}

// The one-pass variance E[x^2] - mean^2 from fp32 (sum, sumsq) loses precision as (mean / std)^2: measured on a 512x512x4
// group, the fp16 output error is 1.04x the rounding floor at |mean| = 10 std and 26x at 100 std.  So the forward also sums
// x - K about a pivot K per (image, group), the group's element at pixel 0, channel g*cpg; about a value drawn from the group
// itself the cancellation is only that of (mean - K) / std.
template <typename T>
__device__ __forceinline__ float gn_pivot(const T* __restrict__ x, int img, int HW, int ld, int g, int cpg) {
    return H<T>::f(x[(int64_t)img * HW * ld + g * cpg]);
}

// stats[(img*G + g)*2 + {0,1}] = (mean, rstd), the same meaning as in the fp32 mode (hp_groupnorm).  Where |mean| <= 8 std
// (fp16 output error within ~1.02x the rounding floor) they come from the plain (sum, sumsq) by the one-pass formula
// mean = S/cnt, var = fma(SS, 1/cnt, -mean^2), written with explicit roundings so the result does not depend on how the
// compiler contracts it; beyond that from the pivoted sums.  The partial rows are [sum, sumsq, sum about K, sumsq about K].
template <typename T>
__global__ void __launch_bounds__(256) gn_moments_kernel(int n_img, int HW, int C, int ld, int G, int vslab, int slabs,
                                                         int chunks, const float* __restrict__ part, const T* __restrict__ x,
                                                         float eps, float* __restrict__ stats) {
    griddep_launch_dependents();
    griddep_wait();
    // one thread per sum, as in gn_finish_kernel (the row loop is latency-bound: one serial chain per thread); the first lane
    // of each group of four takes the other three sums by shuffle.  Every lane of a warp reaches the shuffles.
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = i < n_img * G * 4;
    const float s = valid ? gn_partial_sum<4>(part, i, C, G, vslab, slabs, chunks) : 0.f;
    const float ss = __shfl_down_sync(0xffffffffu, s, 1);
    const float sk = __shfl_down_sync(0xffffffffu, s, 2);
    const float ssk = __shfl_down_sync(0xffffffffu, s, 3);
    if (!valid || (i & 3)) return;
    const int img = i / (4 * G), g = (i - img * 4 * G) >> 2, cpg = C / G;
    const float inv_cnt = 1.0f / ((float)HW * (float)cpg);
    const float d = sk * inv_cnt, var_k = fmaxf(ssk * inv_cnt - d * d, 0.f), mean_k = gn_pivot(x, img, HW, ld, g, cpg) + d;
    float* o = stats + ((int64_t)img * G + g) * 2;
    if (mean_k * mean_k > 64.f * var_k) {
        o[0] = mean_k;
        o[1] = rsqrtf(var_k + eps);
    } else {
        const float mean = __fmul_rn(s, inv_cnt);
        o[0] = mean;
        o[1] = rsqrtf(fmaxf(__fmaf_rn(ss, inv_cnt, -__fmul_rn(mean, mean)), 0.f) + eps);
    }
}

// Per-thread (sum, sumsq) and (sum, sumsq) about the pivot over the group's channels: this kernel writes the chunk's partial
// row.  Channel PAIRS never straddle a group (cpg is even for every SD layer), so each thread keeps 4 of each.
template <typename T>
__global__ void __launch_bounds__(256) gn_stats_kernel(const T* __restrict__ x, int HW, int C, int ld, int G,
                                                       int chunks, int vslab, float* __restrict__ part) {
    const int img = blockIdx.y, cpg = C / G;
    griddep_launch_dependents();
    griddep_wait();
    const GnIdx m = gn_index(HW, vslab, chunks);
    float acc4[4][4] = {};    // [sum, sumsq, sum about K, sumsq about K][channel pair]
    if (m.active) {
        const T* base = x + ((int64_t)img * HW) * ld + 8 * m.v;
        const int lanes = m.lanes;
        float K[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) K[j] = gn_pivot(x, img, HW, ld, (8 * m.v + 2 * j) / cpg, cpg);
        auto acc = [&](const uint4& u) {
            const T* h = reinterpret_cast<const T*>(&u);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float a = H<T>::f(h[2 * j]), b = H<T>::f(h[2 * j + 1]);
                acc4[0][j] += a + b; acc4[1][j] += a * a + b * b;
                float ak = a - K[j], bk = b - K[j];
                acc4[2][j] += ak + bk; acc4[3][j] += ak * ak + bk * bk;
            }
        };
        int p = m.p0 + m.q;
        for (; p + 3 * lanes < m.p1; p += 4 * lanes) {
            uint4 u[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) u[k] = *reinterpret_cast<const uint4*>(base + (int64_t)(p + k * lanes) * ld);
#pragma unroll
            for (int k = 0; k < 4; ++k) acc(u[k]);
        }
        for (; p < m.p1; p += lanes) acc(*reinterpret_cast<const uint4*>(base + (int64_t)p * ld));
    }
    gn_block_partials<4>(acc4, m.active, vslab, cpg, G, chunks, part);
}

// y = act(x * A[c] + B[c]) with A = rstd*gamma, B = beta - mean*rstd*gamma (16 registers per thread).
template <typename T>
__global__ void __launch_bounds__(256) gn_apply_kernel(const T* __restrict__ x, int HW, int C, int ld, int ldy, int G,
                                                       int chunks, int vslab, const float* __restrict__ stats,
                                                       const T* __restrict__ gamma, const T* __restrict__ beta,
                                                       int silu, T* __restrict__ y) {
    griddep_launch_dependents();
    griddep_wait();
    const int img = blockIdx.y, cpg = C / G;
    const GnIdx m = gn_index(HW, vslab, chunks);
    if (!m.active) return;
    const int v = m.v, lanes = m.lanes;
    float A[8], Bc[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        int g = (8 * v + 2 * j) / cpg;
        float mean = stats[((int64_t)img * G + g) * 2], rstd = stats[((int64_t)img * G + g) * 2 + 1];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            float gm = H<T>::f(gamma[8 * v + 2 * j + k]);
            A[2 * j + k] = rstd * gm;
            Bc[2 * j + k] = H<T>::f(beta[8 * v + 2 * j + k]) - mean * rstd * gm;
        }
    }
    const T* xb = x + ((int64_t)img * HW) * ld + 8 * v;
    T* yb = y + ((int64_t)img * HW) * ldy + 8 * v;
    auto body = [&](uint4 u, int p) {
        const T* h = reinterpret_cast<const T*>(&u);
        uint4 o; T* oh = reinterpret_cast<T*>(&o);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float val = fmaf(H<T>::f(h[k]), A[k], Bc[k]);
            if (silu) val = silu_f(val);
            oh[k] = H<T>::t(val);
        }
        *reinterpret_cast<uint4*>(yb + (int64_t)p * ldy) = o;
    };
    int p = m.p0 + m.q;
    for (; p + 3 * lanes < m.p1; p += 4 * lanes) {
        uint4 u[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) u[k] = *reinterpret_cast<const uint4*>(xb + (int64_t)(p + k * lanes) * ld);
#pragma unroll
        for (int k = 0; k < 4; ++k) body(u[k], p + k * lanes);
    }
    for (; p < m.p1; p += lanes) body(*reinterpret_cast<const uint4*>(xb + (int64_t)p * ld), p);
}

// backward pass 1: bstats[(img*G+g)*2] = sum(gamma*dy'), sum(gamma*dy'*xhat), dy' = dz * act'(y) (partial rows, as above)
template <typename T>
__global__ void __launch_bounds__(256) gn_bwd_stats_kernel(const T* __restrict__ x, const T* __restrict__ dz, int HW,
                                                           int C, int G, int chunks, int vslab,
                                                           const float* __restrict__ stats, const T* __restrict__ gamma,
                                                           const T* __restrict__ beta, int silu,
                                                           float* __restrict__ part) {
    griddep_launch_dependents();
    const int img = blockIdx.y, cpg = C / G;
    griddep_wait();
    const GnIdx m = gn_index(HW, vslab, chunks);
    float a12[2][4] = {};   // [sum(gamma*dy'), sum(gamma*dy'*xhat)][channel pair]
    if (m.active) {
        const int v = m.v, lanes = m.lanes;
        // xhat*gamma + beta = x*A + Bc;  xhat = x*rs + ms
        float A[8], Bc[8], gm[8], rs[4], ms[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int g = (8 * v + 2 * j) / cpg;
            float mean = stats[((int64_t)img * G + g) * 2];
            rs[j] = stats[((int64_t)img * G + g) * 2 + 1];
            ms[j] = -mean * rs[j];
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            gm[k] = H<T>::f(gamma[8 * v + k]);
            A[k] = rs[k >> 1] * gm[k];
            Bc[k] = H<T>::f(beta[8 * v + k]) + ms[k >> 1] * gm[k];
        }
        const int64_t base = ((int64_t)img * HW) * C + 8 * v;
        auto acc = [&](const uint4& ux, const uint4& ud) {
            const T* hx = reinterpret_cast<const T*>(&ux); const T* hd = reinterpret_cast<const T*>(&ud);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                float xv = H<T>::f(hx[k]);
                float d = H<T>::f(hd[k]) * gm[k];
                if (silu) d *= silu_grad(fmaf(xv, A[k], Bc[k]));
                a12[0][k >> 1] += d;
                a12[1][k >> 1] = fmaf(d, fmaf(xv, rs[k >> 1], ms[k >> 1]), a12[1][k >> 1]);
            }
        };
        int p = m.p0 + m.q;
        for (; p + lanes < m.p1; p += 2 * lanes) {
            uint4 ux0 = *reinterpret_cast<const uint4*>(x + base + (int64_t)p * C);
            uint4 ud0 = *reinterpret_cast<const uint4*>(dz + base + (int64_t)p * C);
            uint4 ux1 = *reinterpret_cast<const uint4*>(x + base + (int64_t)(p + lanes) * C);
            uint4 ud1 = *reinterpret_cast<const uint4*>(dz + base + (int64_t)(p + lanes) * C);
            acc(ux0, ud0); acc(ux1, ud1);
        }
        for (; p < m.p1; p += lanes)
            acc(*reinterpret_cast<const uint4*>(x + base + (int64_t)p * C), *reinterpret_cast<const uint4*>(dz + base + (int64_t)p * C));
    }
    gn_block_partials<2>(a12, m.active, vslab, cpg, G, chunks, part);
}

// backward pass 2: dx = rstd * (gamma*dy' - (S1 + xhat*S2)/cnt)  (+ dx_add if given); same mapping as gn_apply
template <typename T>
__global__ void __launch_bounds__(256) gn_bwd_apply_kernel(const T* __restrict__ x, const T* __restrict__ dz, int HW,
                                                           int C, int G, int chunks, int vslab,
                                                           const float* __restrict__ stats, const float* __restrict__ bstats,
                                                           const T* __restrict__ gamma, const T* __restrict__ beta,
                                                           int silu, const T* __restrict__ dx_add,
                                                           T* __restrict__ dx) {
    griddep_launch_dependents();
    griddep_wait();
    const int img = blockIdx.y, cpg = C / G;
    const float inv_cnt = 1.0f / ((float)HW * (float)cpg);
    const GnIdx m = gn_index(HW, vslab, chunks);
    if (!m.active) return;
    const int v = m.v, lanes = m.lanes;
    // act'(y) needs y = x*A + Bc (A = rs*gm, Bc = beta + ms*gm, ms = -mean*rs); with xhat = x*rs + ms
    // dx = rs*(gm*d' - S1 - xhat*S2) = d'*A - (x*P + Q),  P = rs^2*S2,  Q = rs*(S1 + ms*S2)
    float A[8], Bc[8], rs[4], ms[4], Pq[4], Qq[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        int g = (8 * v + 2 * j) / cpg;
        int64_t si = ((int64_t)img * G + g) * 2;
        float mean = stats[si];
        rs[j] = stats[si + 1];
        ms[j] = -mean * rs[j];
        float S1 = bstats[si] * inv_cnt, S2 = bstats[si + 1] * inv_cnt;
        Pq[j] = rs[j] * rs[j] * S2;
        Qq[j] = rs[j] * (S1 + ms[j] * S2);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        float gm = H<T>::f(gamma[8 * v + k]);
        A[k] = rs[k >> 1] * gm;
        Bc[k] = H<T>::f(beta[8 * v + k]) + ms[k >> 1] * gm;
    }
    const int64_t base = ((int64_t)img * HW) * C + 8 * v;
    auto body = [&](const uint4& ux, const uint4& ud, const uint4& ua, int64_t off) {
        const T* hx = reinterpret_cast<const T*>(&ux); const T* hd = reinterpret_cast<const T*>(&ud);
        const T* ha = reinterpret_cast<const T*>(&ua);
        uint4 o; T* oh = reinterpret_cast<T*>(&o);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float xv = H<T>::f(hx[k]);
            float d = H<T>::f(hd[k]);
            if (silu) d *= silu_grad(fmaf(xv, A[k], Bc[k]));
            float val = fmaf(d, A[k], -fmaf(xv, Pq[k >> 1], Qq[k >> 1]));
            if (dx_add) val += H<T>::f(ha[k]);
            oh[k] = H<T>::t(val);
        }
        *reinterpret_cast<uint4*>(dx + off) = o;
    };
    const uint4 zero = make_uint4(0, 0, 0, 0);
    int p = m.p0 + m.q;
    for (; p + lanes < m.p1; p += 2 * lanes) {
        const int64_t o0 = base + (int64_t)p * C, o1 = base + (int64_t)(p + lanes) * C;
        uint4 ux0 = *reinterpret_cast<const uint4*>(x + o0), ud0 = *reinterpret_cast<const uint4*>(dz + o0);
        uint4 ux1 = *reinterpret_cast<const uint4*>(x + o1), ud1 = *reinterpret_cast<const uint4*>(dz + o1);
        uint4 ua0 = dx_add ? *reinterpret_cast<const uint4*>(dx_add + o0) : zero;
        uint4 ua1 = dx_add ? *reinterpret_cast<const uint4*>(dx_add + o1) : zero;
        body(ux0, ud0, ua0, o0); body(ux1, ud1, ua1, o1);
    }
    for (; p < m.p1; p += lanes) {
        const int64_t o0 = base + (int64_t)p * C;
        body(*reinterpret_cast<const uint4*>(x + o0), *reinterpret_cast<const uint4*>(dz + o0),
             dx_add ? *reinterpret_cast<const uint4*>(dx_add + o0) : zero, o0);
    }
}

// ----------------------------------------------------------------------------------- LayerNorm (warp per row)
template <typename T>
__global__ void __launch_bounds__(256) layernorm_kernel(const T* __restrict__ x, int64_t M, int C,
                                                        const T* __restrict__ gamma, const T* __restrict__ beta,
                                                        float eps, T* __restrict__ y) {
    // warp per row, 16-byte vectors (C % 8 == 0, C <= 1280 -> at most 5 vectors per lane kept in registers);
    // two-pass mean / centred variance on the register copy
    griddep_launch_dependents();
    griddep_wait();
    int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= M) return;
    const int lane = threadIdx.x & 31, nv = C >> 3;
    const T* xr = x + row * C;
    float vals[40];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        const int v = lane + 32 * k;
        if (v < nv) {
            uint4 u = *reinterpret_cast<const uint4*>(xr + 8 * v);
            const T* h = reinterpret_cast<const T*>(&u);
#pragma unroll
            for (int j = 0; j < 8; ++j) { float f = H<T>::f(h[j]); vals[8 * k + j] = f; s += f; }
        }
    }
    s = warp_sum(s);
    const float mean = s / (float)C;
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        if (lane + 32 * k < nv) {
#pragma unroll
            for (int j = 0; j < 8; ++j) { float d = vals[8 * k + j] - mean; ss += d * d; }
        }
    }
    ss = warp_sum(ss);
    const float rstd = rsqrtf(ss / (float)C + eps);
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        const int v = lane + 32 * k;
        if (v < nv) {
            uint4 ug = *reinterpret_cast<const uint4*>(gamma + 8 * v), ub = *reinterpret_cast<const uint4*>(beta + 8 * v);
            const T* hg = reinterpret_cast<const T*>(&ug); const T* hb = reinterpret_cast<const T*>(&ub);
            uint4 o; T* oh = reinterpret_cast<T*>(&o);
#pragma unroll
            for (int j = 0; j < 8; ++j) oh[j] = H<T>::t((vals[8 * k + j] - mean) * rstd * H<T>::f(hg[j]) + H<T>::f(hb[j]));
            *reinterpret_cast<uint4*>(y + row * C + 8 * v) = o;
        }
    }
}

// GEGLU: out[m, j] = h[m, j] * gelu(h[m, D + j])   (diffusers GEGLU: hidden, gate = chunk(2); hidden * gelu(gate))
template <typename T>
__global__ void __launch_bounds__(256) geglu_kernel(const T* __restrict__ h, int64_t M, int D, T* __restrict__ out) {
    int64_t n = M * (int64_t)(D / 8);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t m = i / (D / 8); int j = (int)(i - m * (D / 8)) * 8;
        uint4 a = *reinterpret_cast<const uint4*>(h + m * 2 * D + j), g = *reinterpret_cast<const uint4*>(h + m * 2 * D + D + j);
        const T* ha = reinterpret_cast<const T*>(&a); const T* hg = reinterpret_cast<const T*>(&g);
        uint4 o; T* oh = reinterpret_cast<T*>(&o);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float gv = H<T>::f(hg[k]);
            oh[k] = H<T>::t(H<T>::f(ha[k]) * (0.5f * gv * (1.0f + erff(gv * 0.70710678118654752f))));
        }
        *reinterpret_cast<uint4*>(out + m * D + j) = o;
    }
}

// nearest-neighbour 2x upsample, NHWC
template <typename T>
__global__ void __launch_bounds__(256) upsample2x_kernel(const T* __restrict__ x, int n, int Hh, int W, int C,
                                                         T* __restrict__ y) {
    int64_t nv = (int64_t)n * 2 * Hh * 2 * W * (C / 8);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (int64_t)gridDim.x * blockDim.x) {
        int c = (int)(i % (C / 8)); int64_t r = i / (C / 8);
        int xo = (int)(r % (2 * W)); r /= 2 * W; int yo = (int)(r % (2 * Hh)); int img = (int)(r / (2 * Hh));
        const uint4* src = reinterpret_cast<const uint4*>(x + (((int64_t)img * Hh + yo / 2) * W + xo / 2) * C) + c;
        reinterpret_cast<uint4*>(y)[i] = *src;
    }
}

// zero-insertion 2x (transpose of a stride-2 gather): y[2i,2j] = x[i,j], else 0
template <typename T>
__global__ void __launch_bounds__(256) zero_insert2x_kernel(const T* __restrict__ x, int n, int Hh, int W, int C,
                                                            T* __restrict__ y) {
    int64_t nv = (int64_t)n * 2 * Hh * 2 * W * (C / 8);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (int64_t)gridDim.x * blockDim.x) {
        int c = (int)(i % (C / 8)); int64_t r = i / (C / 8);
        int xo = (int)(r % (2 * W)); r /= 2 * W; int yo = (int)(r % (2 * Hh)); int img = (int)(r / (2 * Hh));
        uint4 v = make_uint4(0, 0, 0, 0);
        if (((xo | yo) & 1) == 0) v = reinterpret_cast<const uint4*>(x + (((int64_t)img * Hh + yo / 2) * W + xo / 2) * C)[c];
        reinterpret_cast<uint4*>(y)[i] = v;
    }
}

// dst[r, 0:cols] = a*src[r, 0:cols] (+ b*src2[r,0:cols]) with independent row strides (16-byte vectors)
template <typename T>
__global__ void __launch_bounds__(256) axpby2d_kernel(const T* __restrict__ s1, int64_t ld1, float a,
                                                      const T* __restrict__ s2, int64_t ld2, float b, int64_t rows,
                                                      int cols, T* __restrict__ dst, int64_t ldd) {
    int vpr = cols / 8;
    int64_t nv = rows * vpr;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = i / vpr; int c = (int)(i - r * vpr) * 8;
        uint4 u = *reinterpret_cast<const uint4*>(s1 + r * ld1 + c);
        if (!s2 && a == 1.0f) { *reinterpret_cast<uint4*>(dst + r * ldd + c) = u; continue; }
        uint4 w = make_uint4(0, 0, 0, 0);
        if (s2) w = *reinterpret_cast<const uint4*>(s2 + r * ld2 + c);
        const T* hu = reinterpret_cast<const T*>(&u); const T* hw = reinterpret_cast<const T*>(&w);
        uint4 o; T* oh = reinterpret_cast<T*>(&o);
#pragma unroll
        for (int k = 0; k < 8; ++k) oh[k] = H<T>::t(a * H<T>::f(hu[k]) + (s2 ? b * H<T>::f(hw[k]) : 0.f));
        *reinterpret_cast<uint4*>(dst + r * ldd + c) = o;
    }
}

// batched transpose [B, R, C] -> [B, C, R] through a 32x33 shared tile
template <typename T>
__global__ void __launch_bounds__(256) transpose_kernel(const T* __restrict__ x, int R, int C, int64_t ldx,
                                                        int64_t bsx, T* __restrict__ y, int64_t ldy, int64_t bsy) {
    // 64 x 64 tile of 16-bit elements moved as 32-bit pairs on both sides (128-byte warp requests): the load packs two
    // neighbouring columns, the store two neighbouring rows of the input.  Even R, C, ld (checked on the host).
    __shared__ uint32_t tile[64][33];     // [row][column pair]
    const T* xb = x + (int64_t)blockIdx.z * bsx; T* yb = y + (int64_t)blockIdx.z * bsy;
    const int c0 = blockIdx.x * 64, r0 = blockIdx.y * 64;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int j = ty; j < 64; j += 8) {
        int r = r0 + j, c = c0 + 2 * tx;
        uint32_t v = 0;
        if (r < R && c < C) v = *reinterpret_cast<const uint32_t*>(xb + (int64_t)r * ldx + c);
        tile[j][tx] = v;
    }
    __syncthreads();
    for (int j = ty; j < 64; j += 8) {       // output row c0 + j holds input column c0 + j; this thread writes rows r0+2tx, +1
        int c = c0 + j, r = r0 + 2 * tx;
        if (c < C && r < R) {
            uint32_t lo = tile[2 * tx][j >> 1], hi = tile[2 * tx + 1][j >> 1];
            uint32_t a = (j & 1) ? (lo >> 16) : (lo & 0xffffu), bq = (j & 1) ? (hi >> 16) : (hi & 0xffffu);
            *reinterpret_cast<uint32_t*>(yb + (int64_t)c * ldy + r) = a | (bq << 16);
        }
    }
}

// row softmax: y = softmax(scale * x) over `cols`; one block per row
template <typename T>
__global__ void __launch_bounds__(256) softmax_rows_kernel(const T* __restrict__ x, int cols, int64_t ld, float scale,
                                                           T* __restrict__ y) {
    __shared__ float red[8];
    const T* xr = x + (int64_t)blockIdx.x * ld; T* yr = y + (int64_t)blockIdx.x * ld;
    float mx = -3e38f;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) mx = fmaxf(mx, H<T>::f(xr[c]) * scale);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = red[0];
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k) mx = fmaxf(mx, red[k]);
    __syncthreads();
    float s = 0.f;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) s += __expf(H<T>::f(xr[c]) * scale - mx);
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    s = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) s += red[k];
    float inv = 1.0f / s;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) yr[c] = H<T>::t(__expf(H<T>::f(xr[c]) * scale - mx) * inv);
}

// dS = scale * P * (dP - rowsum(P * dP))
template <typename T>
__global__ void __launch_bounds__(256) softmax_bwd_kernel(const T* __restrict__ P, const T* __restrict__ dP, int cols,
                                                          int64_t ld, float scale, T* __restrict__ dS) {
    __shared__ float red[8];
    const T* pr = P + (int64_t)blockIdx.x * ld; const T* dr = dP + (int64_t)blockIdx.x * ld; T* o = dS + (int64_t)blockIdx.x * ld;
    float s = 0.f;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) s += H<T>::f(pr[c]) * H<T>::f(dr[c]);
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    s = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) s += red[k];
    for (int c = threadIdx.x; c < cols; c += blockDim.x) o[c] = H<T>::t(scale * H<T>::f(pr[c]) * (H<T>::f(dr[c]) - s));
}

// fp32 [rows, cin] -> T [rows, cpad]: y = x*scale + shift on the real channels, 0 on the padding
template <typename T>
__global__ void __launch_bounds__(256) pad_convert_kernel(const float* __restrict__ x, int64_t rows, int cin, int cpad,
                                                          float scale, float shift, T* __restrict__ y) {
    // one 16-byte store (8 channels) per thread; cpad % 8 == 0
    const int vpr = cpad >> 3;
    const int64_t n = rows * vpr;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / vpr; const int c0 = (int)(i - r * vpr) * 8;
        uint4 o; T* oh = reinterpret_cast<T*>(&o);
#pragma unroll
        for (int k = 0; k < 8; ++k) oh[k] = H<T>::t((c0 + k < cin) ? fmaf(x[r * cin + c0 + k], scale, shift) : 0.f);
        *reinterpret_cast<uint4*>(y + r * cpad + c0) = o;
    }
}
// N1 (SURVEY.md section 8f): the pre-rendered condition maps stay on the device as the bytes the PNG decode produced
// (data/uncond.py:532-582): depth fp32 [V, HW], normal u8 [V, HW, 3], light u8 [V, E, HW, 18].  One pass gathers the
// (view, env) pairs of the batch, de-quantises (x / 255, the reference's arithmetic) and writes the channel-padded
// ControlNet condition [B, HW, cpad] in the storage dtype: channel order depth | normal | 6 x RGB light (:581-582,:802).
template <typename T>
__global__ void __launch_bounds__(256) cond_gather_kernel(const float* __restrict__ depth, const uint8_t* __restrict__ normal,
                                                          const uint8_t* __restrict__ light, int E, int64_t HW,
                                                          const int32_t* __restrict__ view_ids, const int32_t* __restrict__ env_ids,
                                                          int B, int cpad, T* __restrict__ out) {
    const int vpr = cpad >> 3;
    const int64_t n = (int64_t)B * HW * vpr;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int c0 = (int)(i % vpr) * 8; const int64_t r = i / vpr;
        const int64_t px = r % HW; const int b = (int)(r / HW);
        const int v = view_ids[b], e = env_ids[b];
        const uint8_t* nr = normal + ((int64_t)v * HW + px) * 3;
        const uint8_t* lt = light + (((int64_t)v * E + e) * HW + px) * 18;
        uint4 o; T* oh = reinterpret_cast<T*>(&o);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int c = c0 + k;
            float f = 0.f;
            if (c == 0) f = depth[(int64_t)v * HW + px];
            else if (c < 4) f = (float)nr[c - 1] / 255.0f;
            else if (c < 22) f = (float)lt[c - 4] / 255.0f;
            oh[k] = H<T>::t(f);
        }
        *reinterpret_cast<uint4*>(out + r * cpad + c0) = o;
    }
}

// T [rows, ld] (first cout channels) -> fp32 [rows, cout] * scale
template <typename T>
__global__ void __launch_bounds__(256) unpad_convert_kernel(const T* __restrict__ x, int64_t rows, int ld, int cout,
                                                            float scale, float* __restrict__ y) {
    int64_t n = rows * cout;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = i / cout; int c = (int)(i - r * cout);
        y[i] = H<T>::f(x[r * ld + c]) * scale;
    }
}
// NHWC T [n, HW, ld] (first C channels) -> NCHW fp32 [n, C, HW]
template <typename T>
__global__ void __launch_bounds__(256) nhwc_to_nchw_f32_kernel(const T* __restrict__ x, int n, int HW, int ld, int Cc,
                                                               float* __restrict__ y) {
    int64_t tot = (int64_t)n * Cc * HW;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < tot; i += (int64_t)gridDim.x * blockDim.x) {
        int p = (int)(i % HW); int64_t r = i / HW; int c = (int)(r % Cc); int img = (int)(r / Cc);
        y[i] = H<T>::f(x[((int64_t)img * HW + p) * ld + c]);
    }
}

// posterior sample (DiagonalGaussianDistribution): z = (mean + exp(0.5*clamp(logvar,-30,20)) * eps) * sf
// moments NHWC [n, HW, ld] (mean = ch 0..3, logvar = ch 4..7); z, eps NCHW fp32 [n,4,HW]
template <typename T>
__global__ void __launch_bounds__(256) vae_sample_kernel(const T* __restrict__ mom, int n, int HW, int ld,
                                                         const float* __restrict__ eps, float sf, float* __restrict__ z) {
    int64_t tot = (int64_t)n * 4 * HW;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < tot; i += (int64_t)gridDim.x * blockDim.x) {
        int p = (int)(i % HW); int64_t r = i / HW; int c = (int)(r % 4); int img = (int)(r / 4);
        const T* m = mom + ((int64_t)img * HW + p) * ld;
        float mean = H<T>::f(m[c]), lv = fminf(fmaxf(H<T>::f(m[4 + c]), -30.f), 20.f);
        // diffusers computes the sample in the weights dtype: round the pre-scale sample to T
        float smp = H<T>::f(H<T>::t(mean + H<T>::f(H<T>::t(__expf(0.5f * lv))) * H<T>::f(H<T>::t(eps[i]))));
        z[i] = H<T>::f(H<T>::t(smp * sf));
    }
}
// backward: dmom[.., c] = dz*sf ; dmom[.., 4+c] = dz*sf*eps*0.5*std (0 outside the clamp); padding channels 0
template <typename T>
__global__ void __launch_bounds__(256) vae_sample_bwd_kernel(const T* __restrict__ mom, int n, int HW, int ld,
                                                             const float* __restrict__ eps, float sf,
                                                             const float* __restrict__ dz, T* __restrict__ dmom) {
    int64_t tot = (int64_t)n * HW * ld;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < tot; i += (int64_t)gridDim.x * blockDim.x) {
        int ch = (int)(i % ld); int64_t r = i / ld; int p = (int)(r % HW); int img = (int)(r / HW);
        float v = 0.f;
        if (ch < 4) v = dz[((int64_t)img * 4 + ch) * HW + p] * sf;
        else if (ch < 8) {
            int c = ch - 4;
            float lvr = H<T>::f(mom[i]);
            if (lvr >= -30.f && lvr <= 20.f) {
                float sd = __expf(0.5f * lvr);
                int64_t zi = ((int64_t)img * 4 + c) * HW + p;
                v = dz[zi] * sf * eps[zi] * 0.5f * sd;
            }
        }
        dmom[i] = H<T>::t(v);
    }
}

// add_noise + CFG replication: out[(k*B + b), p, 0:4] = sqrt(ac[t_b]) z + sqrt(1-ac[t_b]) noise, k = 0..rep-1; pad 0
template <typename T>
__global__ void __launch_bounds__(256) add_noise_kernel(const float* __restrict__ z, const float* __restrict__ noise,
                                                        const float* __restrict__ sqrt_ac,
                                                        const float* __restrict__ sqrt_1mac, int B, int HW, int cpad,
                                                        int rep, T* __restrict__ out) {
    int64_t tot = (int64_t)rep * B * HW * cpad;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < tot; i += (int64_t)gridDim.x * blockDim.x) {
        int c = (int)(i % cpad); int64_t r = i / cpad; int p = (int)(r % HW); int bk = (int)(r / HW); int b = bk % B;
        float v = 0.f;
        if (c < 4) { int64_t zi = ((int64_t)b * 4 + c) * HW + p; v = sqrt_ac[b] * z[zi] + sqrt_1mac[b] * noise[zi]; }
        out[i] = H<T>::t(v);
    }
}

// get_timestep_embedding(t, dim, flip_sin_to_cos=True, downscale_freq_shift=0): [cos(t f_k) | sin(t f_k)]
template <typename T>
__global__ void timestep_embed_kernel(const float* __restrict__ t, int n, int dim, T* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int half = dim / 2;
    if (i >= n * half) return;
    int b = i / half, k = i % half;
    float f = expf(-9.210340371976184f * (float)k / (float)half);
    float a = t[b] * f;
    out[b * dim + k] = H<T>::t(cosf(a));
    out[b * dim + half + k] = H<T>::t(sinf(a));
}

template <typename T>
__global__ void __launch_bounds__(256) silu_kernel(const T* __restrict__ x, int64_t n, T* __restrict__ y) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        y[i] = H<T>::t(silu_f(H<T>::f(x[i])));
}

// dx = dy * silu'(z) on the pre-activation z (the backward of a SiLU epilogue whose pre-activation was recomputed)
template <typename T>
__global__ void __launch_bounds__(256) silu_bwd_kernel(const T* __restrict__ z, const T* __restrict__ dy, int64_t n8,
                                                       T* __restrict__ dx) {
    griddep_launch_dependents();
    griddep_wait();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
        const uint4 uz = reinterpret_cast<const uint4*>(z)[i], ud = reinterpret_cast<const uint4*>(dy)[i];
        const T* hz = reinterpret_cast<const T*>(&uz); const T* hd = reinterpret_cast<const T*>(&ud);
        uint4 o; T* oh = reinterpret_cast<T*>(&o);
#pragma unroll
        for (int j = 0; j < 8; ++j) oh[j] = H<T>::t(H<T>::f(hd[j]) * silu_grad(H<T>::f(hz[j])));
        reinterpret_cast<uint4*>(dx)[i] = o;
    }
}

// Gradient of the GEMM epilogue's per-image vector (a resnet's slice of the time-embedding projection): out[img, c] = sum
// over the image's rows of dy[row, c].  Block (v-block, chunk, img): a thread owns one 8-channel vector and the chunk's
// rows [chunk*rpc, +rpc) and writes its sums to partial row part[img][chunk][N]; rowvec_finish_kernel adds an image's
// partial rows in chunk order, so the result is bit-identical from run to run.
template <typename T>
__global__ void __launch_bounds__(128) rowvec_partials_kernel(const T* __restrict__ dy, int64_t ld, int rows_per_img, int N,
                                                              int rpc, float* __restrict__ part) {
    griddep_launch_dependents();
    griddep_wait();
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= N / 8) return;
    const int r0 = blockIdx.y * rpc, r1 = min(rows_per_img, r0 + rpc);
    const T* base = dy + (int64_t)blockIdx.z * rows_per_img * ld + 8 * v;
    float s[8] = {};
    for (int r = r0; r < r1; ++r) {
        const uint4 u = *reinterpret_cast<const uint4*>(base + r * ld);
        const T* h = reinterpret_cast<const T*>(&u);
#pragma unroll
        for (int k = 0; k < 8; ++k) s[k] += H<T>::f(h[k]);
    }
    float* pr = part + ((int64_t)blockIdx.z * gridDim.y + blockIdx.y) * N + 8 * v;
#pragma unroll
    for (int k = 0; k < 8; ++k) pr[k] = s[k];
}

template <typename T>
__global__ void __launch_bounds__(256) rowvec_finish_kernel(const float* __restrict__ part, int chunks, int N, int n_img,
                                                            T* __restrict__ out, int64_t ld_out) {
    griddep_launch_dependents();
    griddep_wait();
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_img * N) return;
    const int img = j / N, c = j - img * N;
    float s = 0.f;
    for (int k = 0; k < chunks; ++k) s += part[((int64_t)img * chunks + k) * N + c];
    out[img * ld_out + c] = H<T>::t(s);
}

// ----------------------------------------------------------------------------------- norm / GEGLU backward
// LayerNorm backward, warp per row (the forward's mapping): mean / rstd recomputed from x with the forward's arithmetic,
// g = dy * gamma, dx = rstd * (g - mean(g) - xhat * mean(g * xhat)) (+ dx_add).  (mean, rstd) of each row go to `rstats`
// for the affine-gradient kernel.
template <typename T>
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const T* __restrict__ x, const T* __restrict__ dy, int64_t M,
                                                            int C, const T* __restrict__ gamma, float eps,
                                                            const T* __restrict__ dx_add, T* __restrict__ dx,
                                                            float* __restrict__ rstats) {
    griddep_launch_dependents();
    griddep_wait();
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= M) return;
    const int lane = threadIdx.x & 31, nv = C >> 3;
    const T* xr = x + row * C;
    float vals[40], g[40];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        const int v = lane + 32 * k;
        if (v < nv) {
            uint4 u = *reinterpret_cast<const uint4*>(xr + 8 * v);
            uint4 ud = *reinterpret_cast<const uint4*>(dy + row * C + 8 * v);
            uint4 ug = *reinterpret_cast<const uint4*>(gamma + 8 * v);
            const T* h = reinterpret_cast<const T*>(&u); const T* hd = reinterpret_cast<const T*>(&ud);
            const T* hg = reinterpret_cast<const T*>(&ug);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float f = H<T>::f(h[j]); vals[8 * k + j] = f; s += f;
                g[8 * k + j] = H<T>::f(hd[j]) * H<T>::f(hg[j]);
            }
        }
    }
    s = warp_sum(s);
    const float mean = s / (float)C;
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        if (lane + 32 * k < nv) {
#pragma unroll
            for (int j = 0; j < 8; ++j) { float d = vals[8 * k + j] - mean; ss += d * d; }
        }
    }
    ss = warp_sum(ss);
    const float rstd = rsqrtf(ss / (float)C + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        if (lane + 32 * k < nv) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                vals[8 * k + j] = (vals[8 * k + j] - mean) * rstd;     // xhat
                s1 += g[8 * k + j];
                s2 = fmaf(g[8 * k + j], vals[8 * k + j], s2);
            }
        }
    }
    s1 = warp_sum(s1) / (float)C;
    s2 = warp_sum(s2) / (float)C;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        const int v = lane + 32 * k;
        if (v < nv) {
            uint4 ua = dx_add ? *reinterpret_cast<const uint4*>(dx_add + row * C + 8 * v) : make_uint4(0, 0, 0, 0);
            const T* ha = reinterpret_cast<const T*>(&ua);
            uint4 o; T* oh = reinterpret_cast<T*>(&o);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float val = rstd * (g[8 * k + j] - s1 - vals[8 * k + j] * s2);
                if (dx_add) val += H<T>::f(ha[j]);
                oh[j] = H<T>::t(val);
            }
            *reinterpret_cast<uint4*>(dx + row * C + 8 * v) = o;
        }
    }
    if (lane == 0) { rstats[2 * row] = mean; rstats[2 * row + 1] = rstd; }
}

// Affine-parameter gradients of LayerNorm (G == 0: stats per row) and GroupNorm (stats per (image, group), HW rows per
// image, optional SiLU after the affine): a thread owns one 8-channel vector and the rows [chunk*rpc, +rpc) and writes its
// sums to its own slots of the chunk's partial row part[chunk][2C] = (sum dy' xhat | sum dy'); affine_finish_kernel adds
// the chunks' rows in chunk order, so the result is bit-identical from run to run.
template <typename T>
__global__ void __launch_bounds__(128) affine_partials_kernel(const T* __restrict__ x, const T* __restrict__ dz, int64_t rows,
                                                              int C, int HW, int G, const float* __restrict__ stats,
                                                              const T* __restrict__ gamma, const T* __restrict__ beta,
                                                              int silu, int rpc, float* __restrict__ part) {
    griddep_launch_dependents();
    griddep_wait();
    const int v = blockIdx.y * blockDim.x + threadIdx.x;
    if (v >= C / 8) return;
    const int64_t r0 = (int64_t)blockIdx.x * rpc, r1 = min(rows, r0 + rpc);
    float gm[8], bt[8], dg[8] = {}, db[8] = {};
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        gm[k] = silu ? H<T>::f(gamma[8 * v + k]) : 0.f;
        bt[k] = silu ? H<T>::f(beta[8 * v + k]) : 0.f;
    }
    const int cpg = G ? C / G : 1;
    for (int64_t r = r0; r < r1; ++r) {
        uint4 ux = *reinterpret_cast<const uint4*>(x + r * C + 8 * v), ud = *reinterpret_cast<const uint4*>(dz + r * C + 8 * v);
        const T* hx = reinterpret_cast<const T*>(&ux); const T* hd = reinterpret_cast<const T*>(&ud);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int64_t si = G ? (r / HW * G + (8 * v + k) / cpg) * 2 : 2 * r;
            const float xhat = (H<T>::f(hx[k]) - stats[si]) * stats[si + 1];
            float d = H<T>::f(hd[k]);
            if (silu) d *= silu_grad(fmaf(xhat, gm[k], bt[k]));
            dg[k] = fmaf(d, xhat, dg[k]);
            db[k] += d;
        }
    }
    float* pr = part + (int64_t)blockIdx.x * 2 * C + 8 * v;
#pragma unroll
    for (int k = 0; k < 8; ++k) { pr[k] = dg[k]; pr[C + k] = db[k]; }
}

__global__ void __launch_bounds__(256) affine_finish_kernel(const float* __restrict__ part, int chunks, int C,
                                                            float* __restrict__ dgamma, float* __restrict__ dbeta) {
    griddep_launch_dependents();
    griddep_wait();
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= 2 * C) return;
    float s = 0.f;
    for (int c = 0; c < chunks; ++c) s += part[(int64_t)c * 2 * C + j];
    if (j < C) dgamma[j] = s; else dbeta[j - C] = s;
}

// GEGLU backward on the interleaved pre-activation of the fused GEGLU epilogue: h [M, 2D] in blocks of 64 columns (32 value
// columns, then their 32 gate columns), out[m, 32b + r] = h[m, 64b + r] * gelu(h[m, 64b + 32 + r]) (erf GELU).
//   dh[value] = dout * gelu(gate),  dh[gate] = dout * value * gelu'(gate),  gelu'(g) = Phi(g) + g phi(g)
template <typename T>
__global__ void __launch_bounds__(256) geglu_bwd_kernel(const T* __restrict__ h, const T* __restrict__ dout, int64_t M, int D,
                                                        T* __restrict__ dh) {
    griddep_launch_dependents();
    griddep_wait();
    const int64_t n = M * (int64_t)(D / 8);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = i / (D / 8);
        const int j = (int)(i - m * (D / 8)) * 8;                  // output column (8 of them)
        const int64_t hv = m * 2 * D + 64 * (j / 32) + j % 32;    // their value columns; gate columns at + 32
        uint4 a = *reinterpret_cast<const uint4*>(h + hv), g = *reinterpret_cast<const uint4*>(h + hv + 32);
        uint4 d = *reinterpret_cast<const uint4*>(dout + m * D + j);
        const T* ha = reinterpret_cast<const T*>(&a); const T* hg = reinterpret_cast<const T*>(&g);
        const T* hd = reinterpret_cast<const T*>(&d);
        uint4 ov, og; T* pv = reinterpret_cast<T*>(&ov); T* pg = reinterpret_cast<T*>(&og);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float gv = H<T>::f(hg[k]), dv = H<T>::f(hd[k]);
            const float cdf = 0.5f * (1.0f + erff(gv * 0.70710678118654752f));
            const float pdf = 0.3989422804014327f * expf(-0.5f * gv * gv);
            pv[k] = H<T>::t(dv * gv * cdf);
            pg[k] = H<T>::t(dv * H<T>::f(ha[k]) * (cdf + gv * pdf));
        }
        *reinterpret_cast<uint4*>(dh + hv) = ov;
        *reinterpret_cast<uint4*>(dh + hv + 32) = og;
    }
}

inline int grid_for(int64_t work, int threads = 256) {
    int64_t b = dm_ceil_div(work, threads);
    int64_t cap = (int64_t)DM_NUM_SMS * 8;
    return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}
inline int gn_vslab(int vpp) {
    for (int d = 32; d > 1; --d) if (vpp % d == 0) return d;
    return 1;
}
// pixel chunks so that chunks * n_img * slabs ~ 8 CTAs per SM, each thread keeping >= 4 pixels to stream
inline int gn_chunks(int n_img, int HW, int slabs, int lanes) {
    int c = (DM_NUM_SMS * 8) / ((n_img > 0 ? n_img : 1) * slabs);
    if (c < 1) c = 1;
    int maxc = HW / (4 * lanes); if (maxc < 1) maxc = 1;
    return c < maxc ? c : maxc;
}

}  // namespace

// partial rows of one GroupNorm call in the library scratch (at least 1 MB, so one allocation serves every layer of a model)
static float* gn_partials(int nv, int n_img, int G, int slabs, int chunks, cudaStream_t st) {
    size_t bytes = (size_t)nv * n_img * G * slabs * chunks * sizeof(float);
    if (bytes < ((size_t)1 << 20)) bytes = (size_t)1 << 20;
    return (float*)dm_scratch(DM_SCRATCH_GN, bytes, st);
}

extern "C" int dm_groupnorm(int bf16, const void* x, int n_img, int HW, int C, int ld, int G, const void* gamma,
                            const void* beta, float eps, int silu, void* y, int ldy, float* stats, void* stream) {
    DM_DTYPE_OK(bf16);
    if (bf16 == 2) return hp_groupnorm((const float*)x, n_img, HW, C, ld, G, (const float*)gamma, (const float*)beta, eps, silu, (float*)y, ldy, stats, stream);
    DM_REQUIRE(x && gamma && beta && y && stats, "null pointer");
    DM_REQUIRE(C % 8 == 0 && C % G == 0 && (C / G) % 2 == 0 && ld % 8 == 0 && ldy % 8 == 0, "channel layout");
    cudaStream_t st = (cudaStream_t)stream;
    const int vslab = gn_vslab(C / 8), slabs = (C / 8) / vslab;
    const int chunks = gn_chunks(n_img, HW, slabs, 256 / vslab);
    const dim3 grid(chunks, n_img, slabs);
    float* part = gn_partials(4, n_img, G, slabs, chunks, st);
    if (!part) return DM_EDRIVER;
    DM_DISPATCH_T(bf16, DM_CHECK_CUDA(dm_launch(gn_stats_kernel<T>, grid, dim3(256), 0, st, (const T*)x, HW, C, ld, G, chunks, vslab, part)));
    DM_CHECK_LAUNCH();
    DM_DISPATCH_T(bf16, DM_CHECK_CUDA(dm_launch(gn_moments_kernel<T>, dim3((unsigned)dm_ceil_div(4 * n_img * G, 256)), dim3(256), 0, st, n_img, HW, C, ld,
                                                G, vslab, slabs, chunks, (const float*)part, (const T*)x, eps, stats)));
    DM_CHECK_LAUNCH();
    DM_DISPATCH_T(bf16, DM_CHECK_CUDA(dm_launch(gn_apply_kernel<T>, grid, dim3(256), 0, st, (const T*)x, HW, C, ld, ldy, G, chunks, vslab, (const float*)stats,
                                                (const T*)gamma, (const T*)beta, silu, (T*)y)));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_groupnorm_bwd(int bf16, const void* x, const void* dz, int n_img, int HW, int C, int G,
                                const void* gamma, const void* beta, float eps, int silu, const float* stats,
                                float* bstats, const void* dx_add, void* dx, void* stream) {
    DM_DTYPE_OK(bf16);
    if (bf16 == 2) return hp_groupnorm_bwd((const float*)x, (const float*)dz, n_img, HW, C, G, (const float*)gamma, (const float*)beta, eps, silu, stats, (const float*)dx_add, (float*)dx, stream);
    DM_REQUIRE(x && dz && gamma && beta && stats && bstats && dx, "null pointer");
    DM_REQUIRE(C % 8 == 0 && C % G == 0 && (C / G) % 2 == 0, "channel layout");
    (void)eps;   // stats already hold (mean, rstd), as in the fp32 mode
    cudaStream_t st = (cudaStream_t)stream;
    const int vslab = gn_vslab(C / 8), slabs = (C / 8) / vslab;
    const int chunks = gn_chunks(n_img, HW, slabs, 256 / vslab);
    const dim3 grid(chunks, n_img, slabs);
    float* part = gn_partials(2, n_img, G, slabs, chunks, st);
    if (!part) return DM_EDRIVER;
    DM_DISPATCH_T(bf16, DM_CHECK_CUDA(dm_launch(gn_bwd_stats_kernel<T>, grid, dim3(256), 0, st,
                            (const T*)x, (const T*)dz, HW, C, G, chunks, vslab, stats, (const T*)gamma, (const T*)beta, silu, part)));
    DM_CHECK_LAUNCH();
    DM_CHECK_CUDA(dm_launch(gn_finish_kernel, dim3((unsigned)dm_ceil_div(2 * n_img * G, 256)), dim3(256), 0, st, n_img, C, G, vslab, slabs, chunks,
                            (const float*)part, bstats));
    DM_CHECK_LAUNCH();
    DM_DISPATCH_T(bf16, DM_CHECK_CUDA(dm_launch(gn_bwd_apply_kernel<T>, grid, dim3(256), 0, st, (const T*)x, (const T*)dz, HW, C, G, chunks, vslab, stats,
                                                (const float*)bstats, (const T*)gamma, (const T*)beta, silu, (const T*)dx_add, (T*)dx)));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_layernorm(int bf16, const void* x, int64_t M, int C, const void* gamma, const void* beta, float eps,
                            void* y, void* stream) {
    DM_DTYPE_OK(bf16);
    if (bf16 == 2) return hp_layernorm((const float*)x, M, C, (const float*)gamma, (const float*)beta, eps, (float*)y, stream);
    DM_REQUIRE(x && gamma && beta && y, "null pointer");
    DM_REQUIRE(C <= 1280 && C % 8 == 0, "C <= 1280, multiple of 8");
    if (M == 0) return DM_OK;
    DM_DISPATCH_T(bf16, DM_CHECK_CUDA(dm_launch(layernorm_kernel<T>, dim3((unsigned)dm_ceil_div(M, 8)), dim3(256), 0, (cudaStream_t)stream,
                                                (const T*)x, M, C, (const T*)gamma, (const T*)beta, eps, (T*)y)));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_geglu(int bf16, const void* h, int64_t M, int D, void* out, void* stream) {
    DM_DTYPE_OK(bf16);
    if (bf16 == 2) return hp_geglu((const float*)h, M, D, (float*)out, stream);
    DM_REQUIRE(h && out && D % 8 == 0, "bad args");
    DM_DISPATCH_T(bf16, geglu_kernel<T><<<grid_for(M * (D / 8)), 256, 0, (cudaStream_t)stream>>>((const T*)h, M, D, (T*)out));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_upsample2x(int bf16, const void* x, int n, int H, int W, int C, int zero_insert, void* y, void* stream) {
    DM_DTYPE_OK(bf16);
    if (bf16 == 2) return dm_upsample2x(0, x, n, H, W, 2 * C, zero_insert, y, stream);
    DM_REQUIRE(x && y && C % 8 == 0, "bad args");
    int64_t nv = (int64_t)n * 4 * H * W * (C / 8);
    if (zero_insert) DM_DISPATCH_T(bf16, zero_insert2x_kernel<T><<<grid_for(nv), 256, 0, (cudaStream_t)stream>>>((const T*)x, n, H, W, C, (T*)y));
    else DM_DISPATCH_T(bf16, upsample2x_kernel<T><<<grid_for(nv), 256, 0, (cudaStream_t)stream>>>((const T*)x, n, H, W, C, (T*)y));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_axpby2d(int bf16, const void* s1, int64_t ld1, float a, const void* s2, int64_t ld2, float b,
                          int64_t rows, int cols, void* dst, int64_t ldd, void* stream) {
    DM_DTYPE_OK(bf16);
    if (bf16 == 2) return hp_axpby2d((const float*)s1, ld1, a, (const float*)s2, ld2, b, rows, cols, (float*)dst, ldd, stream);
    DM_REQUIRE(s1 && dst && cols % 8 == 0 && ld1 % 8 == 0 && ldd % 8 == 0 && (!s2 || ld2 % 8 == 0), "bad args");
    if (rows == 0) return DM_OK;
    DM_DISPATCH_T(bf16, axpby2d_kernel<T><<<grid_for(rows * (cols / 8)), 256, 0, (cudaStream_t)stream>>>((const T*)s1, ld1, a, (const T*)s2, ld2, b,
                                                                                                     rows, cols, (T*)dst, ldd));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_transpose(int bf16, const void* x, int batch, int R, int C, int64_t ldx, int64_t bsx, void* y,
                            int64_t ldy, int64_t bsy, void* stream) {
    DM_DTYPE_OK(bf16);
    if (bf16 == 2) return hp_transpose((const float*)x, batch, R, C, ldx, bsx, (float*)y, ldy, bsy, stream);
    DM_REQUIRE(x && y, "null pointer");
    DM_REQUIRE(((R | C) & 1) == 0 && ((ldx | ldy | bsx | bsy) & 1) == 0 && ((((uintptr_t)x) | ((uintptr_t)y)) & 3) == 0,
               "transpose moves 32-bit pairs: even extents / strides, 4-byte aligned bases");
    dim3 grid((unsigned)dm_ceil_div(C, 64), (unsigned)dm_ceil_div(R, 64), (unsigned)batch);
    DM_DISPATCH_T(bf16, transpose_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>((const T*)x, R, C, ldx, bsx, (T*)y, ldy, bsy));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_softmax_rows(int bf16, const void* x, int64_t rows, int cols, int64_t ld, float scale, void* y,
                               void* stream) {
    DM_DTYPE_OK(bf16);
    DM_REQUIRE(x && y, "null pointer");
    if (rows == 0) return DM_OK;
    DM_DISPATCH_T3(bf16, softmax_rows_kernel<T><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((const T*)x, cols, ld, scale, (T*)y));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_softmax_bwd(int bf16, const void* P, const void* dP, int64_t rows, int cols, int64_t ld, float scale,
                              void* dS, void* stream) {
    DM_DTYPE_OK(bf16);
    DM_REQUIRE(P && dP && dS, "null pointer");
    if (rows == 0) return DM_OK;
    DM_DISPATCH_T3(bf16, softmax_bwd_kernel<T><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>((const T*)P, (const T*)dP, cols, ld, scale, (T*)dS));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_pad_convert(int bf16, const float* x, int64_t rows, int cin, int cpad, float scale, float shift,
                              void* y, void* stream) {
    DM_DTYPE_OK(bf16);
    if (bf16 == 2) return hp_pad_convert(x, rows, cin, cpad, scale, shift, (float*)y, stream);
    DM_REQUIRE(x && y && cpad >= cin && cpad % 8 == 0, "bad args (cpad must be a multiple of 8)");
    DM_DISPATCH_T(bf16, pad_convert_kernel<T><<<grid_for(rows * (cpad / 8)), 256, 0, (cudaStream_t)stream>>>(x, rows, cin, cpad, scale, shift, (T*)y));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_cond_gather(int bf16, const float* depth, const uint8_t* normal, const uint8_t* light, int n_env, int64_t HW,
                              const int32_t* view_ids, const int32_t* env_ids, int B, int cpad, void* out, void* stream) {
    DM_REQUIRE(bf16 == 0 || bf16 == 1, "16-bit storage (the fp32 mode takes the float condition map through dm_pad_convert)");
    DM_REQUIRE(depth && normal && light && view_ids && env_ids && out && cpad >= 22 && cpad % 8 == 0 && n_env > 0, "bad args");
    if (B == 0 || HW == 0) return DM_OK;
    DM_DISPATCH_T(bf16, cond_gather_kernel<T><<<grid_for((int64_t)B * HW * (cpad / 8)), 256, 0, (cudaStream_t)stream>>>(
                            depth, normal, light, n_env, HW, view_ids, env_ids, B, cpad, (T*)out));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_unpad_convert(int bf16, const void* x, int64_t rows, int ld, int cout, float scale, float* y,
                                void* stream) {
    DM_DTYPE_OK(bf16);
    DM_REQUIRE(x && y && ld >= cout, "bad args");
    DM_DISPATCH_T3(bf16, unpad_convert_kernel<T><<<grid_for(rows * cout), 256, 0, (cudaStream_t)stream>>>((const T*)x, rows, ld, cout, scale, y));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_nhwc_to_nchw_f32(int bf16, const void* x, int n, int HW, int ld, int C, float* y, void* stream) {
    DM_DTYPE_OK(bf16);
    DM_REQUIRE(x && y, "null pointer");
    DM_DISPATCH_T3(bf16, nhwc_to_nchw_f32_kernel<T><<<grid_for((int64_t)n * C * HW), 256, 0, (cudaStream_t)stream>>>((const T*)x, n, HW, ld, C, y));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_vae_sample(int bf16, const void* moments, int n, int HW, int ld, const float* eps, float scaling,
                             float* z, void* stream) {
    DM_DTYPE_OK(bf16);
    DM_REQUIRE(moments && eps && z && ld >= 8, "bad args");
    DM_DISPATCH_T3(bf16, vae_sample_kernel<T><<<grid_for((int64_t)n * 4 * HW), 256, 0, (cudaStream_t)stream>>>((const T*)moments, n, HW, ld, eps, scaling, z));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_vae_sample_bwd(int bf16, const void* moments, int n, int HW, int ld, const float* eps, float scaling,
                                 const float* dz, void* dmoments, void* stream) {
    DM_DTYPE_OK(bf16);
    DM_REQUIRE(moments && eps && dz && dmoments && ld >= 8, "bad args");
    DM_DISPATCH_T3(bf16, vae_sample_bwd_kernel<T><<<grid_for((int64_t)n * HW * ld), 256, 0, (cudaStream_t)stream>>>((const T*)moments, n, HW, ld, eps,
                                                                                                               scaling, dz, (T*)dmoments));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_add_noise(int bf16, const float* z, const float* noise, const float* sqrt_ac, const float* sqrt_1mac,
                            int B, int HW, int cpad, int rep, void* out, void* stream) {
    DM_DTYPE_OK(bf16);
    DM_REQUIRE(z && noise && sqrt_ac && sqrt_1mac && out && cpad >= 4, "bad args");
    DM_DISPATCH_T3(bf16, add_noise_kernel<T><<<grid_for((int64_t)rep * B * HW * cpad), 256, 0, (cudaStream_t)stream>>>(z, noise, sqrt_ac, sqrt_1mac, B, HW,
                                                                                                                  cpad, rep, (T*)out));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_timestep_embedding(int bf16, const float* t, int n, int dim, void* out, void* stream) {
    DM_DTYPE_OK(bf16);
    DM_REQUIRE(t && out && dim % 2 == 0, "bad args");
    DM_DISPATCH_T3(bf16, timestep_embed_kernel<T><<<(unsigned)dm_ceil_div((int64_t)n * dim / 2, 128), 128, 0, (cudaStream_t)stream>>>(t, n, dim, (T*)out));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_silu(int bf16, const void* x, int64_t n, void* y, void* stream) {
    DM_DTYPE_OK(bf16);
    DM_REQUIRE(x && y, "null pointer");
    DM_DISPATCH_T3(bf16, silu_kernel<T><<<grid_for(n), 256, 0, (cudaStream_t)stream>>>((const T*)x, n, (T*)y));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_silu_bwd(int bf16, const void* z, const void* dy, int64_t n, void* dx, void* stream) {
    DM_DTYPE_OK(bf16);
    if (bf16 == 2) { dm_set_error("dm_silu_bwd: fp32 storage is not supported (16-bit only)"); return DM_EUNSUPPORTED; }
    DM_REQUIRE(z && dy && dx, "null pointer");
    DM_REQUIRE(n >= 0 && n % 8 == 0 && ((((uintptr_t)z | (uintptr_t)dy | (uintptr_t)dx) & 15) == 0),
               "element count a multiple of 8, 16-byte aligned operands");
    if (n == 0) return DM_OK;
    DM_DISPATCH_T(bf16, DM_CHECK_CUDA(dm_launch(silu_bwd_kernel<T>, dim3((unsigned)grid_for(n / 8)), dim3(256), 0, (cudaStream_t)stream,
                                                (const T*)z, (const T*)dy, n / 8, (T*)dx)));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_rowvec_grad(int bf16, const void* dy, int64_t ld, int n_img, int rows_per_img, int N, void* out,
                              int64_t ld_out, void* stream) {
    DM_DTYPE_OK(bf16);
    if (bf16 == 2) { dm_set_error("dm_rowvec_grad: fp32 storage is not supported (16-bit only)"); return DM_EUNSUPPORTED; }
    DM_REQUIRE(dy && out, "null pointer");
    DM_REQUIRE(n_img > 0 && rows_per_img > 0 && N > 0 && N % 8 == 0, "positive extents, N a multiple of 8");
    DM_REQUIRE(ld % 8 == 0 && ld >= N && ((uintptr_t)dy & 15) == 0, "dy 16-byte aligned, row stride a multiple of 8 elements, at least N");
    DM_REQUIRE(ld_out >= N && ((uintptr_t)out & 1) == 0, "out row stride at least N");
    cudaStream_t st = (cudaStream_t)stream;
    // about 4 CTAs per SM over (images x chunks), at least 16 rows per chunk
    int rpc = (int)dm_ceil_div((int64_t)n_img * rows_per_img, DM_NUM_SMS * 4);
    if (rpc < 16) rpc = 16;
    const int chunks = (int)dm_ceil_div(rows_per_img, rpc);
    float* part = (float*)dm_scratch(DM_SCRATCH_AFFINE, (size_t)n_img * chunks * N * sizeof(float), st);
    if (!part) return DM_EDRIVER;
    DM_DISPATCH_T(bf16, DM_CHECK_CUDA(dm_launch(rowvec_partials_kernel<T>, dim3((unsigned)dm_ceil_div(N / 8, 128), (unsigned)chunks, (unsigned)n_img),
                                                dim3(128), 0, st, (const T*)dy, ld, rows_per_img, N, rpc, part)));
    DM_CHECK_LAUNCH();
    DM_DISPATCH_T(bf16, DM_CHECK_CUDA(dm_launch(rowvec_finish_kernel<T>, dim3((unsigned)dm_ceil_div((int64_t)n_img * N, 256)), dim3(256), 0, st,
                                                (const float*)part, chunks, N, n_img, (T*)out, ld_out)));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

// partial rows of the affine gradients (and LayerNorm's per-row stats) in the library scratch; rows per chunk chosen so
// that there are about 4 CTAs per SM
static int affine_grad(int bf16, const void* x, const void* dz, int64_t rows, int C, int HW, int G, const float* stats,
                       const void* gamma, const void* beta, int silu, float* part, float* dgamma, float* dbeta,
                       cudaStream_t st) {
    const int rpc = (int)(rows / (DM_NUM_SMS * 4)) + 1 < 16 ? 16 : (int)(rows / (DM_NUM_SMS * 4)) + 1;
    const int chunks = (int)dm_ceil_div(rows, rpc);
    DM_DISPATCH_T(bf16, DM_CHECK_CUDA(dm_launch(affine_partials_kernel<T>, dim3((unsigned)chunks, (unsigned)dm_ceil_div(C / 8, 128)),
                                                dim3(128), 0, st, (const T*)x, (const T*)dz, rows, C, HW, G, stats,
                                                (const T*)gamma, (const T*)beta, silu, rpc, part)));
    DM_CHECK_LAUNCH();
    DM_CHECK_CUDA(dm_launch(affine_finish_kernel, dim3((unsigned)dm_ceil_div(2 * C, 256)), dim3(256), 0, st, (const float*)part,
                            chunks, C, dgamma, dbeta));
    DM_CHECK_LAUNCH();
    return DM_OK;
}
static size_t affine_part_bytes(int64_t rows, int C) {
    const int rpc = (int)(rows / (DM_NUM_SMS * 4)) + 1 < 16 ? 16 : (int)(rows / (DM_NUM_SMS * 4)) + 1;
    return (size_t)dm_ceil_div(rows, rpc) * 2 * C * sizeof(float);
}

extern "C" int dm_layernorm_bwd(int bf16, const void* x, const void* dy, int64_t M, int C, const void* gamma, float eps,
                                const void* dx_add, void* dx, float* dgamma, float* dbeta, void* stream) {
    DM_DTYPE_OK(bf16);
    if (bf16 == 2) { dm_set_error("dm_layernorm_bwd: fp32 storage is not supported (16-bit only)"); return DM_EUNSUPPORTED; }
    DM_REQUIRE(x && dy && gamma && dx && dgamma && dbeta, "null pointer");
    DM_REQUIRE(C <= 1280 && C % 8 == 0 && M > 0, "C <= 1280, multiple of 8; M >= 1");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t pb = affine_part_bytes(M, C);
    float* part = (float*)dm_scratch(DM_SCRATCH_AFFINE, pb + (size_t)M * 2 * sizeof(float), st);
    if (!part) return DM_EDRIVER;
    float* rstats = part + pb / sizeof(float);
    DM_DISPATCH_T(bf16, DM_CHECK_CUDA(dm_launch(layernorm_bwd_kernel<T>, dim3((unsigned)dm_ceil_div(M, 8)), dim3(256), 0, st,
                                                (const T*)x, (const T*)dy, M, C, (const T*)gamma, eps, (const T*)dx_add,
                                                (T*)dx, rstats)));
    DM_CHECK_LAUNCH();
    return affine_grad(bf16, x, dy, M, C, 1, 0, rstats, gamma, gamma, 0, part, dgamma, dbeta, st);
}

extern "C" int dm_groupnorm_affine_grad(int bf16, const void* x, const void* dz, int n_img, int HW, int C, int G,
                                        const void* gamma, const void* beta, int silu, const float* stats, float* dgamma,
                                        float* dbeta, void* stream) {
    DM_DTYPE_OK(bf16);
    if (bf16 == 2) { dm_set_error("dm_groupnorm_affine_grad: fp32 storage is not supported (16-bit only)"); return DM_EUNSUPPORTED; }
    DM_REQUIRE(x && dz && stats && dgamma && dbeta && (!silu || (gamma && beta)), "null pointer");
    DM_REQUIRE(C % 8 == 0 && G > 0 && C % G == 0 && n_img > 0 && HW > 0, "channel layout");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t rows = (int64_t)n_img * HW;
    float* part = (float*)dm_scratch(DM_SCRATCH_AFFINE, affine_part_bytes(rows, C), st);
    if (!part) return DM_EDRIVER;
    return affine_grad(bf16, x, dz, rows, C, HW, G, stats, gamma, beta, silu, part, dgamma, dbeta, st);
}

extern "C" int dm_geglu_bwd(int bf16, const void* h, const void* dout, int64_t M, int D, void* dh, void* stream) {
    DM_DTYPE_OK(bf16);
    if (bf16 == 2) { dm_set_error("dm_geglu_bwd: fp32 storage is not supported (16-bit only)"); return DM_EUNSUPPORTED; }
    DM_REQUIRE(h && dout && dh, "null pointer");
    DM_REQUIRE(D % 32 == 0 && M >= 0, "D multiple of 32 (interleaved 32-column value / gate blocks)");
    if (M == 0) return DM_OK;
    DM_DISPATCH_T(bf16, DM_CHECK_CUDA(dm_launch(geglu_bwd_kernel<T>, dim3((unsigned)grid_for(M * (D / 8))), dim3(256), 0,
                                                (cudaStream_t)stream, (const T*)h, (const T*)dout, M, D, (T*)dh)));
    DM_CHECK_LAUNCH();
    return DM_OK;
}
