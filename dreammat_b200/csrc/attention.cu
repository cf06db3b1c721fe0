// attention.cu -- fused softmax(Q K^T / sqrt(d)) V for head_dim 64 on Hopper wgmma tensor cores.
//
// Replaces torch SDPA / diffusers AttnProcessor inside BasicTransformerBlock (self-attention,
// N = 4096 / 1024 / 256 / 64 tokens, and cross-attention over the 77 text tokens) for the UNet and
// ControlNet forward passes (models/guidance/dreammat_guidance.py:218-229, :274-282).
//
// Layout: Q [B, Nq, ldq], K/V [B, Nk, ldk] token-major with all heads side by side (head h lives in
// columns [64h, 64h+64)), so the q/k/v projections' GEMM output is consumed in place -- TMA picks the
// head slice; no split-heads copies.  O is written back in the same layout.
//
// One CTA = 128 queries of one (batch, head); keys are streamed in blocks of 64:
//   warp 8      TMA producer: Q once, then a ring of K/V stages
//   warps 0-7   two consumer warpgroups, 64 query rows each:
//               S = Q K_j^T   (m64n64k16, both operands in shared memory, accumulator in registers)
//               online max / exp2 / sum on the S fragment (a row lives in the 4 lanes of a quad)
//               O += P_j V_j  (P_j straight from registers as the A operand, V_j an MN-major shared-memory operand)
#include <cuda.h>
#include <cuda_bf16.h>
#include "common.cuh"
#include "tc_common.cuh"
#include "dense_hp.cuh"

namespace {

constexpr int AQ = 128;       // queries per CTA
constexpr int AK = 64;        // keys per block
constexpr int HD = 64;        // head dim
constexpr int KV_STAGES = 3;
constexpr int ATT_THREADS = 288;
constexpr int Q_BYTES = AQ * HD * 2;     // 16 KB
constexpr int KV_BYTES = AK * HD * 2;    // 8 KB
constexpr int ATT_SMEM = Q_BYTES + 2 * KV_STAGES * KV_BYTES + 1024 + 256;

struct AttnParams {
    int Nq, Nk, heads;
    void* out; int64_t ldo; int64_t out_batch_stride;
    float scale_log2e;   // (1/sqrt(d)) * log2(e)
    float* lse = nullptr;   // [batch, heads, Nq] natural-log logsumexp of the scaled logits (written when LSE)
};

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

template <typename T> struct PK;
template <> struct PK<__half> {
    static __device__ __forceinline__ uint32_t pack(float a, float b) {
        __half2 h = __floats2half2_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&h);
    }
};
template <> struct PK<__nv_bfloat16> {
    static __device__ __forceinline__ uint32_t pack(float a, float b) {
        __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&h);
    }
};

__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

template <typename T, bool LSE = false>
__global__ void __launch_bounds__(ATT_THREADS, 2) attention_kernel(const __grid_constant__ CUtensorMap tmQ,
                                                                   const __grid_constant__ CUtensorMap tmK,
                                                                   const __grid_constant__ CUtensorMap tmV,
                                                                   const AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sQ = base, sK = sQ + Q_BYTES, sV = sK + KV_STAGES * KV_BYTES;
    const uint32_t bars = sV + KV_STAGES * KV_BYTES;
    const uint32_t q_full = bars;
    auto kv_full = [&](int s) { return bars + 8u * (1 + s); };
    auto kv_empty = [&](int s) { return bars + 8u * (1 + KV_STAGES + s); };

    griddep_launch_dependents();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q_tile = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
    const int nkb = (p.Nk + AK - 1) / AK;

    if (threadIdx.x == 0) {
        prefetch_tmap(&tmQ); prefetch_tmap(&tmK); prefetch_tmap(&tmV);
        mbar_init(q_full, 1);
        for (int s = 0; s < KV_STAGES; ++s) { mbar_init(kv_full(s), 1); mbar_init(kv_empty(s), 2); }
        fence_mbar_init();
    }
    __syncthreads();
    griddep_wait();      // PDL: q/k/v written by the previous kernel are visible from here

    if (warp == 8) {
        if (lane == 0) {
            mbar_expect_tx(q_full, Q_BYTES);
            tma_load_3d(sQ, &tmQ, q_full, head * HD, q_tile * AQ, b);
            int stage = 0; uint32_t phase = 0;
            for (int j = 0; j < nkb; ++j) {
                mbar_wait(kv_empty(stage), phase ^ 1u);
                mbar_expect_tx(kv_full(stage), 2 * KV_BYTES);
                tma_load_3d(sK + stage * KV_BYTES, &tmK, kv_full(stage), head * HD, j * AK, b);
                tma_load_3d(sV + stage * KV_BYTES, &tmV, kv_full(stage), head * HD, j * AK, b);
                if (++stage == KV_STAGES) { stage = 0; phase ^= 1u; }
            }
        }
        return;
    }
    const int wg = warp >> 2;
    const int quad_col = 2 * (lane & 3);                       // fragment columns 8j + quad_col + {0, 1}
    const uint64_t dQ = make_sw128_desc(sQ + (uint32_t)wg * (64 * 128));
    float o[HD / 2];
#pragma unroll
    for (int c = 0; c < HD / 2; ++c) o[c] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // rows r and r + 8 (log2 domain max, partial sums)
    mbar_wait(q_full, 0);
    int stage = 0; uint32_t phase = 0;
    for (int j = 0; j < nkb; ++j) {
        mbar_wait(kv_full(stage), phase);
        float s[AK / 2];
#pragma unroll
        for (int c = 0; c < AK / 2; ++c) s[c] = 0.f;
        const uint64_t dK = make_sw128_desc(sK + stage * KV_BYTES);
        wgmma_fence();
        wgmma_fence_operands(s);
#pragma unroll
        for (int k = 0; k < HD / 16; ++k) Wgmma<AK, T>::ss(s, dQ + (uint64_t)(2 * k), dK + (uint64_t)(2 * k));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operands(s);
        const int kvalid = p.Nk - j * AK;    // keys of this block that exist
        if (kvalid < AK) {                   // ragged last block (cross-attention over 77 tokens): mask the missing keys
#pragma unroll
            for (int c = 0; c < AK / 2; ++c)
                if (8 * (c >> 2) + quad_col + (c & 1) >= kvalid) s[c] = -INFINITY;
        }
        float alpha[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float mx = -INFINITY;
#pragma unroll
            for (int jj = 0; jj < AK / 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
            const float m_new = fmaxf(m_run[h], quad_max(mx) * p.scale_log2e);
            alpha[h] = fast_exp2(m_run[h] - m_new);             // m_run = -inf on the first block -> 0
            m_run[h] = m_new;
            float l = 0.f;
#pragma unroll
            for (int jj = 0; jj < AK / 8; ++jj) {
                float* v = &s[4 * jj + 2 * h];
                v[0] = fast_exp2(fmaf(v[0], p.scale_log2e, -m_new));
                v[1] = fast_exp2(fmaf(v[1], p.scale_log2e, -m_new));
                l += v[0] + v[1];
            }
            l_run[h] = l_run[h] * alpha[h] + l;
        }
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj) {
            o[4 * jj] *= alpha[0]; o[4 * jj + 1] *= alpha[0];
            o[4 * jj + 2] *= alpha[1]; o[4 * jj + 3] *= alpha[1];
        }
        // the S accumulator fragment of columns [16kk, 16kk+16) is the A-operand fragment of k-step kk
        const uint64_t dV = make_sw128_desc_mn(sV + stage * KV_BYTES);
        uint32_t a[AK / 16][4];
#pragma unroll
        for (int kk = 0; kk < AK / 16; ++kk)
#pragma unroll
            for (int r = 0; r < 4; ++r) a[kk][r] = PK<T>::pack(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
        wgmma_fence();
        wgmma_fence_operands(o);
#pragma unroll
        for (int kk = 0; kk < AK / 16; ++kk) Wgmma<HD, T>::rs_bt(o, a[kk], dV + (uint64_t)(128 * kk));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operands(o);
        if ((threadIdx.x & 127) == 0) mbar_arrive(kv_empty(stage));
        if (++stage == KV_STAGES) { stage = 0; phase ^= 1u; }
    }
    const int row = q_tile * AQ + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int q = row + 8 * h;
        const float l = quad_sum(l_run[h]);      // every lane of the quad shuffles: before any branch
        const float inv = 1.0f / l;
        if (q >= p.Nq) continue;
        if constexpr (LSE) {   // logsumexp_k(scale q.k) = ln2 * (m + log2 l), m and l in the log2 domain of the loop
            if ((lane & 3) == 0) p.lse[((int64_t)b * p.heads + head) * p.Nq + q] = (m_run[h] + log2f(l)) * 0.6931471805599453f;
        }
        T* orow = reinterpret_cast<T*>(p.out) + (int64_t)b * p.out_batch_stride + (int64_t)q * p.ldo + head * HD;
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj)
            *reinterpret_cast<uint32_t*>(orow + 8 * jj + quad_col) = PK<T>::pack(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    }
}

// ---------------------------------------------------------------------------------------------------- backward
// dQ, dK and dV of O = softmax(scale Q K^T) V, from q, k, v, O, dO and the forward's lse.  Every output element is owned
// by one CTA and summed in one fixed order (no atomics), at the price of computing S = Q K^T and dP = dO V^T twice:
//   attn_delta_kernel   delta = rowsum(dO o O) per (batch, head, query), fp32
//   attn_dkdv_kernel    a CTA owns 128 keys of one (batch, head) and streams 64-query blocks of Q / dO:
//                       S^T = K Q^T, P^T = exp2(S^T scale log2e - lse log2e), dV += P^T dO, dP^T = V dO^T,
//                       dS^T = P^T o (dP^T - delta), dK += dS^T Q  (dK scaled at the end)
//   attn_dq_kernel      a CTA owns 128 queries and streams 64-key blocks of K / V:
//                       S = Q K^T, P, dP = dO V^T, dS = P o (dP - delta), dQ += dS K  (scaled at the end)
// Both big kernels have the forward's shape: warp 8 loads the CTA's own 128-row tiles once and then a TMA ring of 64-row
// block pairs; warpgroups 0 / 1 own 64 rows each.  The same 128B-swizzled tile of a streamed block is the K-major B operand
// of an ss product and the MN-major B operand of a register-A product, as V is in the forward.
constexpr int BWD_STAGES = 3;
constexpr int VEC_BYTES = 2 * AK * 4;    // per stage: lse * log2(e) and delta of the streamed queries
constexpr int BWD_SMEM = 2 * Q_BYTES + BWD_STAGES * (2 * KV_BYTES + VEC_BYTES) + 1024 + 256;

struct BwdParams {
    int Nq, Nk, heads;
    const float* lse; const float* delta;   // [batch, heads, Nq]
    void* dq; int64_t lddq, dq_bs;
    void* dk; int64_t lddk, dk_bs;
    void* dv; int64_t lddv, dv_bs;
    float scale, scale_log2e;
};

template <typename T> __device__ __forceinline__ float2 unpack2(uint32_t u);
template <> __device__ __forceinline__ float2 unpack2<__half>(uint32_t u) { return __half22float2(*reinterpret_cast<__half2*>(&u)); }
template <> __device__ __forceinline__ float2 unpack2<__nv_bfloat16>(uint32_t u) {
    return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
}

template <typename T>
__global__ void __launch_bounds__(256) attn_delta_kernel(const T* o, int64_t ldo, int64_t o_bs, const T* dout, int64_t lddo,
                                                         int64_t do_bs, float* delta, int heads, int Nq, int64_t total) {
    griddep_launch_dependents();
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    griddep_wait();
    if (t >= total) return;
    const int h = (int)(t % heads);
    const int64_t bq = t / heads;
    const int q = (int)(bq % Nq);
    const int64_t b = bq / Nq;
    const uint4* po = reinterpret_cast<const uint4*>(o + b * o_bs + (int64_t)q * ldo + h * HD);
    const uint4* pd = reinterpret_cast<const uint4*>(dout + b * do_bs + (int64_t)q * lddo + h * HD);
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) {
        const uint4 a = po[i], d = pd[i];
        const uint32_t av[4] = {a.x, a.y, a.z, a.w}, dv[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 fa = unpack2<T>(av[j]), fd = unpack2<T>(dv[j]);
            acc = fmaf(fa.x, fd.x, acc);
            acc = fmaf(fa.y, fd.y, acc);
        }
    }
    delta[(b * heads + h) * Nq + q] = acc;
}

// Shared memory of both kernels: own tiles A, B (128 rows each), the ring of streamed 64-row tiles X, Y, per stage the
// streamed queries' lse * log2(e) and delta (dK / dV kernel), then the barriers.
struct BwdSmem {
    uint32_t sA, sB, sX, sY, own_full, bars;
    float* vec;
    __device__ BwdSmem(uint8_t* raw) {
        sA = (smem_u32(raw) + 1023u) & ~1023u;
        sB = sA + Q_BYTES; sX = sB + Q_BYTES; sY = sX + BWD_STAGES * KV_BYTES;
        const uint32_t sVec = sY + BWD_STAGES * KV_BYTES;
        vec = reinterpret_cast<float*>(raw + (sVec - smem_u32(raw)));
        own_full = sVec + BWD_STAGES * VEC_BYTES;
        bars = own_full + 8u;
    }
    __device__ uint32_t full(int s) const { return bars + 8u * s; }
    __device__ uint32_t empty(int s) const { return bars + 8u * (BWD_STAGES + s); }
    __device__ float* lse2(int s) const { return vec + s * 2 * AK; }
    __device__ float* delta(int s) const { return vec + s * 2 * AK + AK; }
};

// Barrier init, PDL wait, and the producer warp (which returns true: its caller exits).  With lse != nullptr the producer
// also stages the streamed queries' lse * log2(e) and delta, bound-checked against Nq: queries past Nq get lse = +inf, so
// their P is 0 however TMA filled the tile.  Every lane arrives on `full` after its own stores (count 32).
__device__ __forceinline__ bool bwd_prologue_and_produce(const BwdSmem& sm, const CUtensorMap* tA, const CUtensorMap* tB,
                                                         const CUtensorMap* tX, const CUtensorMap* tY, int own_row, int nblk,
                                                         const float* lse, const float* delta, int Nq) {
    griddep_launch_dependents();
    if (threadIdx.x == 0) {
        prefetch_tmap(tA); prefetch_tmap(tB); prefetch_tmap(tX); prefetch_tmap(tY);
        mbar_init(sm.own_full, 1);
        for (int s = 0; s < BWD_STAGES; ++s) { mbar_init(sm.full(s), 32); mbar_init(sm.empty(s), 2); }
        fence_mbar_init();
    }
    __syncthreads();
    griddep_wait();      // PDL: inputs written by the previous kernels are visible from here
    if ((threadIdx.x >> 5) != 8) return false;
    const int lane = threadIdx.x & 31, col = blockIdx.y * HD, b = blockIdx.z;
    if (lane == 0) {
        mbar_expect_tx(sm.own_full, 2 * Q_BYTES);
        tma_load_3d(sm.sA, tA, sm.own_full, col, own_row, b);
        tma_load_3d(sm.sB, tB, sm.own_full, col, own_row, b);
    }
    int stage = 0; uint32_t phase = 0;
    for (int j = 0; j < nblk; ++j) {
        mbar_wait(sm.empty(stage), phase ^ 1u);
        if (lse) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int i = 2 * lane + e, q = j * AK + i;
                sm.lse2(stage)[i] = q < Nq ? lse[q] * 1.4426950408889634f : INFINITY;
                sm.delta(stage)[i] = q < Nq ? delta[q] : 0.f;
            }
        }
        if (lane == 0) {
            mbar_expect_tx(sm.full(stage), 2 * KV_BYTES);
            tma_load_3d(sm.sX + stage * KV_BYTES, tX, sm.full(stage), col, j * AK, b);
            tma_load_3d(sm.sY + stage * KV_BYTES, tY, sm.full(stage), col, j * AK, b);
        } else {
            mbar_arrive(sm.full(stage));
        }
        if (++stage == BWD_STAGES) { stage = 0; phase ^= 1u; }
    }
    return true;
}

// rows r and r + 8 of a warpgroup's 64 x 64 fp32 fragment, scaled, to a [rows, ld] 16-bit matrix (rows >= nrows dropped)
template <typename T>
__device__ __forceinline__ void store_frag(const float (&acc)[32], float s, T* base, int64_t ld, int row0, int nrows) {
    const int lane = threadIdx.x & 31, quad_col = 2 * (lane & 3);
    const int row = row0 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (row + 8 * h >= nrows) continue;
        T* r = base + (int64_t)(row + 8 * h) * ld;
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj)
            *reinterpret_cast<uint32_t*>(r + 8 * jj + quad_col) = PK<T>::pack(acc[4 * jj + 2 * h] * s, acc[4 * jj + 2 * h + 1] * s);
    }
}

// own tiles A = K, B = V (keys [128 kt, +128)); streamed X = Q, Y = dO (64-query blocks)
template <typename T>
__global__ void __launch_bounds__(ATT_THREADS, 1) attn_dkdv_kernel(const __grid_constant__ CUtensorMap tmK,
                                                                   const __grid_constant__ CUtensorMap tmV,
                                                                   const __grid_constant__ CUtensorMap tmQ,
                                                                   const __grid_constant__ CUtensorMap tmdO,
                                                                   const BwdParams p) {
    extern __shared__ uint8_t smem_raw[];
    const BwdSmem sm(smem_raw);
    const int k_tile = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
    const int nqb = (p.Nq + AK - 1) / AK;
    const int64_t bh = ((int64_t)b * p.heads + head) * p.Nq;
    if (bwd_prologue_and_produce(sm, &tmK, &tmV, &tmQ, &tmdO, k_tile * AQ, nqb, p.lse + bh, p.delta + bh, p.Nq)) return;

    const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
    const int quad_col = 2 * (lane & 3);
    const uint64_t dK = make_sw128_desc(sm.sA + (uint32_t)wg * (64 * 128));
    const uint64_t dV = make_sw128_desc(sm.sB + (uint32_t)wg * (64 * 128));
    float dk[HD / 2], dv[HD / 2];
#pragma unroll
    for (int c = 0; c < HD / 2; ++c) { dk[c] = 0.f; dv[c] = 0.f; }
    mbar_wait(sm.own_full, 0);
    int stage = 0; uint32_t phase = 0;
    for (int j = 0; j < nqb; ++j) {
        mbar_wait(sm.full(stage), phase);
        // S^T first: P^T is packed to 16 bits before dP^T is computed, so S^T and dP^T are never live together
        float s[AK / 2];
#pragma unroll
        for (int c = 0; c < AK / 2; ++c) s[c] = 0.f;
        const uint32_t xq = sm.sX + stage * KV_BYTES, xdo = sm.sY + stage * KV_BYTES;
        const uint64_t dQb = make_sw128_desc(xq), ddOb = make_sw128_desc(xdo);
        const uint64_t ddOmn = make_sw128_desc_mn(xdo), dQmn = make_sw128_desc_mn(xq);
        const float* lse2 = sm.lse2(stage);
        const float* dlt = sm.delta(stage);
        wgmma_fence();
        wgmma_fence_operands(s);
#pragma unroll
        for (int k = 0; k < HD / 16; ++k) Wgmma<AK, T>::ss(s, dK + (uint64_t)(2 * k), dQb + (uint64_t)(2 * k));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operands(s);
        // element c sits at query column 8 (c / 4) + quad_col + c % 2 of the block; the accumulator fragment of columns
        // [16kk, 16kk+16) is the A-operand fragment of k-step kk
        uint32_t ap[AK / 16][4];
#pragma unroll
        for (int kk = 0; kk < AK / 16; ++kk)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int i = 16 * kk + 8 * (r >> 1) + quad_col;
                ap[kk][r] = PK<T>::pack(fast_exp2(fmaf(s[8 * kk + 2 * r], p.scale_log2e, -lse2[i])),
                                        fast_exp2(fmaf(s[8 * kk + 2 * r + 1], p.scale_log2e, -lse2[i + 1])));
            }
        float dp[AK / 2];
#pragma unroll
        for (int c = 0; c < AK / 2; ++c) dp[c] = 0.f;
        wgmma_fence();
        wgmma_fence_operands(dp);
        wgmma_fence_operands(dv);
#pragma unroll
        for (int k = 0; k < HD / 16; ++k) Wgmma<AK, T>::ss(dp, dV + (uint64_t)(2 * k), ddOb + (uint64_t)(2 * k));
#pragma unroll
        for (int kk = 0; kk < AK / 16; ++kk) Wgmma<HD, T>::rs_bt(dv, ap[kk], ddOmn + (uint64_t)(128 * kk));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operands(dp);
        wgmma_fence_operands(dv);
        // dS^T / scale = P^T o (dP^T - delta), with the 16-bit P^T that dV used
        uint32_t ads[AK / 16][4];
#pragma unroll
        for (int kk = 0; kk < AK / 16; ++kk)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int i = 16 * kk + 8 * (r >> 1) + quad_col;
                const float2 pr = unpack2<T>(ap[kk][r]);
                ads[kk][r] = PK<T>::pack(pr.x * (dp[8 * kk + 2 * r] - dlt[i]), pr.y * (dp[8 * kk + 2 * r + 1] - dlt[i + 1]));
            }
        wgmma_fence();
        wgmma_fence_operands(dk);
#pragma unroll
        for (int kk = 0; kk < AK / 16; ++kk) Wgmma<HD, T>::rs_bt(dk, ads[kk], dQmn + (uint64_t)(128 * kk));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operands(dk);
        if ((threadIdx.x & 127) == 0) mbar_arrive(sm.empty(stage));
        if (++stage == BWD_STAGES) { stage = 0; phase ^= 1u; }
    }
    const int row0 = k_tile * AQ + wg * 64;
    store_frag<T>(dk, p.scale, reinterpret_cast<T*>(p.dk) + (int64_t)b * p.dk_bs + head * HD, p.lddk, row0, p.Nk);
    store_frag<T>(dv, 1.f, reinterpret_cast<T*>(p.dv) + (int64_t)b * p.dv_bs + head * HD, p.lddv, row0, p.Nk);
}

// own tiles A = Q, B = dO (queries [128 qt, +128)); streamed X = K, Y = V (64-key blocks)
template <typename T>
__global__ void __launch_bounds__(ATT_THREADS, 1) attn_dq_kernel(const __grid_constant__ CUtensorMap tmQ,
                                                                 const __grid_constant__ CUtensorMap tmdO,
                                                                 const __grid_constant__ CUtensorMap tmK,
                                                                 const __grid_constant__ CUtensorMap tmV,
                                                                 const BwdParams p) {
    extern __shared__ uint8_t smem_raw[];
    const BwdSmem sm(smem_raw);
    const int q_tile = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
    const int nkb = (p.Nk + AK - 1) / AK;
    if (bwd_prologue_and_produce(sm, &tmQ, &tmdO, &tmK, &tmV, q_tile * AQ, nkb, nullptr, nullptr, 0)) return;

    const int warp = threadIdx.x >> 5, wg = warp >> 2, lane = threadIdx.x & 31;
    const int quad_col = 2 * (lane & 3);
    const uint64_t dQ = make_sw128_desc(sm.sA + (uint32_t)wg * (64 * 128));
    const uint64_t ddO = make_sw128_desc(sm.sB + (uint32_t)wg * (64 * 128));
    const int row = q_tile * AQ + wg * 64 + (warp & 3) * 16 + (lane >> 2);
    float lse2[2], dlt[2];   // rows row, row + 8; rows >= Nq are never stored, lse = +inf keeps them finite
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int64_t i = ((int64_t)b * p.heads + head) * p.Nq + row + 8 * h;
        lse2[h] = row + 8 * h < p.Nq ? p.lse[i] * 1.4426950408889634f : INFINITY;
        dlt[h] = row + 8 * h < p.Nq ? p.delta[i] : 0.f;
    }
    float dq[HD / 2];
#pragma unroll
    for (int c = 0; c < HD / 2; ++c) dq[c] = 0.f;
    mbar_wait(sm.own_full, 0);
    int stage = 0; uint32_t phase = 0;
    for (int j = 0; j < nkb; ++j) {
        mbar_wait(sm.full(stage), phase);
        float s[AK / 2], dp[AK / 2];
#pragma unroll
        for (int c = 0; c < AK / 2; ++c) { s[c] = 0.f; dp[c] = 0.f; }
        const uint32_t xk = sm.sX + stage * KV_BYTES, xv = sm.sY + stage * KV_BYTES;
        const uint64_t dKb = make_sw128_desc(xk), dVb = make_sw128_desc(xv);
        wgmma_fence();
        wgmma_fence_operands(s);
        wgmma_fence_operands(dp);
#pragma unroll
        for (int k = 0; k < HD / 16; ++k) Wgmma<AK, T>::ss(s, dQ + (uint64_t)(2 * k), dKb + (uint64_t)(2 * k));
#pragma unroll
        for (int k = 0; k < HD / 16; ++k) Wgmma<AK, T>::ss(dp, ddO + (uint64_t)(2 * k), dVb + (uint64_t)(2 * k));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operands(s);
        wgmma_fence_operands(dp);
        const int kvalid = p.Nk - j * AK;    // keys >= Nk (zero-filled K / V) get P = 0
#pragma unroll
        for (int c = 0; c < AK / 2; ++c) {
            const int h = (c >> 1) & 1;
            const float pr = 8 * (c >> 2) + quad_col + (c & 1) < kvalid ? fast_exp2(fmaf(s[c], p.scale_log2e, -lse2[h])) : 0.f;
            dp[c] = pr * (dp[c] - dlt[h]);                             // dS / scale
        }
        uint32_t a[AK / 16][4];
#pragma unroll
        for (int kk = 0; kk < AK / 16; ++kk)
#pragma unroll
            for (int r = 0; r < 4; ++r) a[kk][r] = PK<T>::pack(dp[8 * kk + 2 * r], dp[8 * kk + 2 * r + 1]);
        const uint64_t dKmn = make_sw128_desc_mn(xk);
        wgmma_fence();
        wgmma_fence_operands(dq);
#pragma unroll
        for (int kk = 0; kk < AK / 16; ++kk) Wgmma<HD, T>::rs_bt(dq, a[kk], dKmn + (uint64_t)(128 * kk));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operands(dq);
        if ((threadIdx.x & 127) == 0) mbar_arrive(sm.empty(stage));
        if (++stage == BWD_STAGES) { stage = 0; phase ^= 1u; }
    }
    store_frag<T>(dq, p.scale, reinterpret_cast<T*>(p.dq) + (int64_t)b * p.dq_bs + head * HD, p.lddq, q_tile * AQ + wg * 64, p.Nq);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int encode3(CUtensorMap* m, int bf16, const void* base, uint64_t cols, uint64_t rows, uint64_t batch, uint64_t ld,
            uint64_t bs, uint32_t box_rows) {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr; cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)ptr;
    }
    if (!fn) { dm_set_error("cuTensorMapEncodeTiled unavailable"); return DM_EDRIVER; }
    cuuint64_t gd[3] = {cols, rows, batch};
    cuuint64_t gs[2] = {ld * 2, bs * 2};
    cuuint32_t bx[3] = {HD, box_rows, 1}, es[3] = {1, 1, 1};
    CUresult r = fn(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), gd, gs,
                    bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { dm_set_error("attention tensor map encode failed (%d)", (int)r); return DM_EDRIVER; }
    return DM_OK;
}

}  // namespace

extern "C" int dm_tune_attention(int mode) {
    if (mode == 0) return DM_OK;
    dm_set_error("dm_tune_attention: mode %d does not exist (0 = fp32 exponentials, rescale every block)", mode);
    return DM_EINVAL;
}

extern "C" int dm_attention(int bf16, const void* q, int64_t ldq, int64_t q_batch_stride, const void* k, const void* v,
                            int64_t ldkv, int64_t kv_batch_stride, void* out, int64_t ldo, int64_t out_batch_stride,
                            int batch, int heads, int Nq, int Nk, int head_dim, float scale, void* stream) {
    DM_REQUIRE(q && k && v && out, "null pointer");
    DM_REQUIRE(head_dim == HD, "head_dim 64 only (VAE mid-block attention uses the GEMM path)");
    DM_REQUIRE(bf16 >= 0 && bf16 <= 2, "dtype selector: 0 fp16, 1 bf16, 2 fp32");
    if (bf16 == 2)   // fp32 storage (high-precision mode): SIMT online-softmax kernel of dense_hp.cu
        return hp_attention((const float*)q, ldq, q_batch_stride, (const float*)k, (const float*)v, ldkv, kv_batch_stride,
                            (float*)out, ldo, out_batch_stride, batch, heads, Nq, Nk, scale, stream);
    DM_REQUIRE(ldq % 8 == 0 && ldkv % 8 == 0 && ldo % 8 == 0, "row strides must be multiples of 8 elements");
    DM_REQUIRE(Nq > 0 && Nk > 0 && batch > 0 && heads > 0, "sizes");
    CUtensorMap tq, tk, tv;
    int rc = encode3(&tq, bf16, q, (uint64_t)heads * HD, (uint64_t)Nq, (uint64_t)batch, (uint64_t)ldq, (uint64_t)q_batch_stride, AQ); if (rc) return rc;
    rc = encode3(&tk, bf16, k, (uint64_t)heads * HD, (uint64_t)Nk, (uint64_t)batch, (uint64_t)ldkv, (uint64_t)kv_batch_stride, AK); if (rc) return rc;
    rc = encode3(&tv, bf16, v, (uint64_t)heads * HD, (uint64_t)Nk, (uint64_t)batch, (uint64_t)ldkv, (uint64_t)kv_batch_stride, AK); if (rc) return rc;
    AttnParams p;
    p.Nq = Nq; p.Nk = Nk; p.heads = heads; p.out = out; p.ldo = ldo; p.out_batch_stride = out_batch_stride;
    p.scale_log2e = scale * 1.4426950408889634f;
    dim3 grid((unsigned)dm_ceil_div(Nq, AQ), (unsigned)heads, (unsigned)batch);
    static bool cfg_h = false, cfg_b = false;
    if (bf16) {
        if (!cfg_b) { DM_CHECK_CUDA(cudaFuncSetAttribute(attention_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM)); cfg_b = true; }
        DM_CHECK_CUDA(dm_launch(attention_kernel<__nv_bfloat16>, grid, dim3(ATT_THREADS), (size_t)ATT_SMEM, (cudaStream_t)stream, tq, tk, tv, p));
    } else {
        if (!cfg_h) { DM_CHECK_CUDA(cudaFuncSetAttribute(attention_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM)); cfg_h = true; }
        DM_CHECK_CUDA(dm_launch(attention_kernel<__half>, grid, dim3(ATT_THREADS), (size_t)ATT_SMEM, (cudaStream_t)stream, tq, tk, tv, p));
    }
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_attention_lse(int bf16, const void* q, int64_t ldq, int64_t q_batch_stride, const void* k, const void* v,
                                int64_t ldkv, int64_t kv_batch_stride, void* out, int64_t ldo, int64_t out_batch_stride,
                                int batch, int heads, int Nq, int Nk, int head_dim, float scale, float* lse, void* stream) {
    DM_REQUIRE(q && k && v && out && lse, "null pointer");
    DM_REQUIRE(head_dim == HD, "head_dim 64 only");
    DM_REQUIRE(bf16 >= 0 && bf16 <= 2, "dtype selector: 0 fp16, 1 bf16, 2 fp32");
    if (bf16 == 2) { dm_set_error("dm_attention_lse: fp32 storage has no attention backward"); return DM_EUNSUPPORTED; }
    DM_REQUIRE(Nq > 0 && Nk > 0 && batch > 0 && heads > 0 && batch <= 65535 && heads <= 65535, "sizes");
    const int64_t lds[3] = {ldq, ldkv, ldo}, bss[3] = {q_batch_stride, kv_batch_stride, out_batch_stride};
    for (int i = 0; i < 3; ++i) {
        DM_REQUIRE(lds[i] % 8 == 0 && lds[i] >= (int64_t)heads * HD, "row strides must be multiples of 8 elements and at least heads * 64");
        DM_REQUIRE(bss[i] % 8 == 0 && bss[i] >= 0, "batch strides must be non-negative multiples of 8 elements");
    }
    const void* ptrs[4] = {q, k, v, out};
    for (int i = 0; i < 4; ++i) DM_REQUIRE(((uintptr_t)ptrs[i] & 15) == 0, "16-bit operands must be 16-byte aligned");
    DM_REQUIRE(((uintptr_t)lse & 3) == 0, "lse must be 4-byte aligned");
    CUtensorMap tq, tk, tv;
    int rc = encode3(&tq, bf16, q, (uint64_t)heads * HD, (uint64_t)Nq, (uint64_t)batch, (uint64_t)ldq, (uint64_t)q_batch_stride, AQ); if (rc) return rc;
    rc = encode3(&tk, bf16, k, (uint64_t)heads * HD, (uint64_t)Nk, (uint64_t)batch, (uint64_t)ldkv, (uint64_t)kv_batch_stride, AK); if (rc) return rc;
    rc = encode3(&tv, bf16, v, (uint64_t)heads * HD, (uint64_t)Nk, (uint64_t)batch, (uint64_t)ldkv, (uint64_t)kv_batch_stride, AK); if (rc) return rc;
    AttnParams p;
    p.Nq = Nq; p.Nk = Nk; p.heads = heads; p.out = out; p.ldo = ldo; p.out_batch_stride = out_batch_stride;
    p.scale_log2e = scale * 1.4426950408889634f;
    p.lse = lse;
    dim3 grid((unsigned)dm_ceil_div(Nq, AQ), (unsigned)heads, (unsigned)batch);
    static bool cfg_h = false, cfg_b = false;
    if (bf16) {
        if (!cfg_b) { DM_CHECK_CUDA(cudaFuncSetAttribute(attention_kernel<__nv_bfloat16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM)); cfg_b = true; }
        DM_CHECK_CUDA(dm_launch(attention_kernel<__nv_bfloat16, true>, grid, dim3(ATT_THREADS), (size_t)ATT_SMEM, (cudaStream_t)stream, tq, tk, tv, p));
    } else {
        if (!cfg_h) { DM_CHECK_CUDA(cudaFuncSetAttribute(attention_kernel<__half, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM)); cfg_h = true; }
        DM_CHECK_CUDA(dm_launch(attention_kernel<__half, true>, grid, dim3(ATT_THREADS), (size_t)ATT_SMEM, (cudaStream_t)stream, tq, tk, tv, p));
    }
    DM_CHECK_LAUNCH();
    return DM_OK;
}

namespace {
template <typename T>
int attention_bwd_launch(const CUtensorMap (&own_q)[2], const CUtensorMap (&blk_q)[2], const CUtensorMap (&own_k)[2],
                         const CUtensorMap (&blk_k)[2], const void* o, int64_t ldo, int64_t o_bs, const void* dout,
                         int64_t lddo, int64_t do_bs, const BwdParams& p, int batch, cudaStream_t st) {
    static bool cfg = false;
    if (!cfg) {
        DM_CHECK_CUDA(cudaFuncSetAttribute(attn_dkdv_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM));
        DM_CHECK_CUDA(cudaFuncSetAttribute(attn_dq_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM));
        cfg = true;
    }
    const int64_t total = (int64_t)batch * p.heads * p.Nq;
    DM_CHECK_CUDA(dm_launch(attn_delta_kernel<T>, dim3((unsigned)dm_ceil_div(total, 256)), dim3(256), 0, st, (const T*)o, ldo,
                            o_bs, (const T*)dout, lddo, do_bs, const_cast<float*>(p.delta), p.heads, p.Nq, total));
    DM_CHECK_LAUNCH();
    DM_CHECK_CUDA(dm_launch(attn_dkdv_kernel<T>, dim3((unsigned)dm_ceil_div(p.Nk, AQ), (unsigned)p.heads, (unsigned)batch),
                            dim3(ATT_THREADS), (size_t)BWD_SMEM, st, own_k[0], own_k[1], blk_q[0], blk_q[1], p));
    DM_CHECK_LAUNCH();
    DM_CHECK_CUDA(dm_launch(attn_dq_kernel<T>, dim3((unsigned)dm_ceil_div(p.Nq, AQ), (unsigned)p.heads, (unsigned)batch),
                            dim3(ATT_THREADS), (size_t)BWD_SMEM, st, own_q[0], own_q[1], blk_k[0], blk_k[1], p));
    DM_CHECK_LAUNCH();
    return DM_OK;
}
}  // namespace

extern "C" int dm_attention_bwd(int bf16, const void* q, int64_t ldq, int64_t q_batch_stride, const void* k, const void* v,
                                int64_t ldkv, int64_t kv_batch_stride, const void* o, int64_t ldo, int64_t o_batch_stride,
                                const void* dout, int64_t lddo, int64_t do_batch_stride, const float* lse, void* dq,
                                int64_t lddq, int64_t dq_batch_stride, void* dk, int64_t lddk, int64_t dk_batch_stride,
                                void* dv, int64_t lddv, int64_t dv_batch_stride, float* delta, int batch, int heads, int Nq,
                                int Nk, int head_dim, float scale, void* stream) {
    DM_REQUIRE(bf16 >= 0 && bf16 <= 2, "dtype selector: 0 fp16, 1 bf16, 2 fp32");
    if (bf16 == 2) { dm_set_error("dm_attention_bwd: fp32 storage is not supported (16-bit tensor-core kernel)"); return DM_EUNSUPPORTED; }
    DM_REQUIRE(q && k && v && o && dout && lse && dq && dk && dv && delta, "null pointer");
    DM_REQUIRE(head_dim == HD, "head_dim 64 only");
    DM_REQUIRE(Nq > 0 && Nk > 0 && batch > 0 && heads > 0 && batch <= 65535 && heads <= 65535, "sizes");
    const int64_t C = (int64_t)heads * HD;
    const int64_t lds[7] = {ldq, ldkv, ldo, lddo, lddq, lddk, lddv};
    const int64_t bss[7] = {q_batch_stride, kv_batch_stride, o_batch_stride, do_batch_stride, dq_batch_stride, dk_batch_stride, dv_batch_stride};
    for (int i = 0; i < 7; ++i) {
        DM_REQUIRE(lds[i] % 8 == 0 && lds[i] >= C, "row strides must be multiples of 8 elements and at least heads * 64");
        DM_REQUIRE(bss[i] % 8 == 0 && bss[i] >= 0, "batch strides must be non-negative multiples of 8 elements");
    }
    const void* ptrs[9] = {q, k, v, o, dout, dq, dk, dv, nullptr};
    for (int i = 0; ptrs[i]; ++i) DM_REQUIRE(((uintptr_t)ptrs[i] & 15) == 0, "16-bit operands must be 16-byte aligned");
    DM_REQUIRE(((uintptr_t)lse & 3) == 0 && ((uintptr_t)delta & 3) == 0, "lse / delta must be 4-byte aligned");
    CUtensorMap own_q[2], blk_q[2], own_k[2], blk_k[2];
    const uint64_t cols = (uint64_t)C;
    int rc;
    if ((rc = encode3(&own_q[0], bf16, q, cols, Nq, batch, ldq, q_batch_stride, AQ))) return rc;
    if ((rc = encode3(&own_q[1], bf16, dout, cols, Nq, batch, lddo, do_batch_stride, AQ))) return rc;
    if ((rc = encode3(&blk_q[0], bf16, q, cols, Nq, batch, ldq, q_batch_stride, AK))) return rc;
    if ((rc = encode3(&blk_q[1], bf16, dout, cols, Nq, batch, lddo, do_batch_stride, AK))) return rc;
    if ((rc = encode3(&own_k[0], bf16, k, cols, Nk, batch, ldkv, kv_batch_stride, AQ))) return rc;
    if ((rc = encode3(&own_k[1], bf16, v, cols, Nk, batch, ldkv, kv_batch_stride, AQ))) return rc;
    if ((rc = encode3(&blk_k[0], bf16, k, cols, Nk, batch, ldkv, kv_batch_stride, AK))) return rc;
    if ((rc = encode3(&blk_k[1], bf16, v, cols, Nk, batch, ldkv, kv_batch_stride, AK))) return rc;
    BwdParams p;
    p.Nq = Nq; p.Nk = Nk; p.heads = heads; p.lse = lse; p.delta = delta;
    p.dq = dq; p.lddq = lddq; p.dq_bs = dq_batch_stride;
    p.dk = dk; p.lddk = lddk; p.dk_bs = dk_batch_stride;
    p.dv = dv; p.lddv = lddv; p.dv_bs = dv_batch_stride;
    p.scale = scale; p.scale_log2e = scale * 1.4426950408889634f;
    return bf16 ? attention_bwd_launch<__nv_bfloat16>(own_q, blk_q, own_k, blk_k, o, ldo, o_batch_stride, dout, lddo,
                                                      do_batch_stride, p, batch, (cudaStream_t)stream)
                : attention_bwd_launch<__half>(own_q, blk_q, own_k, blk_k, o, ldo, o_batch_stride, dout, lddo, do_batch_stride,
                                               p, batch, (cudaStream_t)stream);
}
