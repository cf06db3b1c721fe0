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

template <typename T>
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
        const float inv = 1.0f / quad_sum(l_run[h]);
        if (q >= p.Nq) continue;
        T* orow = reinterpret_cast<T*>(p.out) + (int64_t)b * p.out_batch_stride + (int64_t)q * p.ldo + head * HD;
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj)
            *reinterpret_cast<uint32_t*>(orow + 8 * jj + quad_col) = PK<T>::pack(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    }
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
