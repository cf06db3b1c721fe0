// tc_gemm.cu -- wgmma tensor-core GEMM / implicit-GEMM convolution for sm_90a.
//
// Every dense contraction of the VAE encoder, the UNet and the ControlNet runs through this file
// (rows a7/a8 of SURVEY.md section 8; reference call sites models/guidance/dreammat_guidance.py:
// 218-229 ControlNetModel.forward, :274-282 UNet2DConditionModel.forward, :290 AutoencoderKL.encode,
// which run cuDNN/cuBLAS kernels through diffusers):
//
//   D[M,N] = epilogue( A[M,K] . B[N,K]^T )        fp16 or bf16 operands, fp32 accumulation in registers
//
//   * linear / 1x1 conv : A = activations [batch, M, K] through a 3-D TMA map
//   * 3x3 conv (NHWC)   : A is never materialised (no im2col).  The K loop walks (tap, 64-channel
//                         slab); each step TMA-loads a shifted 4-D box {64 ch, tile_w, tile_h, tile_n}
//                         of the input, out-of-bounds rows/cols zero-filled by the TMA unit = padding.
//                         Stride-2 convs use the map's element strides.
//   * B = weights [N, K] (K-major), K index = tap * Cin + c.
//
// tc_gemm_kernel<BN,T>: persistent, warp-specialised, one CTA per SM walking 128 x BN output tiles.  CTA = 544 threads:
// warps 0-7 are two MMA warpgroups (rows 0-63 / 64-127 of the tile, m64nBNk16 wgmma with both operands in shared
// memory), warps 8-15 are two epilogue warpgroups (two threads per tile row), warp 16 is the TMA producer.  Operand tiles
// live in the 128-byte swizzled K-major layout shared by TMA and the wgmma descriptors; a ring of mbarrier-guarded stages
// lets the producer run ahead across tile boundaries.  After a tile's K loop the MMA warpgroups hand the accumulators to
// the epilogue warpgroups through a shared-memory staging tile (mbarriers epi_full / epi_empty) and start the next tile's
// K loop at once, so the epilogue (fused bias / per-image vector / residual / SiLU / GELU / GEGLU / scale, or a split-K
// partial tile), which reads whole output rows, overlaps the next tile's loads and MMAs.  A 16-bit output moves by TMA:
// residual boxes are loaded into a shared output tile, combined in place and stored as boxes (see the epilogue role).
// choose_tile() picks the tile width and split-K.
//
// Weight gradients (dm_conv2d_wgrad / dm_gemm_wgrad) run the same kernel in its WGRAD mode: D[Cout, taps*Cin] (fp32) reduces
// over the pixel / token axis, with both operands MN-major boxes of the NHWC / token-major dY and x (see WG_BOX).
// Input gradients (dm_conv2d_dgrad / dm_gemm_dgrad) run it in its DGRAD mode: A = dY exactly as a forward activation, B =
// MN-major boxes of the forward weight itself (see MODE_DGRAD), so no flipped / transposed weight copy ever exists.
#include <cuda.h>
#include <cuda_bf16.h>
#include "common.cuh"
#include "tc_common.cuh"

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int MMA_THREADS = 256;                              // two MMA warpgroups
constexpr int EPI_THREADS = 2 * BM;                           // two epilogue warpgroups: two threads per tile row
constexpr int NTHREADS = MMA_THREADS + EPI_THREADS + 32;      // + the TMA producer warp

struct GemmParams {
    int M, N, K;                  // GEMM view; conv: M = n_img*Ho*Wo, K = taps*Cin
    int batch;                    // grid.z (plain GEMM only)
    int b_batched;                // B indexed by blockIdx.z as well
    int is_conv, Cin, taps, kw_n; // kw_n = kernel width (3 or 1)
    int Ho, Wo, tile_w, tile_h, tile_n;
    int stride, pad_t, pad_l;
    // epilogue
    void* out; int ldc; int64_t out_batch_stride; int out_f32;
    int tma_out;                  // 16-bit output (and residual) tiles move by TMA through shared memory (see dispatch)
    const void* bias;                       // [N]
    const void* rowvec; int rows_per_vec; int ld_rowvec;   // [M / rows_per_vec, N]
    const void* residual; int ld_res; int64_t res_batch_stride;
    float alpha;                            // applied to the accumulator first
    float out_scale;                        // applied last
    int act;                                // 0 none, 1 silu, 2 gelu(erf), 3 geglu (interleaved value|gate)
    int split_k; float* ws;                 // split-K: split sp stores its fp32 partial tile in slice sp of ws[S][batch][M][N]; splitk_finish_kernel sums the slices in order and applies the epilogue
    // fused CSD epilogue of the UNet's conv_out (dm_conv2d_csd): rows are [branch][view][pixel]; a CTA walks the three
    // branch tiles of the same 128 pixels back to back and combines them in registers
    int csd; int csd_B; int csd_hw; int csd_groups;       // csd_groups = B*hw / 128 row tiles per branch
    const float* csd_noise; const float* csd_w; const float* csd_coef;   // coef[5] = c_text, c_uncond, c_null, c_noise, dlat_scale (device)
    float* csd_grad; float* csd_dlat; float* csd_norms; float* csd_eps;
};

// i-th tile of this CTA (persistent walk); -1 past the end.  Plain mode: t = first + i * step.  CSD mode: the walk
// visits GROUPS of three row tiles (k * groups + g, k = branch) so that one CTA sees all three noise predictions of a pixel.
__device__ __forceinline__ int tile_at(const GemmParams& p, int i, int first, int step, int total_tiles) {
    if (!p.csd) { const int t = first + i * step; return t < total_tiles ? t : -1; }
    const int g = first + (i / 3) * step;
    return g < p.csd_groups ? (i % 3) * p.csd_groups + g : -1;
}

template <typename T> struct Cvt;
template <> struct Cvt<__half> {
    static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
    static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
};
template <> struct Cvt<__nv_bfloat16> {
    static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
    static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};

// The fp32 staging tile has BN floats per row, without padding.  Its 16-byte chunks are XOR-swizzled by the row
// (chunk ^ epi_swz(row)), so that both the MMA warps' fragment stores (rows r..r+3 x 8 columns per half-warp) and the
// epilogue's row reads (8 consecutive rows per quarter-warp) touch 32 distinct banks.
__device__ __forceinline__ int epi_swz(int row) { const int k = row & 7; return ((k & 3) << 1) | (k >> 2); }
__device__ __forceinline__ int epi_idx(int row, int col) { return ((((col >> 2) ^ epi_swz(row))) << 2) + (col & 3); }

// R staging columns c0 .. c0 + R - 1 of the row starting at `er`, whose swizzle is sw
template <int R>
__device__ __forceinline__ void ld_row(const float* er, int sw, int c0, float (&f)[R]) {
#pragma unroll
    for (int q = 0; q < R / 4; ++q) {
        const float4 t = reinterpret_cast<const float4*>(er)[((c0 >> 2) + q) ^ sw];
        f[4 * q] = t.x; f[4 * q + 1] = t.y; f[4 * q + 2] = t.z; f[4 * q + 3] = t.w;
    }
}

// The 16-bit output tile in shared memory (TMA path): BN / 32 boxes of 128 rows x 32 columns (8 KB each, 64 bytes per
// row) in the TMA map's 64-byte swizzle.  Byte offset of 16-byte chunk q (columns 8q .. 8q + 7) of `row` in a box; the
// 8 rows of a quarter-warp hit 8 distinct bank groups.
constexpr int OBOX_BYTES = BM * 64;
__device__ __forceinline__ int obox_off(int row, int q) { return row * 64 + ((q ^ ((row >> 1) & 3)) << 4); }

// f[j] += vec[n0 + j] for the 8 columns n0 .. n0 + 7; columns >= N are skipped
template <typename T>
__device__ __forceinline__ void add8(float* f, const T* vec, int n0, int N) {
    if (n0 + 8 <= N && ((uintptr_t)(vec + n0) & 15) == 0) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(vec + n0));
        const T* h = reinterpret_cast<const T*>(&u);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] += Cvt<T>::to_f(h[j]);
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) if (n0 + j < N) f[j] += Cvt<T>::to_f(vec[n0 + j]);
    }
}

// Epilogue of one output row of a 128 x BN tile: `er` is the row's fp32 accumulator in the staging tile (swizzle sw);
// this thread handles the column chunks c0 = c_first, c_first + c_step, ... (32 wide, 64 for GEGLU):
// acc*alpha + bias + rowvec -> act -> + residual -> * out_scale -> 16-bit output.  On the TMA path (p.tma_out) the
// residual is read from, and the output written to, the shared output tile `ot` (row `row` of each 32-column box); the
// caller stores the boxes.  Otherwise both go straight to global memory with 16-byte accesses where aligned.
template <int BN, typename T>
__device__ __forceinline__ void epilogue_row(const GemmParams& p, const float* er, int sw, uint8_t* ot, int row, int64_t m,
                                             int z, int sp, int n_tile, int c_first, int c_step) {
    const bool row_ok = m < p.M;
    if (!row_ok) return;
    if (p.ws) {
        // split-K partial tile: raw fp32 sums into this split's own slice (no atomics: the finish kernel adds the slices in a
        // fixed order, so the result does not depend on which split finishes first); the epilogue proper runs there
        const int64_t slice = (int64_t)(p.batch > 0 ? p.batch : 1) * p.M * p.N;
        float* wrow = p.ws + sp * slice + ((int64_t)z * p.M + m) * p.N;
#pragma unroll 1
        for (int c0 = c_first; c0 < BN; c0 += c_step) {
            const int n0 = n_tile * BN + c0;
            if (n0 >= p.N) continue;
            float v[32];
            ld_row<32>(er, sw, c0, v);
            if (n0 + 32 <= p.N && (p.N & 3) == 0) {
#pragma unroll
                for (int q = 0; q < 8; ++q)
                    reinterpret_cast<float4*>(wrow + n0)[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
            } else {
#pragma unroll
                for (int j = 0; j < 32; ++j) if (n0 + j < p.N) wrow[n0 + j] = v[j];
            }
        }
        return;
    }
    const T* bias = (const T*)p.bias;
    const T* rowvec = p.rowvec ? (const T*)p.rowvec + (int64_t)(m / p.rows_per_vec) * p.ld_rowvec : nullptr;
    const T* res = p.residual ? (const T*)p.residual + (int64_t)z * p.res_batch_stride + m * (int64_t)p.ld_res : nullptr;
    char* outp = (char*)p.out + ((int64_t)z * p.out_batch_stride + m * (int64_t)p.ldc) * (p.out_f32 ? 4 : 2);
    if (p.act == 3) {
        // GEGLU epilogue: the weight rows come interleaved as [32 value | 32 gate] blocks (host side,
        // dense_ops.geglu_interleave), so every 64 accumulator columns give 32 outputs value * gelu(gate)
        // and the [M, N] projection never goes to HBM.  Output row length is N / 2.
#pragma unroll 1
        for (int c0 = c_first; c0 < BN; c0 += c_step) {
            const int n0 = n_tile * BN + c0;
            if (n0 >= p.N) continue;
            T* o = reinterpret_cast<T*>(outp) + (n0 >> 1);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                float a[8], b[8];
                ld_row<8>(er, sw, c0 + 8 * q, a);
                ld_row<8>(er, sw, c0 + 32 + 8 * q, b);
#pragma unroll
                for (int j = 0; j < 8; ++j) { a[j] *= p.alpha; b[j] *= p.alpha; }
                if (bias) { add8(a, bias, n0 + q * 8, p.N); add8(b, bias, n0 + 32 + q * 8, p.N); }
                uint4 u;
                T* h = reinterpret_cast<T*>(&u);
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    h[j] = Cvt<T>::from_f(a[j] * (0.5f * b[j] * (1.0f + erff(b[j] * 0.70710678118654752f))) * p.out_scale);
                if (p.tma_out) *reinterpret_cast<uint4*>(ot + (c0 >> 6) * OBOX_BYTES + obox_off(row, q)) = u;
                else if ((p.ldc & 7) == 0) reinterpret_cast<uint4*>(o)[q] = u;
                else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) o[8 * q + j] = h[j];
                }
            }
        }
        return;
    }
#pragma unroll 1
    for (int c0 = c_first; c0 < BN; c0 += c_step) {
        const int n0 = n_tile * BN + c0;
        if (n0 >= p.N) continue;
        float f[32];
        ld_row<32>(er, sw, c0, f);
#pragma unroll
        for (int j = 0; j < 32; ++j) f[j] *= p.alpha;
        const bool full = (n0 + 32 <= p.N);
        if (bias) {
#pragma unroll
            for (int q = 0; q < 4; ++q) add8(f + 8 * q, bias, n0 + 8 * q, p.N);
        }
        if (rowvec) {
#pragma unroll
            for (int q = 0; q < 4; ++q) add8(f + 8 * q, rowvec, n0 + 8 * q, p.N);
        }
        if (p.act == 1) {
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] = f[j] / (1.0f + __expf(-f[j]));
        } else if (p.act == 2) {
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] = 0.5f * f[j] * (1.0f + erff(f[j] * 0.70710678118654752f));
        }
        uint8_t* obox = ot + (c0 >> 5) * OBOX_BYTES;
        if (p.tma_out) {
            // residual chunks were loaded into the box by TMA (zeros past N / M); each chunk is read and then
            // overwritten with the output by this thread, and the box store clips to [M, N]
            if (res) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const uint4 u = *reinterpret_cast<const uint4*>(obox + obox_off(row, q));
                    const T* h = reinterpret_cast<const T*>(&u);
#pragma unroll
                    for (int j = 0; j < 8; ++j) f[q * 8 + j] += Cvt<T>::to_f(h[j]);
                }
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                uint4 u;
                T* h = reinterpret_cast<T*>(&u);
#pragma unroll
                for (int j = 0; j < 8; ++j) h[j] = Cvt<T>::from_f(f[q * 8 + j] * p.out_scale);
                *reinterpret_cast<uint4*>(obox + obox_off(row, q)) = u;
            }
            continue;
        }
        if (res) {
            if (full && ((p.ld_res & 7) == 0)) {
                const uint4* r4 = reinterpret_cast<const uint4*>(res + n0);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    uint4 u = r4[q];
                    const T* h = reinterpret_cast<const T*>(&u);
#pragma unroll
                    for (int j = 0; j < 8; ++j) f[q * 8 + j] += Cvt<T>::to_f(h[j]);
                }
            } else {
#pragma unroll
                for (int j = 0; j < 32; ++j) if (n0 + j < p.N) f[j] += Cvt<T>::to_f(res[n0 + j]);
            }
        }
#pragma unroll
        for (int j = 0; j < 32; ++j) f[j] *= p.out_scale;
        if (p.out_f32) {
            float* o = reinterpret_cast<float*>(outp) + n0;
            if (full && ((p.ldc & 3) == 0)) {
#pragma unroll
                for (int q = 0; q < 8; ++q) reinterpret_cast<float4*>(o)[q] = make_float4(f[4 * q], f[4 * q + 1], f[4 * q + 2], f[4 * q + 3]);
            } else {
#pragma unroll
                for (int j = 0; j < 32; ++j) if (n0 + j < p.N) o[j] = f[j];
            }
        } else {
            T* o = reinterpret_cast<T*>(outp) + n0;
            if (full && ((p.ldc & 7) == 0)) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    uint4 u;
                    T* h = reinterpret_cast<T*>(&u);
#pragma unroll
                    for (int j = 0; j < 8; ++j) h[j] = Cvt<T>::from_f(f[q * 8 + j]);
                    reinterpret_cast<uint4*>(o)[q] = u;
                }
            } else {
#pragma unroll
                for (int j = 0; j < 32; ++j) if (n0 + j < p.N) o[j] = Cvt<T>::from_f(f[j]);
            }
        }
    }
}

// CSD epilogue (dreammat_guidance.py:475-481 compute_grad_sds tail, :584 nan_to_num, the 8 logged norms of :483-495 and
// loss_sds of :590-594) on the accumulator row of branch k = 0 text | 1 uncond | 2 null.  The thread's row is pixel
// r = g*128 + row of the [view][pixel] axis; its 4 noise predictions (rounded to the storage dtype like the reference's
// `.sample` in weights_dtype) wait in `e` until the third branch arrives, then
//   grad = nan_to_num(w[b] * (c_t e_text + c_u e_uncond + c_n e_null + c_s noise)),  dlatents = grad * dlat_scale
// are written (NCHW fp32) and the ten squared sums are reduced per warp and added to norms[10].
template <typename T>
__device__ __forceinline__ void epilogue_csd(const GemmParams& p, const float* er, int64_t m, int lane, float (&e)[2][4]) {
    const int64_t per_branch = (int64_t)p.csd_groups * BM;
    const int k = (int)(m / per_branch);
    const int64_t r = m - (int64_t)k * per_branch;
    const int b = (int)(r / p.csd_hw), px = (int)(r - (int64_t)b * p.csd_hw);
    const T* bias = (const T*)p.bias;
    float cur[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        float f = er[c];
        if (bias) f += Cvt<T>::to_f(bias[c]);
        cur[c] = Cvt<T>::to_f(Cvt<T>::from_f(f));
        if (p.csd_eps) p.csd_eps[(((int64_t)k * p.csd_B + b) * 4 + c) * p.csd_hw + px] = cur[c];
    }
    if (k < 2) {
#pragma unroll
        for (int c = 0; c < 4; ++c) e[k][c] = cur[c];
        return;
    }
    const float ct = p.csd_coef[0], cu = p.csd_coef[1], cn = p.csd_coef[2], cs = p.csd_coef[3], ds = p.csd_coef[4];
    const float wb = p.csd_w[b];
    float acc[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int64_t o = ((int64_t)b * 4 + c) * p.csd_hw + px;
        const float et = e[0][c], eu = e[1][c], en = cur[c], nz = p.csd_noise[o];
        float g = wb * (ct * et + cu * eu + cn * en + cs * nz);
        if (isnan(g)) g = 0.f; else if (isinf(g)) g = g > 0 ? 3.4028234663852886e38f : -3.4028234663852886e38f;
        if (p.csd_grad) p.csd_grad[o] = g;
        if (p.csd_dlat) p.csd_dlat[o] = g * ds;
        acc[0] += 0.5f * g * g; acc[1] += g * g;
        acc[2] += (eu - nz) * (eu - nz); acc[3] += (et - nz) * (et - nz); acc[4] += (et - eu) * (et - eu);
        acc[5] += (et - en) * (et - en); acc[6] += (en - eu) * (en - eu);
        acc[7] += nz * nz; acc[8] += eu * eu; acc[9] += et * et;
    }
#pragma unroll
    for (int q = 0; q < 10; ++q) {
        const float sum = warp_sum(acc[q]);
        if (lane == q) atomicAdd(p.csd_norms + q, sum);
    }
}

// ~128 KB operand ring + the fp32 staging tile of the epilogue (swizzled, see epi_idx) + the 16-bit output tile.
template <int BN> struct Cfg {
    static constexpr int A_BYTES = BM * BK * 2;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = 131072 / STAGE_BYTES;        // 4 (BN = 128) or 5 (BN = 64)
    static constexpr int EPI_BYTES = BM * BN * 4;
    static constexpr int OUT_BYTES = (BN / 32) * OBOX_BYTES;
    static constexpr int SMEM = STAGES * STAGE_BYTES + EPI_BYTES + OUT_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(SMEM <= 227 * 1024, "shared memory budget");
};

// Weight-gradient mode (WG): D[M' = Cout, N' = taps*Cin] = sum over K' = pixels (tokens) of dY[K', M'] . x_tap[K', N'].
// Both operands are MN-major: a stage holds 64 pixels (one K-block) of each, as 64-channel TMA boxes of 64 rows x 128 B
// straight from the NHWC / token-major buffers: two boxes of dY (the 128 rows of the tile, one per MMA warpgroup) and
// BN / 64 boxes of x, each loaded at its own tap's shifted origin.  Out-of-bounds pixels (padding, the ragged end of the
// pixel axis) are zero-filled by TMA in both operands.
constexpr int WG_BOX = 64 * 128;                     // bytes of one 64-channel x 64-pixel box
constexpr int WG_PIX = 64;                           // pixels per K-block

// Input-gradient mode (DGRAD): D[M = pixels (tokens), N = Cin (K_in)] = sum over K = (tap, co) of dY . W, with the B
// operand read from the forward weight W[Cout, taps*Cin] ([N_out, K_in] for a linear) as it is.  A is dY, K-major, loaded
// like a forward activation (a conv shifts it by k-1-pad, the host passes that as the padding).  For K-block (tap, 64
// output channels co) and the tile's input channels ci0.., B is BN / 64 MN-major boxes of 64 contiguous ci x 64 rows co
// at column (taps-1-tap)*Cin + ci0: the tap flip of the transposed convolution is a coordinate.  The K order (tap-major,
// then co) and every product are those of the forward kernel on a flipped, transposed weight copy, so the result is
// bit-identical to it.  Columns of a box past Cin hold the next tap's weights (or TMA zeros): they only reach output
// columns >= N, which the epilogue drops.
constexpr int MODE_FWD = 0, MODE_WGRAD = 1, MODE_DGRAD = 2;

// Persistent kernel: grid = min(#tiles, #SMs); every CTA walks tiles t = blockIdx.x, +gridDim.x, ...
template <int BN, typename T, int MODE = MODE_FWD>
__global__ void __launch_bounds__(NTHREADS, 1) tc_gemm_kernel(const __grid_constant__ CUtensorMap tmA,
                                                             const __grid_constant__ CUtensorMap tmB,
                                                             const __grid_constant__ CUtensorMap tmO,
                                                             const __grid_constant__ CUtensorMap tmR,
                                                             const GemmParams p) {
    using C = Cfg<BN>;
    constexpr bool WG = MODE == MODE_WGRAD, DG = MODE == MODE_DGRAD;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t raw_u32 = smem_u32(smem_raw);
    const uint32_t smem_base = (raw_u32 + 1023u) & ~1023u;
    float* epi = reinterpret_cast<float*>(smem_raw + (smem_base - raw_u32) + C::STAGES * C::STAGE_BYTES);
    uint8_t* otile = reinterpret_cast<uint8_t*>(epi) + C::EPI_BYTES;
    const uint32_t otile_u32 = smem_base + C::STAGES * C::STAGE_BYTES + C::EPI_BYTES;
    const uint32_t bar_base = otile_u32 + C::OUT_BYTES;
    // barriers: full[STAGES] (TMA bytes landed), empty[STAGES] (both MMA warpgroups done reading), epi_full (the staging
    // tile holds a tile's accumulators), epi_empty (the epilogue warpgroups have finished reading them), res_full[2]
    // (TMA path: epilogue warpgroup h's boxes of the output tile are free and hold the tile's residual, if any)
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (C::STAGES + s); };
    const uint32_t epi_full = bar_base + 16u * C::STAGES, epi_empty = epi_full + 8u;
    auto res_full = [&](int h) { return epi_full + 16u + 8u * h; };

    griddep_launch_dependents();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nk = p.K / BK;
    const int n_tiles = (p.N + BN - 1) / BN, m_tiles = (p.M + BM - 1) / BM;
    const int tiles_per_z = n_tiles * m_tiles;
    const int S = p.split_k > 1 ? p.split_k : 1;       // split-K: S CTAs share an output tile, partial sums go to p.ws
    const int total_tiles = tiles_per_z * (p.batch > 0 ? p.batch : 1) * S;

    if (threadIdx.x == 0) {
        prefetch_tmap(&tmA);
        prefetch_tmap(&tmB);
        if (p.tma_out) {
            prefetch_tmap(&tmO);
            if (p.residual) prefetch_tmap(&tmR);
        }
        for (int s = 0; s < C::STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 2); }
        mbar_init(epi_full, MMA_THREADS / 32);      // one arrival per warp (lane 0, after __syncwarp)
        mbar_init(epi_empty, EPI_THREADS / 32);
        mbar_init(res_full(0), 1);
        mbar_init(res_full(1), 1);
        fence_mbar_init();
    }
    __syncthreads();
    griddep_wait();      // PDL: everything above overlapped the previous kernel's tail; its outputs are visible from here

    if (warp == (MMA_THREADS + EPI_THREADS) / 32) {
        if (lane == 0 && WG) {
            // ------------------------------------------------ TMA producer, weight-gradient mode
            const int tiles_w = p.is_conv ? p.Wo / p.tile_w : 1, tiles_h = p.is_conv ? p.Ho / p.tile_h : 1;
            int stage = 0; uint32_t phase = 0;
            for (int i = 0, t; (t = tile_at(p, i, blockIdx.x, gridDim.x, total_tiles)) >= 0; ++i) {
                const int sp = t % S, r = t / S;
                const int m_tile = r / n_tiles, n_tile = r - m_tile * n_tiles;
                const int kb0 = (int)((int64_t)sp * nk / S), kb1 = (int)((int64_t)(sp + 1) * nk / S);
                // boxes wholly past Cout / N' are not loaded: they would only feed rows / columns the epilogue drops
                const int a_boxes = min(2, (p.M - m_tile * BM + 63) / 64), b_boxes = min(BN / 64, (p.N - n_tile * BN + 63) / 64);
                for (int kb = kb0; kb < kb1; ++kb) {
                    mbar_wait(empty_bar(stage), phase ^ 1u);
                    const uint32_t a_dst = smem_base + stage * C::STAGE_BYTES;
                    const uint32_t b_dst = a_dst + C::A_BYTES;
                    mbar_expect_tx(full_bar(stage), (uint32_t)(a_boxes + b_boxes) * WG_BOX);
                    if (p.is_conv) {
                        const int tw = kb % tiles_w, th = (kb / tiles_w) % tiles_h, tn = kb / (tiles_w * tiles_h);
                        const int ow0 = tw * p.tile_w, oh0 = th * p.tile_h, n0 = tn * p.tile_n;
                        for (int h = 0; h < a_boxes; ++h)
                            tma_load_4d(a_dst + h * WG_BOX, &tmA, full_bar(stage), m_tile * BM + 64 * h, ow0, oh0, n0);
                        for (int j = 0; j < b_boxes; ++j) {
                            // a 128-wide tile may straddle two taps: each 64-channel box takes its own tap's shift
                            const int col = n_tile * BN + 64 * j, tap = col / p.Cin, kh = tap / p.kw_n, kw = tap - kh * p.kw_n;
                            tma_load_4d(b_dst + j * WG_BOX, &tmB, full_bar(stage), col - tap * p.Cin,
                                        ow0 * p.stride - p.pad_l + kw, oh0 * p.stride - p.pad_t + kh, n0);
                        }
                    } else {
                        for (int h = 0; h < a_boxes; ++h)
                            tma_load_3d(a_dst + h * WG_BOX, &tmA, full_bar(stage), m_tile * BM + 64 * h, kb * WG_PIX, 0);
                        for (int j = 0; j < b_boxes; ++j)
                            tma_load_3d(b_dst + j * WG_BOX, &tmB, full_bar(stage), n_tile * BN + 64 * j, kb * WG_PIX, 0);
                    }
                    if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
                }
            }
        } else if (lane == 0) {
            // ------------------------------------------------ TMA producer
            const int slabs = p.is_conv ? (p.Cin / BK) : nk;
            const int tiles_w = p.is_conv ? p.Wo / p.tile_w : 1, tiles_h = p.is_conv ? p.Ho / p.tile_h : 1;
            int stage = 0; uint32_t phase = 0;
            for (int i = 0, t; (t = tile_at(p, i, blockIdx.x, gridDim.x, total_tiles)) >= 0; ++i) {
                const int sp = t % S, tt = t / S;
                const int z = tt / tiles_per_z, r = tt - z * tiles_per_z;
                const int m_tile = r / n_tiles, n_tile = r - m_tile * n_tiles;
                const int kb0 = (int)((int64_t)sp * nk / S), kb1 = (int)((int64_t)(sp + 1) * nk / S);
                int c_n = 0, c_h = 0, c_w = 0;
                if (p.is_conv) {
                    int tw = m_tile % tiles_w, th = (m_tile / tiles_w) % tiles_h, tn = m_tile / (tiles_w * tiles_h);
                    c_w = tw * p.tile_w * p.stride - p.pad_l;
                    c_h = th * p.tile_h * p.stride - p.pad_t;
                    c_n = tn * p.tile_n;
                }
                for (int kb = kb0; kb < kb1; ++kb) {
                    mbar_wait(empty_bar(stage), phase ^ 1u);
                    const uint32_t a_dst = smem_base + stage * C::STAGE_BYTES;
                    const uint32_t b_dst = a_dst + C::A_BYTES;
                    // DGRAD: weight boxes wholly past N are not loaded (they would only feed columns the epilogue drops)
                    const int b_boxes = DG ? min(BN / 64, (p.N - n_tile * BN + 63) / 64) : 0;
                    mbar_expect_tx(full_bar(stage), DG ? (uint32_t)(C::A_BYTES + b_boxes * WG_BOX) : (uint32_t)C::STAGE_BYTES);
                    int tap = 0, slab = kb;
                    if (p.is_conv) {
                        tap = kb / slabs; slab = kb - tap * slabs;
                        int kh = tap / p.kw_n, kw = tap - kh * p.kw_n;
                        tma_load_4d(a_dst, &tmA, full_bar(stage), slab * BK, c_w + kw, c_h + kh, c_n);
                    } else {
                        tma_load_3d(a_dst, &tmA, full_bar(stage), kb * BK, m_tile * BM, z);
                    }
                    if constexpr (DG) {
                        for (int j = 0; j < b_boxes; ++j)
                            tma_load_3d(b_dst + j * WG_BOX, &tmB, full_bar(stage), (p.taps - 1 - tap) * p.N + n_tile * BN + 64 * j, slab * BK, 0);
                    } else {
                        tma_load_3d(b_dst, &tmB, full_bar(stage), kb * BK, n_tile * BN, p.b_batched ? z : 0);
                    }
                    if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
                }
            }
        }
        return;
    }
    uint32_t epi_phase = 0;
    if (threadIdx.x >= MMA_THREADS) {
        // ---------------------------------------------------- epilogue warpgroups: threads row and row + 128 share a tile row
        const int row = threadIdx.x & (BM - 1), half = (threadIdx.x - MMA_THREADS) >> 7;
        const int sw = epi_swz(row);
        const float* er = epi + row * BN;
        const int step = p.act == 3 ? 64 : 32;
        // TMA path: warpgroup `half` owns the output boxes of its chunks c0 = half * step + 2 * step * k (box c0 / step;
        // GEGLU writes 32 outputs per 64-column chunk) and runs their round trip: its leader thread loads the residual
        // boxes of a tile into shared memory, the warpgroup adds them in place, the leader stores the boxes and, once
        // the store has read them, loads the next tile's residual (or just releases the boxes when there is none).
        const bool leader = (threadIdx.x & 127) == 0;
        const uint32_t rbar = res_full(half);
        auto fill = [&](int t) {
            const int z = (t / S) / tiles_per_z, r_ = (t / S) - z * tiles_per_z;
            const int m_tile = r_ / n_tiles, n_tile = r_ - m_tile * n_tiles;
            if (!p.residual) { mbar_arrive(rbar); return; }
            uint32_t bytes = 0;
            for (int c0 = half * step; c0 < BN; c0 += 2 * step) if (n_tile * BN + c0 < p.N) bytes += OBOX_BYTES;
            mbar_expect_tx(rbar, bytes);
            for (int c0 = half * step; c0 < BN; c0 += 2 * step)
                if (n_tile * BN + c0 < p.N) tma_load_3d(otile_u32 + (c0 / step) * OBOX_BYTES, &tmR, rbar, n_tile * BN + c0, m_tile * BM, z);
        };
        uint32_t res_phase = 0;
        if (p.tma_out && leader) {
            const int t0 = tile_at(p, 0, blockIdx.x, gridDim.x, total_tiles);
            if (t0 >= 0) fill(t0);
        }
        float csd_e[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
        for (int i = 0, t; (t = tile_at(p, i, blockIdx.x, gridDim.x, total_tiles)) >= 0; ++i) {
            const int sp = t % S, tt = t / S;
            const int z = tt / tiles_per_z, r_ = tt - z * tiles_per_z;
            const int m_tile = r_ / n_tiles, n_tile = r_ - m_tile * n_tiles;
            const int64_t m = (int64_t)m_tile * BM + row;
            mbar_wait(epi_full, epi_phase);
            if (p.tma_out) mbar_wait(rbar, res_phase);
            if (BN == 64 && p.csd) {
                if (half == 0) epilogue_csd<T>(p, er + (sw << 2), m, lane, csd_e);     // csd_e carries a pixel's branches
            } else {
                epilogue_row<BN, T>(p, er, sw, otile, row, m, z, sp, n_tile, half * step, 2 * step);   // GEGLU chunks are 64 wide
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(epi_empty);
            epi_phase ^= 1u;
            if (p.tma_out) {
                fence_proxy_async_smem();
                named_bar_sync(1 + half, 128);
                if (leader) {
                    const int n_out0 = p.act == 3 ? (n_tile * BN) / 2 : n_tile * BN;
                    for (int c0 = half * step; c0 < BN; c0 += 2 * step)
                        if (n_tile * BN + c0 < p.N) tma_store_3d(&tmO, otile_u32 + (c0 / step) * OBOX_BYTES, n_out0 + (c0 / step) * 32, m_tile * BM, z);
                    bulk_commit();
                    bulk_wait_read();
                    const int tn = tile_at(p, i + 1, blockIdx.x, gridDim.x, total_tiles);
                    if (tn >= 0) fill(tn);
                }
                res_phase ^= 1u;
            }
        }
        if (p.tma_out && leader) bulk_wait_all();     // dependent kernels (PDL) read the output
        return;
    }
    // -------------------------------------------------------- MMA warpgroups 0 / 1
    const int wg = warp >> 2;
    const int frag_row = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // accumulator fragment rows frag_row, frag_row + 8
    const int frag_col = 2 * (lane & 3);
    int stage = 0; uint32_t phase = 0;
    float acc[BN / 2];
    for (int i = 0, t; (t = tile_at(p, i, blockIdx.x, gridDim.x, total_tiles)) >= 0; ++i) {
        const int sp = t % S;
        const int kb0 = (int)((int64_t)sp * nk / S), kb1 = (int)((int64_t)(sp + 1) * nk / S);
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
        int prev = -1;
        for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait(full_bar(stage), phase);
            const uint32_t a_addr = smem_base + stage * C::STAGE_BYTES;
            // WG: MN-major, warpgroup wg's 64 rows are dY box wg, B spans BN / 64 boxes WG_BOX apart, and a K step of 16
            // pixel rows is +2048 bytes (+128 in the descriptor's 16-byte units)
            const uint64_t da = WG ? make_sw128_desc_mn(a_addr + (uint32_t)wg * WG_BOX, WG_BOX)
                                   : make_sw128_desc(a_addr + (uint32_t)wg * (64 * 128));
            const uint64_t db = (WG || DG) ? make_sw128_desc_mn(a_addr + C::A_BYTES, WG_BOX) : make_sw128_desc(a_addr + C::A_BYTES);
            wgmma_fence();
            wgmma_fence_operands(acc);
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
                if constexpr (WG) Wgmma<BN, T>::ss_tt(acc, da + (uint64_t)(128 * k), db + (uint64_t)(128 * k));
                else if constexpr (DG) Wgmma<BN, T>::ss_nt(acc, da + (uint64_t)(2 * k), db + (uint64_t)(128 * k));
                else Wgmma<BN, T>::ss(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k));
            }
            wgmma_commit();
            wgmma_fence_operands(acc);
            wgmma_wait<1>();                       // the previous k-block's MMAs are done: hand its stage back
            if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(empty_bar(prev));
            prev = stage;
            if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
        }
        wgmma_wait<0>();
        wgmma_fence_operands(acc);
        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(empty_bar(prev));
        mbar_wait(epi_empty, epi_phase ^ 1u);      // the epilogue warpgroups have finished reading the previous tile
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            *reinterpret_cast<float2*>(epi + frag_row * BN + epi_idx(frag_row, 8 * j + frag_col)) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(epi + (frag_row + 8) * BN + epi_idx(frag_row + 8, 8 * j + frag_col)) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(epi_full);
        epi_phase ^= 1u;
    }
}

// ------------------------------------------------------------------------------------- host side

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)ptr;
    }
    return fn;
}

int encode_map(CUtensorMap* m, int bf16, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
               const uint32_t* box, const uint32_t* estr, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
    EncodeTiledFn fn = get_encode();
    if (!fn) { dm_set_error("cuTensorMapEncodeTiled unavailable"); return DM_EDRIVER; }
    cuuint64_t gd[5]; cuuint64_t gs[4]; cuuint32_t bx[5]; cuuint32_t es[5];
    for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = estr[i]; }
    for (int i = 0; i < rank - 1; ++i) gs[i] = strides_bytes[i];
    CUresult r = fn(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank,
                    const_cast<void*>(base), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        dm_set_error("cuTensorMapEncodeTiled failed (%d) rank=%d dims=%llu,%llu,%llu,%llu box=%u,%u,%u,%u", (int)r, rank,
                     (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
                     (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
                     rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
        return DM_EDRIVER;
    }
    return DM_OK;
}

// A 16-bit [batch][M][ld] output or residual is addressable by TMA when its base and strides are multiples of 16 bytes.
int64_t out_batch_pitch(int M, int batch, int64_t ld, int64_t batch_stride) { return batch > 1 ? batch_stride : (int64_t)M * ld; }
bool tma_addressable(const void* base, int M, int batch, int64_t ld, int64_t batch_stride) {
    const int64_t zs = out_batch_pitch(M, batch, ld, batch_stride);
    return ((uintptr_t)base & 15) == 0 && (ld & 7) == 0 && (zs & 7) == 0 && zs > 0;
}
// its 3-D map [batch][M][n] for the TMA epilogue: 128 x 32 boxes in the 64-byte swizzle of obox_off
int out_map(CUtensorMap* m, int bf16, const void* base, int n, int M, int batch, int64_t ld, int64_t batch_stride) {
    uint64_t dims[3] = {(uint64_t)n, (uint64_t)M, (uint64_t)batch};
    uint64_t str[2] = {(uint64_t)ld * 2, (uint64_t)out_batch_pitch(M, batch, ld, batch_stride) * 2};
    uint32_t box[3] = {32, BM, 1}, es[3] = {1, 1, 1};
    return encode_map(m, bf16, base, 3, dims, str, box, es, CU_TENSOR_MAP_SWIZZLE_64B);
}

template <int BN, typename T, int MODE = MODE_FWD>
int launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, const CUtensorMap& tmR,
           const GemmParams& p, int64_t work_items, cudaStream_t st) {
    static bool configured = false;
    auto kern = tc_gemm_kernel<BN, T, MODE>;
    if (!configured) {
        DM_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::SMEM));
        configured = true;
    }
    unsigned grid = (unsigned)(work_items < DM_NUM_SMS ? work_items : DM_NUM_SMS);   // persistent: one CTA per SM
    DM_CHECK_CUDA(dm_launch(kern, dim3(grid), dim3(NTHREADS), (size_t)Cfg<BN>::SMEM, st, tmA, tmB, tmO, tmR, p));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

// ---- split-K: few-tile, long-K layers (8x8 / 16x16 latents of a one-view batch) leave most SMs idle; S CTAs share a tile,
// each stores its fp32 partial tile in its own workspace slice, and this kernel adds the S slices in order and applies the
// epilogue.
float* g_ws = nullptr;
size_t g_ws_floats = 0;
int g_gemm_splitk = 1;
constexpr size_t WS_FLOATS = 8u << 20;   // recommended size, 32 MB: S*M*N <= 8 M elements (dm_gemm_workspace_bytes)

// The workspace is owned by the caller (dm_gemm_set_workspace): no hidden allocation inside the library.  Without one,
// split-K is simply not used.
template <typename T>
__global__ void __launch_bounds__(256) splitk_finish_kernel(const GemmParams p) {
    griddep_launch_dependents();
    griddep_wait();
    const int64_t n4 = p.N >> 2;
    const int64_t total = (int64_t)(p.batch > 0 ? p.batch : 1) * p.M * n4;
    const T* bias = (const T*)p.bias;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / n4; const int c = (int)(i - row * n4) * 4;
        const int z = (int)(row / p.M); const int64_t m = row - (int64_t)z * p.M;
        const int64_t slice = total * 4;
        float4 a = *reinterpret_cast<const float4*>(p.ws + row * p.N + c);
        for (int sp = 1; sp < p.split_k; ++sp) {
            const float4 b = *reinterpret_cast<const float4*>(p.ws + sp * slice + row * p.N + c);
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        float f[4] = {a.x * p.alpha, a.y * p.alpha, a.z * p.alpha, a.w * p.alpha};
        if (bias) {
#pragma unroll
            for (int j = 0; j < 4; ++j) f[j] += Cvt<T>::to_f(bias[c + j]);
        }
        if (p.rowvec) {
            const T* rv = (const T*)p.rowvec + (m / p.rows_per_vec) * (int64_t)p.ld_rowvec;
#pragma unroll
            for (int j = 0; j < 4; ++j) f[j] += Cvt<T>::to_f(rv[c + j]);
        }
        if (p.act == 1) {
#pragma unroll
            for (int j = 0; j < 4; ++j) f[j] = f[j] / (1.0f + __expf(-f[j]));
        } else if (p.act == 2) {
#pragma unroll
            for (int j = 0; j < 4; ++j) f[j] = 0.5f * f[j] * (1.0f + erff(f[j] * 0.70710678118654752f));
        }
        if (p.residual) {
            const T* res = (const T*)p.residual + (int64_t)z * p.res_batch_stride + m * (int64_t)p.ld_res;
#pragma unroll
            for (int j = 0; j < 4; ++j) f[j] += Cvt<T>::to_f(res[c + j]);
        }
        const int64_t o = (int64_t)z * p.out_batch_stride + m * (int64_t)p.ldc + c;
        if (p.out_f32) {
#pragma unroll
            for (int j = 0; j < 4; ++j) reinterpret_cast<float*>(p.out)[o + j] = f[j] * p.out_scale;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) reinterpret_cast<T*>(p.out)[o + j] = Cvt<T>::from_f(f[j] * p.out_scale);
        }
    }
}

// ---- bias gradient of the weight-gradient mode: db[c] = sum over rows of dy[r, c], without atomics.  Block (cb, k) adds
// rows k*rows_per_part .. of columns 64cb .. 64cb + 63 in a fixed order (four row lanes, then the lanes in order) into
// partial row k; bias_grad_finish_kernel adds the partial rows in order.
template <typename T>
__global__ void __launch_bounds__(256) bias_grad_partial_kernel(const T* __restrict__ dy, int64_t ld, int64_t rows, int N,
                                                                int64_t rows_per_part, float* __restrict__ part) {
    griddep_launch_dependents();
    griddep_wait();
    __shared__ float red[4][64];
    const int cl = threadIdx.x & 63, q = threadIdx.x >> 6, c = blockIdx.x * 64 + cl;
    const int64_t r0 = (int64_t)blockIdx.y * rows_per_part, r1 = min(rows, r0 + rows_per_part);
    float s = 0.f;
    if (c < N)
        for (int64_t r = r0 + q; r < r1; r += 4) s += Cvt<T>::to_f(dy[r * ld + c]);
    red[q][cl] = s;
    __syncthreads();
    if (q == 0 && c < N) part[(int64_t)blockIdx.y * N + c] = ((red[0][cl] + red[1][cl]) + red[2][cl]) + red[3][cl];
}

__global__ void __launch_bounds__(256) bias_grad_finish_kernel(const float* __restrict__ part, int parts, int N, float* __restrict__ db) {
    griddep_launch_dependents();
    griddep_wait();
    const int c = blockIdx.x * 256 + threadIdx.x;
    if (c >= N) return;
    float s = 0.f;
    for (int k = 0; k < parts; ++k) s += part[(int64_t)k * N + c];
    db[c] = s;
}

int bias_grad(int bf16, const void* dy, int64_t ld, int64_t rows, int N, float* db, cudaStream_t st) {
    int64_t per = dm_ceil_div(rows, 256);                 // at most 256 partial rows, at least 128 dy rows each
    if (per < 128) per = 128;
    const int parts = (int)dm_ceil_div(rows, per);
    float* part = (float*)dm_scratch(DM_SCRATCH_WGRAD, (size_t)parts * N * sizeof(float), st);
    if (!part) return DM_EDRIVER;
    const dim3 grid((unsigned)dm_ceil_div(N, 64), (unsigned)parts);
    if (bf16) DM_CHECK_CUDA(dm_launch(bias_grad_partial_kernel<__nv_bfloat16>, grid, dim3(256), 0, st, (const __nv_bfloat16*)dy, ld, rows, N, per, part));
    else DM_CHECK_CUDA(dm_launch(bias_grad_partial_kernel<__half>, grid, dim3(256), 0, st, (const __half*)dy, ld, rows, N, per, part));
    DM_CHECK_LAUNCH();
    DM_CHECK_CUDA(dm_launch(bias_grad_finish_kernel, dim3((unsigned)dm_ceil_div(N, 256)), dim3(256), 0, st, (const float*)part, parts, N, db));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

struct TileChoice { int bn; int split; };   // split: 0 = let dispatch decide, >= 1 fixed

// Tile width: 64 when there are fewer 128 x 128 tiles than SMs (low-resolution UNet levels) or N <= 64, else 128.  The
// 128 x 128 tile keeps both warpgroups' m64n128 accumulators (64 fp32 registers per thread) and a four-stage operand ring
// in one SM; a 256-wide tile would not leave room for the epilogue's staging tile, so a 256 hint gets 128.
int pick_bn(int64_t M, int N, int bn_hint) {
    if (bn_hint == 64) return 64;
    if (bn_hint == 128 || bn_hint == 256) return 128;
    if (N <= 64) return 64;
    int64_t tiles128 = dm_ceil_div(M, BM) * dm_ceil_div(N, 128);
    if (tiles128 < (int64_t)DM_NUM_SMS && N % 64 == 0) return 64;
    return 128;
}

// split factor for `tiles` output tiles with nk K-blocks (1 = no split): only when at most half the SMs would have a
// tile and the K loop is long enough to amortise the workspace pass.  The split also keeps each CTA's accumulation chain
// near 64 K-blocks: the wgmma fp32 accumulator drifts over longer chains (fp32-mode error vs fp64 measured on the
// H100: 4.4e-6 at 60 blocks, 1.5e-5 at 160, 2.1e-5 at 360), which the 6x-long K of the fp32 mode would otherwise hit.
int pick_split(int64_t tiles, int nk, int64_t mn, int N, int act) {
    if (!g_gemm_splitk || act == 3 || (N & 3)) return 1;
    if (tiles * 2 > DM_NUM_SMS || nk < 32) return 1;
    int s = (int)(DM_NUM_SMS / tiles);
    if (s < (nk + 63) / 64) s = (nk + 63) / 64;
    if (s > nk / 8) s = nk / 8;
    if (s > 16) s = 16;
    if (g_ws != nullptr && (size_t)mn * s > g_ws_floats) s = (int)(g_ws_floats / (size_t)mn);   // one workspace slice per split
    if (s < 2 || g_ws == nullptr) return 1;
    return s;
}

TileChoice choose_tile(int64_t M, int N, int bn_hint) { return {pick_bn(M, N, bn_hint), 0}; }

int dispatch(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p_in, const TileChoice& tc, int bf16, cudaStream_t st,
             int mode = MODE_FWD) {
    GemmParams p = p_in;
    const int64_t batch = p.batch > 0 ? p.batch : 1;
    const int64_t tiles = dm_ceil_div(p.N, tc.bn) * dm_ceil_div(p.M, BM) * batch;
    const int split = tc.split >= 1 ? tc.split : pick_split(tiles, p.K / BK, batch * p.M * p.N, p.N, p.act);
    p.split_k = split;
    p.ws = split > 1 ? g_ws : nullptr;
    // The epilogue moves 16-bit output and residual tiles by TMA, except for fp32 output, split-K partial tiles and
    // rows whose pitch TMA cannot address; those keep per-thread global loads and stores.
    CUtensorMap tmO, tmR;
    memset(&tmO, 0, sizeof(tmO)); memset(&tmR, 0, sizeof(tmR));
    p.tma_out = split <= 1 && !p.out_f32 && tma_addressable(p.out, p.M, (int)batch, p.ldc, p.out_batch_stride) &&
                (!p.residual || tma_addressable(p.residual, p.M, (int)batch, p.ld_res, p.res_batch_stride));
    int rc;
    if (p.tma_out) {
        rc = out_map(&tmO, bf16, p.out, p.act == 3 ? p.N / 2 : p.N, p.M, (int)batch, p.ldc, p.out_batch_stride);
        if (rc) return rc;
        if (p.residual) {
            rc = out_map(&tmR, bf16, p.residual, p.N, p.M, (int)batch, p.ld_res, p.res_batch_stride);
            if (rc) return rc;
        }
    }
    const int64_t work = tiles * split;
    if (mode == MODE_WGRAD) {
        if (tc.bn == 64) rc = bf16 ? launch<64, __nv_bfloat16, MODE_WGRAD>(tmA, tmB, tmO, tmR, p, work, st) : launch<64, __half, MODE_WGRAD>(tmA, tmB, tmO, tmR, p, work, st);
        else rc = bf16 ? launch<128, __nv_bfloat16, MODE_WGRAD>(tmA, tmB, tmO, tmR, p, work, st) : launch<128, __half, MODE_WGRAD>(tmA, tmB, tmO, tmR, p, work, st);
    } else if (mode == MODE_DGRAD) {
        if (tc.bn == 64) rc = bf16 ? launch<64, __nv_bfloat16, MODE_DGRAD>(tmA, tmB, tmO, tmR, p, work, st) : launch<64, __half, MODE_DGRAD>(tmA, tmB, tmO, tmR, p, work, st);
        else rc = bf16 ? launch<128, __nv_bfloat16, MODE_DGRAD>(tmA, tmB, tmO, tmR, p, work, st) : launch<128, __half, MODE_DGRAD>(tmA, tmB, tmO, tmR, p, work, st);
    } else if (tc.bn == 64) rc = bf16 ? launch<64, __nv_bfloat16>(tmA, tmB, tmO, tmR, p, work, st) : launch<64, __half>(tmA, tmB, tmO, tmR, p, work, st);
    else rc = bf16 ? launch<128, __nv_bfloat16>(tmA, tmB, tmO, tmR, p, work, st) : launch<128, __half>(tmA, tmB, tmO, tmR, p, work, st);
    if (rc || split <= 1) return rc;
    const int64_t n4 = batch * p.M * (p.N >> 2);
    int64_t blocks = dm_ceil_div(n4, 256);
    if (blocks > DM_NUM_SMS * 8) blocks = DM_NUM_SMS * 8;
    if (bf16) DM_CHECK_CUDA(dm_launch(splitk_finish_kernel<__nv_bfloat16>, dim3((unsigned)blocks), dim3(256), 0, st, p));
    else DM_CHECK_CUDA(dm_launch(splitk_finish_kernel<__half>, dim3((unsigned)blocks), dim3(256), 0, st, p));
    DM_CHECK_LAUNCH();
    return DM_OK;
}

void fill_epilogue(GemmParams& p, const dm_epilogue* e, int N) {
    p.bias = e ? e->bias : nullptr;
    p.rowvec = e ? e->rowvec : nullptr;
    p.rows_per_vec = (e && e->rows_per_vec > 0) ? e->rows_per_vec : 1;
    p.ld_rowvec = (e && e->ld_rowvec > 0) ? e->ld_rowvec : N;
    p.residual = e ? e->residual : nullptr;
    p.ld_res = (e && e->ld_res > 0) ? e->ld_res : N;
    p.res_batch_stride = e ? e->res_batch_stride : 0;
    p.alpha = e ? e->alpha : 1.0f;
    p.out_scale = e ? e->out_scale : 1.0f;
    p.act = e ? e->act : 0;
    p.out_f32 = e ? e->out_f32 : 0;
}

// Weight gradient: p holds the GEMM view [M' = Cout, N', K' = 64 * pixel blocks] and the operand geometry; dW [M', N'] is
// written in fp32 (overwritten, row pitch N').  Planned by the forward's choose_tile / pick_split, so dm_gemm_plan(M', N',
// K') reports the tile and split this call uses; a split goes through the workspace slices and splitk_finish_kernel.
int wgrad_run(const CUtensorMap& tmA, const CUtensorMap& tmB, GemmParams& p, int bf16, float* dw, cudaStream_t st) {
    p.batch = 1;
    p.out = dw; p.ldc = p.N; p.out_f32 = 1;
    p.alpha = 1.0f; p.out_scale = 1.0f; p.rows_per_vec = 1;
    return dispatch(tmA, tmB, p, choose_tile(p.M, p.N, 0), bf16, st, MODE_WGRAD);
}

}  // namespace

// Pure query of the tile heuristic (no launch): which kernel / tile width / split-K a [M, N, K] contraction would get.
// kernel_out is always 0 (one single-CTA kernel); split_out is what pick_split would choose given the registered
// workspace.  Lets host-side tests pin the choices.
extern "C" int dm_gemm_plan(int64_t M, int N, int K, int act, int bn_hint, int* kernel_out, int* bn_out, int* split_out) {
    DM_REQUIRE(M > 0 && N > 0 && K > 0 && K % BK == 0 && kernel_out && bn_out && split_out, "bad args");
    TileChoice tc = choose_tile(M, N, bn_hint);
    *kernel_out = 0;
    *bn_out = tc.bn;
    *split_out = pick_split(dm_ceil_div(N, tc.bn) * dm_ceil_div(M, BM), K / BK, M * N, N, act);
    return DM_OK;
}

extern "C" size_t dm_gemm_workspace_bytes(void) { return WS_FLOATS * sizeof(float); }

extern "C" int dm_gemm_set_workspace(void* ptr, size_t bytes) {
    g_ws = (float*)ptr;
    g_ws_floats = ptr ? bytes / sizeof(float) : 0;
    return DM_OK;
}

extern "C" int dm_tune_gemm(int code) {
    if (code == 20 || code == 21) { g_gemm_splitk = code - 20; return DM_OK; }   // split-K of few-tile long-K layers: off | on
    dm_set_error("dm_tune_gemm: unknown code %d (20 / 21: split-K off / on)", code);
    return DM_EINVAL;
}

extern "C" int dm_gemm(int bf16, const void* A, int64_t lda, int64_t a_batch_stride, const void* B, int64_t ldb,
                       int64_t b_batch_stride, void* C, int64_t ldc, int64_t c_batch_stride, int M, int N, int K,
                       int batch, const dm_epilogue* ep, int bn_hint, void* stream) {
    DM_REQUIRE(A && B && C, "null pointer");
    DM_REQUIRE(bf16 == 0 || bf16 == 1, "16-bit operands only: fp32 storage goes through dm_hp_split -> bf16 GEMM -> dm_hp_epilogue");
    DM_REQUIRE(M > 0 && N > 0 && K > 0 && K % BK == 0, "K must be a positive multiple of 64");
    DM_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "row strides must be multiples of 8 elements (16 bytes)");
    DM_REQUIRE((((uintptr_t)A | (uintptr_t)B) & 15) == 0, "16-byte aligned operands");
    if (batch < 1) batch = 1;
    if (ep && ep->act == 3) {
        DM_REQUIRE(N % 64 == 0 && !ep->residual && !ep->rowvec && !ep->out_f32,
                   "GEGLU epilogue: N multiple of 64 (interleaved value/gate rows), 16-bit output of N/2 columns");
    }
    TileChoice tc = choose_tile((int64_t)M * batch, N, bn_hint);
    const int bn = tc.bn;
    CUtensorMap tmA, tmB;
    {
        uint64_t dims[3] = {(uint64_t)K, (uint64_t)M, (uint64_t)batch};
        uint64_t str[2] = {(uint64_t)lda * 2, (uint64_t)(batch > 1 ? a_batch_stride : (int64_t)M * lda) * 2};
        uint32_t box[3] = {BK, BM, 1}, es[3] = {1, 1, 1};
        int rc = encode_map(&tmA, bf16, A, 3, dims, str, box, es); if (rc) return rc;
    }
    {
        uint64_t dims[3] = {(uint64_t)K, (uint64_t)N, (uint64_t)(b_batch_stride ? batch : 1)};
        uint64_t str[2] = {(uint64_t)ldb * 2, (uint64_t)(b_batch_stride ? b_batch_stride : (int64_t)N * ldb) * 2};
        uint32_t box[3] = {BK, (uint32_t)bn, 1}, es[3] = {1, 1, 1};
        int rc = encode_map(&tmB, bf16, B, 3, dims, str, box, es); if (rc) return rc;
    }
    if (batch > 1 && !b_batch_stride) {
        // B shared across the batch: fold the batch into M (A, C and the residual must be densely stacked)
        bool dense = a_batch_stride == (int64_t)M * lda && c_batch_stride == (int64_t)M * ldc &&
                     (!ep || !ep->residual || ep->res_batch_stride == (int64_t)M * (ep->ld_res > 0 ? ep->ld_res : N));
        if (!dense) { dm_set_error("batched A with shared B requires densely stacked A/C/residual"); return DM_EUNSUPPORTED; }
        return dm_gemm(bf16, A, lda, 0, B, ldb, 0, C, ldc, 0, M * batch, N, K, 1, ep, bn_hint, stream);
    }
    GemmParams p; memset(&p, 0, sizeof(p));
    p.M = M; p.N = N; p.K = K; p.batch = batch; p.b_batched = (batch > 1) ? 1 : 0; p.is_conv = 0;
    p.out = C; p.ldc = (int)ldc; p.out_batch_stride = c_batch_stride;
    fill_epilogue(p, ep, N);
    return dispatch(tmA, tmB, p, tc, bf16, (cudaStream_t)stream);
}

extern "C" int dm_conv2d(int bf16, const void* x, int n_img, int H, int W, int Cin, const void* w, int Cout, int ksize,
                         int stride, int pad_t, int pad_l, int Ho, int Wo, void* y, int64_t ldc, const dm_epilogue* ep,
                         int bn_hint, void* stream) {
    DM_REQUIRE(x && w && y, "null pointer");
    DM_REQUIRE(bf16 == 0 || bf16 == 1, "16-bit operands only: fp32 storage goes through dm_hp_split -> bf16 conv -> dm_hp_epilogue");
    DM_REQUIRE(Cin % BK == 0, "Cin must be a multiple of 64 (pad the channels)");
    DM_REQUIRE(ksize == 3 || ksize == 1, "3x3 or 1x1");
    DM_REQUIRE(stride == 1 || stride == 2, "stride 1 or 2");
    int tile_w = Wo < BM ? Wo : BM;
    int tile_h = (BM / tile_w) < Ho ? (BM / tile_w) : Ho;
    int tile_n = BM / (tile_w * tile_h);
    DM_REQUIRE(tile_w * tile_h * tile_n == BM && Wo % tile_w == 0 && Ho % tile_h == 0,
               "output extent must tile into 128-pixel boxes (power-of-two sizes)");
    TileChoice tc = choose_tile((int64_t)n_img * Ho * Wo, Cout, bn_hint);
    const int bn = tc.bn;
    CUtensorMap tmA, tmB;
    {
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)n_img};
        uint64_t str[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
        uint32_t box[4] = {BK, (uint32_t)(tile_w * stride), (uint32_t)(tile_h * stride), (uint32_t)tile_n};
        uint32_t es[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
        int rc = encode_map(&tmA, bf16, x, 4, dims, str, box, es); if (rc) return rc;
    }
    int K = ksize * ksize * Cin;
    {
        uint64_t dims[3] = {(uint64_t)K, (uint64_t)Cout, 1};
        uint64_t str[2] = {(uint64_t)K * 2, (uint64_t)K * Cout * 2};
        uint32_t box[3] = {BK, (uint32_t)bn, 1}, es[3] = {1, 1, 1};
        int rc = encode_map(&tmB, bf16, w, 3, dims, str, box, es); if (rc) return rc;
    }
    GemmParams p; memset(&p, 0, sizeof(p));
    p.M = n_img * Ho * Wo; p.N = Cout; p.K = K; p.batch = 1; p.is_conv = 1; p.Cin = Cin; p.taps = ksize * ksize; p.kw_n = ksize;
    p.Ho = Ho; p.Wo = Wo; p.tile_w = tile_w; p.tile_h = tile_h; p.tile_n = tile_n; p.stride = stride; p.pad_t = pad_t; p.pad_l = pad_l;
    p.out = y; p.ldc = (int)ldc; p.out_batch_stride = 0;
    fill_epilogue(p, ep, Cout);
    return dispatch(tmA, tmB, p, tc, bf16, (cudaStream_t)stream);
}

static int wgrad_storage_check(int bf16, const char* name) {
    if (bf16 == 2) {
        dm_set_error("%s: weight gradients in fp32 storage (high-precision mode) are not implemented", name);
        return DM_EUNSUPPORTED;
    }
    DM_REQUIRE(bf16 == 0 || bf16 == 1, "storage selector: 0 fp16, 1 bf16");
    return DM_OK;
}

extern "C" int dm_conv2d_wgrad(int bf16, const void* x, int n_img, int H, int W, int Cin, const void* dy, int64_t ld_dy,
                               int Cout, int ksize, int stride, int pad_t, int pad_l, int Ho, int Wo, float* dw, float* db,
                               void* stream) {
    if (int rc = wgrad_storage_check(bf16, "dm_conv2d_wgrad")) return rc;
    DM_REQUIRE(x && dy && dw, "null pointer");
    DM_REQUIRE((((uintptr_t)x | (uintptr_t)dy | (uintptr_t)dw) & 15) == 0 && ((uintptr_t)db & 3) == 0,
               "x, dy and dw 16-byte aligned, db 4-byte aligned");
    DM_REQUIRE(n_img > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && Cout > 0, "positive extents");
    DM_REQUIRE(Cin > 0 && Cin % BK == 0, "Cin must be a multiple of 64 (pad the channels)");
    DM_REQUIRE(ksize == 3 || ksize == 1, "3x3 or 1x1");
    DM_REQUIRE(stride == 1 || stride == 2, "stride 1 or 2");
    DM_REQUIRE(pad_t >= 0 && pad_l >= 0, "non-negative padding");
    DM_REQUIRE(ld_dy % 8 == 0 && ld_dy >= Cout, "dy pixel stride: a multiple of 8 elements (16 bytes), at least Cout");
    // the forward's tiling rule at 64 pixels: a K-block is one box {tile_w, tile_h, tile_n} of output pixels; images past
    // n_img are zero-filled, so the pixel count need not be a multiple of 64
    const int tile_w = Wo < WG_PIX ? Wo : WG_PIX;
    const int tile_h = (WG_PIX / tile_w) < Ho ? (WG_PIX / tile_w) : Ho;
    const int tile_n = WG_PIX / (tile_w * tile_h);
    DM_REQUIRE(tile_w * tile_h * tile_n == WG_PIX && Wo % tile_w == 0 && Ho % tile_h == 0,
               "output extent must tile into 64-pixel boxes (power-of-two sizes)");
    const int64_t nk = (int64_t)(Wo / tile_w) * (Ho / tile_h) * dm_ceil_div(n_img, tile_n);
    DM_REQUIRE(nk * WG_PIX < (1ll << 31), "at most 2^31 output pixels");
    const int taps = ksize * ksize;
    CUtensorMap tmA, tmB;
    {
        // dY [n, Ho, Wo, ld_dy], first Cout channels: boxes {64 channels, tile_w, tile_h, tile_n}
        uint64_t dims[4] = {(uint64_t)Cout, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)n_img};
        uint64_t str[3] = {(uint64_t)ld_dy * 2, (uint64_t)Wo * ld_dy * 2, (uint64_t)Ho * Wo * ld_dy * 2};
        uint32_t box[4] = {64, (uint32_t)tile_w, (uint32_t)tile_h, (uint32_t)tile_n}, es[4] = {1, 1, 1, 1};
        int rc = encode_map(&tmA, bf16, dy, 4, dims, str, box, es); if (rc) return rc;
    }
    {
        // x through the forward's map: the same pixels at a tap's shifted origin, element strides for stride 2
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)n_img};
        uint64_t str[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
        uint32_t box[4] = {64, (uint32_t)(tile_w * stride), (uint32_t)(tile_h * stride), (uint32_t)tile_n};
        uint32_t es[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
        int rc = encode_map(&tmB, bf16, x, 4, dims, str, box, es); if (rc) return rc;
    }
    GemmParams p; memset(&p, 0, sizeof(p));
    p.M = Cout; p.N = taps * Cin; p.K = (int)(nk * WG_PIX);
    p.is_conv = 1; p.Cin = Cin; p.taps = taps; p.kw_n = ksize;
    p.Ho = Ho; p.Wo = Wo; p.tile_w = tile_w; p.tile_h = tile_h; p.tile_n = tile_n; p.stride = stride; p.pad_t = pad_t; p.pad_l = pad_l;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = wgrad_run(tmA, tmB, p, bf16, dw, st);
    if (rc || !db) return rc;
    return bias_grad(bf16, dy, ld_dy, (int64_t)n_img * Ho * Wo, Cout, db, st);
}

extern "C" int dm_gemm_wgrad(int bf16, const void* dy, int64_t ld_dy, const void* x, int64_t ldx, int M, int N, int K,
                             float* dw, float* db, void* stream) {
    if (int rc = wgrad_storage_check(bf16, "dm_gemm_wgrad")) return rc;
    DM_REQUIRE(dy && x && dw, "null pointer");
    DM_REQUIRE((((uintptr_t)x | (uintptr_t)dy | (uintptr_t)dw) & 15) == 0 && ((uintptr_t)db & 3) == 0,
               "x, dy and dw 16-byte aligned, db 4-byte aligned");
    DM_REQUIRE(M > 0 && M <= (1 << 30) && N > 0 && K > 0 && K % BK == 0, "1 <= M <= 2^30, N >= 1, K a positive multiple of 64");
    DM_REQUIRE(ld_dy % 8 == 0 && ldx % 8 == 0 && ld_dy >= N && ldx >= K,
               "row strides: multiples of 8 elements (16 bytes), at least N (dy) and K (x)");
    CUtensorMap tmA, tmB;
    {
        // dY [M, ld_dy] and x [M, ldx] token-major: boxes of 64 columns x 64 rows, rows past M zero-filled
        uint64_t dims[3] = {(uint64_t)N, (uint64_t)M, 1};
        uint64_t str[2] = {(uint64_t)ld_dy * 2, (uint64_t)M * ld_dy * 2};
        uint32_t box[3] = {64, WG_PIX, 1}, es[3] = {1, 1, 1};
        int rc = encode_map(&tmA, bf16, dy, 3, dims, str, box, es); if (rc) return rc;
    }
    {
        uint64_t dims[3] = {(uint64_t)K, (uint64_t)M, 1};
        uint64_t str[2] = {(uint64_t)ldx * 2, (uint64_t)M * ldx * 2};
        uint32_t box[3] = {64, WG_PIX, 1}, es[3] = {1, 1, 1};
        int rc = encode_map(&tmB, bf16, x, 3, dims, str, box, es); if (rc) return rc;
    }
    GemmParams p; memset(&p, 0, sizeof(p));
    p.M = N; p.N = K; p.K = (int)dm_ceil_div(M, WG_PIX) * WG_PIX;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = wgrad_run(tmA, tmB, p, bf16, dw, st);
    if (rc || !db) return rc;
    return bias_grad(bf16, dy, ld_dy, M, N, db, st);
}

// ---- input gradients.  Both plan like the forward contraction they equal (dm_gemm_plan(M, N = Cin / K_in, K = taps*Cout /
// N_out, act, bn_hint) reports the tile and split), and honour the whole dm_epilogue.
static int dgrad_storage_check(int bf16, const char* name) {
    if (bf16 == 2) {
        dm_set_error("%s: input gradients in fp32 storage (high-precision mode) are not implemented", name);
        return DM_EUNSUPPORTED;
    }
    DM_REQUIRE(bf16 == 0 || bf16 == 1, "storage selector: 0 fp16, 1 bf16");
    return DM_OK;
}
// B operand of the DGRAD mode: the forward weight [rows, ld] (first `cols` columns) as boxes of 64 columns x 64 rows
static int dgrad_weight_map(CUtensorMap* m, int bf16, const void* w, int64_t cols, int64_t rows, int64_t ld) {
    uint64_t dims[3] = {(uint64_t)cols, (uint64_t)rows, 1};
    uint64_t str[2] = {(uint64_t)ld * 2, (uint64_t)rows * ld * 2};
    uint32_t box[3] = {64, BK, 1}, es[3] = {1, 1, 1};
    return encode_map(m, bf16, w, 3, dims, str, box, es);
}
static int dgrad_epilogue_check(const dm_epilogue* ep, const void* dx, int64_t ldc, int N) {
    const int per16 = (ep && ep->out_f32) ? 4 : 8;      // elements per 16 bytes of dx
    DM_REQUIRE(((uintptr_t)dx & 15) == 0 && ldc >= N && ldc % per16 == 0,
               "dx 16-byte aligned, row stride at least the gradient's width and a multiple of 16 bytes");
    DM_REQUIRE(!ep || ep->act != 3, "the GEGLU epilogue has no meaning for an input gradient");
    DM_REQUIRE(!ep || !ep->residual || ep->ld_res == 0 || ep->ld_res >= N, "residual row stride at least the gradient's width");
    return DM_OK;
}

extern "C" int dm_conv2d_dgrad(int bf16, const void* dy, int n_img, int H, int W, int Cout, const void* w, int Cin, int ksize,
                               int pad_t, int pad_l, void* dx, int64_t ldc, const dm_epilogue* ep, int bn_hint, void* stream) {
    if (int rc = dgrad_storage_check(bf16, "dm_conv2d_dgrad")) return rc;
    DM_REQUIRE(dy && w && dx, "null pointer");
    DM_REQUIRE((((uintptr_t)dy | (uintptr_t)w) & 15) == 0, "dy and w 16-byte aligned");
    DM_REQUIRE(n_img > 0 && H > 0 && W > 0, "positive extents");
    DM_REQUIRE(Cout > 0 && Cout % BK == 0, "Cout must be a multiple of 64 (it is the reduction axis)");
    DM_REQUIRE(Cin > 0 && Cin % 8 == 0, "Cin must be a multiple of 8");
    DM_REQUIRE(ksize == 3 || ksize == 1, "3x3 or 1x1");
    DM_REQUIRE(pad_t >= 0 && pad_t < ksize && pad_l >= 0 && pad_l < ksize, "padding of the forward convolution: 0 .. ksize-1");
    if (int rc = dgrad_epilogue_check(ep, dx, ldc, Cin)) return rc;
    int tile_w = W < BM ? W : BM;
    int tile_h = (BM / tile_w) < H ? (BM / tile_w) : H;
    int tile_n = BM / (tile_w * tile_h);
    DM_REQUIRE(tile_w * tile_h * tile_n == BM && W % tile_w == 0 && H % tile_h == 0,
               "extent must tile into 128-pixel boxes (power-of-two sizes)");
    const int taps = ksize * ksize;
    TileChoice tc = choose_tile((int64_t)n_img * H * W, Cin, bn_hint);
    CUtensorMap tmA, tmB;
    {
        uint64_t dims[4] = {(uint64_t)Cout, (uint64_t)W, (uint64_t)H, (uint64_t)n_img};
        uint64_t str[3] = {(uint64_t)Cout * 2, (uint64_t)W * Cout * 2, (uint64_t)H * W * Cout * 2};
        uint32_t box[4] = {BK, (uint32_t)tile_w, (uint32_t)tile_h, (uint32_t)tile_n}, es[4] = {1, 1, 1, 1};
        int rc = encode_map(&tmA, bf16, dy, 4, dims, str, box, es); if (rc) return rc;
    }
    if (int rc = dgrad_weight_map(&tmB, bf16, w, (int64_t)taps * Cin, Cout, (int64_t)taps * Cin)) return rc;
    GemmParams p; memset(&p, 0, sizeof(p));
    p.M = n_img * H * W; p.N = Cin; p.K = taps * Cout; p.batch = 1; p.is_conv = 1; p.Cin = Cout; p.taps = taps; p.kw_n = ksize;
    p.Ho = H; p.Wo = W; p.tile_w = tile_w; p.tile_h = tile_h; p.tile_n = tile_n; p.stride = 1;
    p.pad_t = ksize - 1 - pad_t; p.pad_l = ksize - 1 - pad_l;
    p.out = dx; p.ldc = (int)ldc; p.out_batch_stride = 0;
    fill_epilogue(p, ep, Cin);
    return dispatch(tmA, tmB, p, tc, bf16, (cudaStream_t)stream, MODE_DGRAD);
}

extern "C" int dm_gemm_dgrad(int bf16, const void* dy, int64_t ld_dy, const void* w, int64_t ldw, void* dx, int64_t ldc, int M,
                             int N_out, int K_in, const dm_epilogue* ep, int bn_hint, void* stream) {
    if (int rc = dgrad_storage_check(bf16, "dm_gemm_dgrad")) return rc;
    DM_REQUIRE(dy && w && dx, "null pointer");
    DM_REQUIRE((((uintptr_t)dy | (uintptr_t)w) & 15) == 0, "dy and w 16-byte aligned");
    DM_REQUIRE(M > 0 && N_out > 0 && N_out % BK == 0 && K_in > 0 && K_in % 8 == 0,
               "M >= 1, N_out a positive multiple of 64 (it is the reduction axis), K_in a multiple of 8");
    DM_REQUIRE(ld_dy % 8 == 0 && ldw % 8 == 0 && ld_dy >= N_out && ldw >= K_in,
               "row strides: multiples of 8 elements (16 bytes), at least N_out (dy) and K_in (w)");
    if (int rc = dgrad_epilogue_check(ep, dx, ldc, K_in)) return rc;
    TileChoice tc = choose_tile(M, K_in, bn_hint);
    CUtensorMap tmA, tmB;
    {
        uint64_t dims[3] = {(uint64_t)N_out, (uint64_t)M, 1};
        uint64_t str[2] = {(uint64_t)ld_dy * 2, (uint64_t)M * ld_dy * 2};
        uint32_t box[3] = {BK, BM, 1}, es[3] = {1, 1, 1};
        int rc = encode_map(&tmA, bf16, dy, 3, dims, str, box, es); if (rc) return rc;
    }
    if (int rc = dgrad_weight_map(&tmB, bf16, w, K_in, N_out, ldw)) return rc;
    GemmParams p; memset(&p, 0, sizeof(p));
    p.M = M; p.N = K_in; p.K = N_out; p.batch = 1; p.taps = 1;
    p.out = dx; p.ldc = (int)ldc; p.out_batch_stride = 0;
    fill_epilogue(p, ep, K_in);
    return dispatch(tmA, tmB, p, tc, bf16, (cudaStream_t)stream, MODE_DGRAD);
}


// conv_out of the UNet with the CSD combination fused into its epilogue (SURVEY.md section 8b `dm_unet_fwd_sds`, north_star
// "SDS noise-residual scale/weight fused into the final UNet epilogue").  x [3B, H, W, Cin] ordered [branch][view], 3x3, pad 1,
// 4 output channels; replaces conv_out + `.sample` layout change + compute_grad_sds' tail (dreammat_guidance.py:274-282,475-495).
extern "C" int dm_conv2d_csd(int bf16, const void* x, int B, int H, int W, int Cin, const void* w, const void* bias,
                             const dm_csd* c, void* stream) {
    DM_REQUIRE(x && w && c && c->noise && c->w && c->coef && c->norms, "null pointer");
    DM_REQUIRE(bf16 == 0 || bf16 == 1, "16-bit storage only (fp32 mode uses conv_out + dm_sds_grad)");
    DM_REQUIRE(Cin % BK == 0 && B > 0, "Cin must be a multiple of 64");
    const int hw = H * W, n_img = 3 * B;
    DM_REQUIRE(((int64_t)B * hw) % BM == 0, "views x latent pixels must be a multiple of 128");
    int tile_w = W < BM ? W : BM;
    int tile_h = (BM / tile_w) < H ? (BM / tile_w) : H;
    int tile_n = BM / (tile_w * tile_h);
    DM_REQUIRE(tile_w * tile_h * tile_n == BM && W % tile_w == 0 && H % tile_h == 0 && (tile_n == 1 || B % tile_n == 0),
               "output extent must tile into 128-pixel boxes inside one branch");
    const int Cout = 4, K = 9 * Cin;
    CUtensorMap tmA, tmB;
    {
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)n_img};
        uint64_t str[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
        uint32_t box[4] = {BK, (uint32_t)tile_w, (uint32_t)tile_h, (uint32_t)tile_n}, es[4] = {1, 1, 1, 1};
        int rc = encode_map(&tmA, bf16, x, 4, dims, str, box, es); if (rc) return rc;
    }
    {
        uint64_t dims[3] = {(uint64_t)K, (uint64_t)Cout, 1};
        uint64_t str[2] = {(uint64_t)K * 2, (uint64_t)K * Cout * 2};
        uint32_t box[3] = {BK, 64, 1}, es[3] = {1, 1, 1};
        int rc = encode_map(&tmB, bf16, w, 3, dims, str, box, es); if (rc) return rc;
    }
    GemmParams p; memset(&p, 0, sizeof(p));
    p.M = n_img * hw; p.N = Cout; p.K = K; p.batch = 1; p.is_conv = 1; p.Cin = Cin; p.taps = 9; p.kw_n = 3;
    p.Ho = H; p.Wo = W; p.tile_w = tile_w; p.tile_h = tile_h; p.tile_n = tile_n; p.stride = 1; p.pad_t = 1; p.pad_l = 1;
    p.bias = bias; p.alpha = 1.0f; p.out_scale = 1.0f; p.rows_per_vec = 1; p.split_k = 1;
    p.csd = 1; p.csd_B = B; p.csd_hw = hw; p.csd_groups = (int)(((int64_t)B * hw) / BM);
    p.csd_noise = c->noise; p.csd_w = c->w; p.csd_coef = c->coef;
    p.csd_grad = c->grad; p.csd_dlat = c->dlatents; p.csd_norms = c->norms; p.csd_eps = c->eps_out;
    // persistent 64-wide kernel, one CTA per tile GROUP (three row tiles)
    cudaStream_t st = (cudaStream_t)stream;
    CUtensorMap none;      // the CSD epilogue writes fp32 per thread: no output / residual maps
    memset(&none, 0, sizeof(none));
    return bf16 ? launch<64, __nv_bfloat16>(tmA, tmB, none, none, p, p.csd_groups, st)
                : launch<64, __half>(tmA, tmB, none, none, p, p.csd_groups, st);
}
