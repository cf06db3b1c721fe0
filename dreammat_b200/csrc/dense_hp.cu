// dense_hp.cu -- the fp32-storage ("high precision") mode of the dense path.
//
// The reference can run its diffusion networks with fp32 weights (half_precision_weights=false,
// models/guidance/dreammat_guidance.py:56,92-94; BASELINE config 1 is that mode).  the tensor cores have no fp32 MMA,
// so the contractions keep running on the bf16 tensor-core kernel of tc_gemm.cu with BOTH operands split into
// three bf16 terms (x = x1 + x2 + x3, 24 mantissa bits) and the six significant partial products laid side by
// side along K:
//
//     A' = [a1 | a2 | a1 | a3 | a2 | a1]      B' = [b1 | b1 | b2 | b1 | b2 | b3]       (K' = 6 K)
//     A' . B'^T = a1b1 + a2b1 + a1b2 + a3b1 + a2b2 + a1b3 = A . B^T  up to 2^-24 relative terms
//
// accumulated in fp32 in TMEM by the unchanged kernel (for a 3x3 convolution the six segments are channel
// slabs of an NHWC tensor with 6 Cin channels, so the implicit-GEMM tap walk is untouched).  This file holds the
// pieces around that: the splitter, the fp32 epilogue (bias / per-image vector / activation / residual / scale /
// GEGLU applied to the raw fp32 accumulators), and plain fp32 versions of the streaming kernels
// (GroupNorm fwd/bwd, LayerNorm, GEGLU, axpby, transpose, pad) and of the fused attention (SIMT, online softmax).
// Throughput is not the point of this mode; fp32-class agreement with the reference is.
#include <cuda_bf16.h>
#include "common.cuh"
#include "dense_hp.cuh"

namespace {

inline int hp_grid(int64_t work, int threads = 256) {
    int64_t b = dm_ceil_div(work, threads);
    int64_t cap = (int64_t)DM_NUM_SMS * 16;
    return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

__global__ void __launch_bounds__(256) hp_split_kernel(const float* __restrict__ x, int64_t rows, int cols, int64_t ldx,
                                                       int pattern, __nv_bfloat16* __restrict__ out) {
    const int64_t n = rows * cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / cols; const int c = (int)(i - r * cols);
        const float v = x[r * ldx + c];
        const __nv_bfloat16 b1 = __float2bfloat16_rn(v);
        const float r1 = v - __bfloat162float(b1);
        const __nv_bfloat16 b2 = __float2bfloat16_rn(r1);
        const float r2 = r1 - __bfloat162float(b2);
        const __nv_bfloat16 b3 = __float2bfloat16_rn(r2);
        __nv_bfloat16* o = out + r * 6 * (int64_t)cols + c;
        if (pattern == 0) {   // A operand: a1 a2 a1 a3 a2 a1
            o[0] = b1; o[cols] = b2; o[2 * cols] = b1; o[3 * cols] = b3; o[4 * cols] = b2; o[5 * cols] = b1;
        } else {              // B operand: b1 b1 b2 b1 b2 b3
            o[0] = b1; o[cols] = b1; o[2 * cols] = b2; o[3 * cols] = b1; o[4 * cols] = b2; o[5 * cols] = b3;
        }
    }
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float silu_acc(float x) { return x / (1.0f + expf(-x)); }
__device__ __forceinline__ float silu_grad_acc(float x) {
    const float s = 1.0f / (1.0f + expf(-x));
    return s * (1.0f + x * (1.0f - s));
}

struct HpEpi {
    const float* raw; int64_t rows; int N; int64_t rows_per_batch;
    const float* bias; const float* rowvec; int rows_per_vec; int64_t ld_rowvec;
    const float* residual; int64_t ld_res; int64_t res_bs;
    float alpha, out_scale; int act;
    float* out; int64_t ldc; int64_t out_bs;
};

__global__ void __launch_bounds__(256) hp_epilogue_kernel(const HpEpi p) {
    const int No = p.act == 3 ? p.N / 2 : p.N;
    const int64_t n = p.rows * No;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = i / No; const int c = (int)(i - m * No);
        const int64_t z = m / p.rows_per_batch, mm = m - z * p.rows_per_batch;
        float v;
        if (p.act == 3) {
            // interleaved [32 value | 32 gate] column blocks (dense_ops.geglu_interleave)
            const int cv = (c >> 5) * 64 + (c & 31), cg = cv + 32;
            float a = p.raw[m * p.N + cv] * p.alpha, g = p.raw[m * p.N + cg] * p.alpha;
            if (p.bias) { a += p.bias[cv]; g += p.bias[cg]; }
            v = a * gelu_erf(g);
        } else {
            v = p.raw[m * p.N + c] * p.alpha;
            if (p.bias) v += p.bias[c];
            if (p.rowvec) v += p.rowvec[(mm / p.rows_per_vec) * p.ld_rowvec + c];
            if (p.act == 1) v = silu_acc(v);
            else if (p.act == 2) v = gelu_erf(v);
            if (p.residual) v += p.residual[z * p.res_bs + mm * p.ld_res + c];
        }
        p.out[z * p.out_bs + mm * p.ldc + c] = v * p.out_scale;
    }
}

// block reduction of two doubles (sum over the block); result valid in every thread
__device__ __forceinline__ void block_sum2(double& a, double& b) {
    __shared__ double sa[32], sb[32];
    __syncthreads();
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    if (l == 0) { sa[w] = a; sb[w] = b; }
    __syncthreads();
    a = 0.0; b = 0.0;
    for (int k = 0; k < nw; ++k) { a += sa[k]; b += sb[k]; }
}

// one block per (group, image): mean / centred variance in two passes, then the apply pass
__global__ void __launch_bounds__(256) hp_groupnorm_kernel(const float* __restrict__ x, int HW, int C, int ld, int G,
                                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                                           float eps, int silu, float* __restrict__ y, int ldy,
                                                           float* __restrict__ stats) {
    const int g = blockIdx.x, img = blockIdx.y, cpg = C / G;
    const float* xb = x + (int64_t)img * HW * ld + g * cpg;
    float* yb = y + (int64_t)img * HW * ldy + g * cpg;
    const int64_t cnt = (int64_t)HW * cpg;
    double s = 0.0, dummy = 0.0;
    for (int64_t i = threadIdx.x; i < cnt; i += blockDim.x) s += xb[(i / cpg) * ld + (i % cpg)];
    block_sum2(s, dummy);
    const float mean = (float)(s / (double)cnt);
    double ss = 0.0; dummy = 0.0;
    for (int64_t i = threadIdx.x; i < cnt; i += blockDim.x) { const float d = xb[(i / cpg) * ld + (i % cpg)] - mean; ss += (double)d * d; }
    block_sum2(ss, dummy);
    const float rstd = (float)(1.0 / sqrt(ss / (double)cnt + (double)eps));
    if (threadIdx.x == 0) { stats[((int64_t)img * G + g) * 2] = mean; stats[((int64_t)img * G + g) * 2 + 1] = rstd; }
    for (int64_t i = threadIdx.x; i < cnt; i += blockDim.x) {
        const int64_t p = i / cpg; const int c = (int)(i % cpg);
        float v = (xb[p * ld + c] - mean) * rstd * gamma[g * cpg + c] + beta[g * cpg + c];
        if (silu) v = silu_acc(v);
        yb[p * ldy + c] = v;
    }
}

// dx = rstd * (gamma*d' - mean_grp(gamma*d') - xhat * mean_grp(gamma*d'*xhat)) (+ dx_add),  d' = dz * act'(GN(x))
__global__ void __launch_bounds__(256) hp_groupnorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dz, int HW,
                                                               int C, int G, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, int silu,
                                                               const float* __restrict__ stats, const float* __restrict__ dx_add,
                                                               float* __restrict__ dx) {
    const int g = blockIdx.x, img = blockIdx.y, cpg = C / G;
    const int64_t base = (int64_t)img * HW * C + g * cpg;
    const int64_t cnt = (int64_t)HW * cpg;
    const float mean = stats[((int64_t)img * G + g) * 2], rstd = stats[((int64_t)img * G + g) * 2 + 1];
    double s1 = 0.0, s2 = 0.0;
    for (int64_t i = threadIdx.x; i < cnt; i += blockDim.x) {
        const int64_t o = base + (i / cpg) * C + (i % cpg); const int c = g * cpg + (int)(i % cpg);
        const float xh = (x[o] - mean) * rstd;
        float d = dz[o];
        if (silu) d *= silu_grad_acc(xh * gamma[c] + beta[c]);
        d *= gamma[c];
        s1 += d; s2 += (double)d * xh;
    }
    block_sum2(s1, s2);
    const float m1 = (float)(s1 / (double)cnt), m2 = (float)(s2 / (double)cnt);
    for (int64_t i = threadIdx.x; i < cnt; i += blockDim.x) {
        const int64_t o = base + (i / cpg) * C + (i % cpg); const int c = g * cpg + (int)(i % cpg);
        const float xh = (x[o] - mean) * rstd;
        float d = dz[o];
        if (silu) d *= silu_grad_acc(xh * gamma[c] + beta[c]);
        d *= gamma[c];
        float v = rstd * (d - m1 - xh * m2);
        if (dx_add) v += dx_add[o];
        dx[o] = v;
    }
}

__global__ void __launch_bounds__(128) hp_layernorm_kernel(const float* __restrict__ x, int C, const float* __restrict__ gamma,
                                                           const float* __restrict__ beta, float eps, float* __restrict__ y) {
    const float* xr = x + (int64_t)blockIdx.x * C; float* yr = y + (int64_t)blockIdx.x * C;
    double s = 0.0, dummy = 0.0;
    for (int c = threadIdx.x; c < C; c += blockDim.x) s += xr[c];
    block_sum2(s, dummy);
    const float mean = (float)(s / C);
    double ss = 0.0; dummy = 0.0;
    for (int c = threadIdx.x; c < C; c += blockDim.x) { const float d = xr[c] - mean; ss += (double)d * d; }
    block_sum2(ss, dummy);
    const float rstd = (float)(1.0 / sqrt(ss / C + (double)eps));
    for (int c = threadIdx.x; c < C; c += blockDim.x) yr[c] = (xr[c] - mean) * rstd * gamma[c] + beta[c];
}

__global__ void __launch_bounds__(256) hp_geglu_kernel(const float* __restrict__ h, int64_t M, int D, float* __restrict__ out) {
    const int64_t n = M * D;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t m = i / D; const int j = (int)(i - m * D);
        out[i] = h[m * 2 * D + j] * gelu_erf(h[m * 2 * D + D + j]);
    }
}

__global__ void __launch_bounds__(256) hp_axpby2d_kernel(const float* __restrict__ s1, int64_t ld1, float a,
                                                         const float* __restrict__ s2, int64_t ld2, float b, int64_t rows,
                                                         int cols, float* __restrict__ dst, int64_t ldd) {
    const int64_t n = rows * cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / cols; const int c = (int)(i - r * cols);
        float v = a * s1[r * ld1 + c];
        if (s2) v += b * s2[r * ld2 + c];
        dst[r * ldd + c] = v;
    }
}

__global__ void __launch_bounds__(256) hp_transpose_kernel(const float* __restrict__ x, int R, int C, int64_t ldx, int64_t bsx,
                                                           float* __restrict__ y, int64_t ldy, int64_t bsy) {
    __shared__ float tile[32][33];
    const float* xb = x + (int64_t)blockIdx.z * bsx; float* yb = y + (int64_t)blockIdx.z * bsy;
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int j = ty; j < 32; j += 8) {
        const int r = r0 + j, c = c0 + tx;
        tile[j][tx] = (r < R && c < C) ? xb[(int64_t)r * ldx + c] : 0.f;
    }
    __syncthreads();
    for (int j = ty; j < 32; j += 8) {
        const int c = c0 + j, r = r0 + tx;
        if (c < C && r < R) yb[(int64_t)c * ldy + r] = tile[tx][j];
    }
}

__global__ void __launch_bounds__(256) hp_pad_convert_kernel(const float* __restrict__ x, int64_t rows, int cin, int cpad,
                                                             float scale, float shift, float* __restrict__ y) {
    const int64_t n = rows * cpad;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / cpad; const int c = (int)(i - r * cpad);
        y[i] = c < cin ? fmaf(x[r * cin + c], scale, shift) : 0.f;
    }
}

// Attention, head_dim 64, fp32 SIMT: a warp owns one query row; keys are visited in tiles of 32 (lane = key for
// the scores, lane = output dims {lane, lane+32} for P.V); the block's four warps share the staged K / V tile.
constexpr int HPA_WARPS = 4;
__global__ void __launch_bounds__(HPA_WARPS * 32) hp_attention_kernel(const float* __restrict__ q, int64_t ldq, int64_t q_bs,
                                                                      const float* __restrict__ k, const float* __restrict__ v,
                                                                      int64_t ldkv, int64_t kv_bs, float* __restrict__ out,
                                                                      int64_t ldo, int64_t out_bs, int Nq, int Nk, float scale) {
    __shared__ float sk[32][65], sv[32][64], sq[HPA_WARPS][64];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int head = blockIdx.y, b = blockIdx.z;
    const int qi = blockIdx.x * HPA_WARPS + warp;
    const bool qok = qi < Nq;
    const float* qp = q + (int64_t)b * q_bs + (int64_t)(qok ? qi : 0) * ldq + head * 64;
    sq[warp][lane] = qp[lane] * scale; sq[warp][lane + 32] = qp[lane + 32] * scale;
    float m = -INFINITY, l = 0.f, o0 = 0.f, o1 = 0.f;
    const float* kb = k + (int64_t)b * kv_bs + head * 64;
    const float* vb = v + (int64_t)b * kv_bs + head * 64;
    for (int k0 = 0; k0 < Nk; k0 += 32) {
        __syncthreads();
        for (int i = threadIdx.x; i < 32 * 64; i += blockDim.x) {
            const int r = i >> 6, c = i & 63;
            const bool ok = k0 + r < Nk;
            sk[r][c] = ok ? kb[(int64_t)(k0 + r) * ldkv + c] : 0.f;
            sv[r][c] = ok ? vb[(int64_t)(k0 + r) * ldkv + c] : 0.f;
        }
        __syncthreads();
        float s = 0.f;
#pragma unroll 16
        for (int d = 0; d < 64; ++d) s = fmaf(sq[warp][d], sk[lane][d], s);
        if (k0 + lane >= Nk) s = -INFINITY;
        float tm = s;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) tm = fmaxf(tm, __shfl_xor_sync(0xffffffffu, tm, o));
        const float mn = fmaxf(m, tm);
        const float corr = expf(m - mn);            // exp(-inf) = 0 on the first tile
        const float pexp = expf(s - mn);
        l = l * corr + warp_sum(pexp);
        o0 *= corr; o1 *= corr;
#pragma unroll 8
        for (int j = 0; j < 32; ++j) {
            const float pj = __shfl_sync(0xffffffffu, pexp, j);
            o0 = fmaf(pj, sv[j][lane], o0); o1 = fmaf(pj, sv[j][lane + 32], o1);
        }
        m = mn;
    }
    if (qok) {
        float* op = out + (int64_t)b * out_bs + (int64_t)qi * ldo + head * 64;
        const float inv = 1.0f / l;
        op[lane] = o0 * inv; op[lane + 32] = o1 * inv;
    }
}

}  // namespace

// ---- C-ABI additions of the high-precision mode -------------------------------------------------------------------

extern "C" int dm_hp_split(const float* x, int64_t rows, int cols, int64_t ldx, int pattern, void* out_bf16, void* stream) {
    DM_REQUIRE(x && out_bf16 && rows >= 0 && cols > 0 && ldx >= cols && (pattern == 0 || pattern == 1), "bad args");
    if (rows == 0) return DM_OK;
    hp_split_kernel<<<hp_grid(rows * cols), 256, 0, (cudaStream_t)stream>>>(x, rows, cols, ldx, pattern, (__nv_bfloat16*)out_bf16);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_hp_epilogue(const float* raw, int64_t rows, int N, int64_t rows_per_batch, const dm_epilogue* ep, float* out,
                              int64_t ldc, int64_t out_batch_stride, void* stream) {
    DM_REQUIRE(raw && out && ep && rows >= 0 && N > 0 && rows_per_batch > 0, "bad args");
    DM_REQUIRE(ep->act != 3 || (N % 64 == 0 && !ep->residual && !ep->rowvec), "GEGLU epilogue: N multiple of 64, no residual / rowvec");
    if (rows == 0) return DM_OK;
    HpEpi p;
    p.raw = raw; p.rows = rows; p.N = N; p.rows_per_batch = rows_per_batch;
    p.bias = (const float*)ep->bias; p.rowvec = (const float*)ep->rowvec;
    p.rows_per_vec = ep->rows_per_vec > 0 ? ep->rows_per_vec : 1; p.ld_rowvec = ep->ld_rowvec > 0 ? ep->ld_rowvec : N;
    p.residual = (const float*)ep->residual; p.ld_res = ep->ld_res > 0 ? ep->ld_res : N; p.res_bs = ep->res_batch_stride;
    p.alpha = ep->alpha; p.out_scale = ep->out_scale; p.act = ep->act;
    p.out = out; p.ldc = ldc; p.out_bs = out_batch_stride;
    hp_epilogue_kernel<<<hp_grid(rows * (int64_t)N), 256, 0, (cudaStream_t)stream>>>(p);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

// ---- fp32 variants behind the dtype selector of the existing entry points -------------------------------------------

int hp_groupnorm(const float* x, int n_img, int HW, int C, int ld, int G, const float* gamma, const float* beta, float eps,
                 int silu, float* y, int ldy, float* stats, void* stream) {
    DM_REQUIRE(C % G == 0 && ld >= C && ldy >= C, "channel layout");
    hp_groupnorm_kernel<<<dim3(G, n_img), 256, 0, (cudaStream_t)stream>>>(x, HW, C, ld, G, gamma, beta, eps, silu, y, ldy, stats);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

int hp_groupnorm_bwd(const float* x, const float* dz, int n_img, int HW, int C, int G, const float* gamma, const float* beta,
                     float eps, int silu, const float* stats, const float* dx_add, float* dx, void* stream) {
    (void)eps;   // stats already hold (mean, rstd) in this mode
    DM_REQUIRE(C % G == 0, "channel layout");
    hp_groupnorm_bwd_kernel<<<dim3(G, n_img), 256, 0, (cudaStream_t)stream>>>(x, dz, HW, C, G, gamma, beta, silu, stats, dx_add, dx);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

int hp_layernorm(const float* x, int64_t M, int C, const float* gamma, const float* beta, float eps, float* y, void* stream) {
    if (M == 0) return DM_OK;
    hp_layernorm_kernel<<<(unsigned)M, 128, 0, (cudaStream_t)stream>>>(x, C, gamma, beta, eps, y);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

int hp_geglu(const float* h, int64_t M, int D, float* out, void* stream) {
    hp_geglu_kernel<<<hp_grid(M * D), 256, 0, (cudaStream_t)stream>>>(h, M, D, out);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

int hp_axpby2d(const float* s1, int64_t ld1, float a, const float* s2, int64_t ld2, float b, int64_t rows, int cols,
               float* dst, int64_t ldd, void* stream) {
    if (rows == 0) return DM_OK;
    hp_axpby2d_kernel<<<hp_grid(rows * cols), 256, 0, (cudaStream_t)stream>>>(s1, ld1, a, s2, ld2, b, rows, cols, dst, ldd);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

int hp_transpose(const float* x, int batch, int R, int C, int64_t ldx, int64_t bsx, float* y, int64_t ldy, int64_t bsy,
                 void* stream) {
    dim3 grid((unsigned)dm_ceil_div(C, 32), (unsigned)dm_ceil_div(R, 32), (unsigned)batch);
    hp_transpose_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, R, C, ldx, bsx, y, ldy, bsy);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

int hp_pad_convert(const float* x, int64_t rows, int cin, int cpad, float scale, float shift, float* y, void* stream) {
    hp_pad_convert_kernel<<<hp_grid(rows * cpad), 256, 0, (cudaStream_t)stream>>>(x, rows, cin, cpad, scale, shift, y);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

int hp_attention(const float* q, int64_t ldq, int64_t q_bs, const float* k, const float* v, int64_t ldkv, int64_t kv_bs,
                 float* out, int64_t ldo, int64_t out_bs, int batch, int heads, int Nq, int Nk, float scale, void* stream) {
    dim3 grid((unsigned)dm_ceil_div(Nq, HPA_WARPS), (unsigned)heads, (unsigned)batch);
    hp_attention_kernel<<<grid, HPA_WARPS * 32, 0, (cudaStream_t)stream>>>(q, ldq, q_bs, k, v, ldkv, kv_bs, out, ldo, out_bs, Nq, Nk, scale);
    DM_CHECK_LAUNCH();
    return DM_OK;
}
