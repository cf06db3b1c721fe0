// misc.cu -- error plumbing, compaction / canvas scatter (a2, a6), Adam (a9), CSD combine (a8 tail).
#include <stdarg.h>
#include <map>
#include <mutex>
#include <vector>
#include "common.cuh"

int g_dm_pdl = 1;   // programmatic dependent launch for the dense-section kernels (dm_tune "pdl")

static thread_local char g_err[512] = "";

void dm_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

static long long g_launches = 0;
void dm_count_launch() { __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED); }
extern "C" long long dm_launch_count(void) { return __atomic_load_n(&g_launches, __ATOMIC_RELAXED); }

extern "C" const char* dm_last_error(void) { return g_err; }

void* dm_scratch(int slot, size_t bytes, cudaStream_t st) {
    struct Buf { void* p; size_t bytes; };
    static std::mutex mu;
    static std::map<std::pair<int, int>, Buf> bufs;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { dm_set_error("dm_scratch: no current device"); return nullptr; }
    std::lock_guard<std::mutex> lock(mu);
    Buf& b = bufs[{dev, slot}];
    if (b.p && b.bytes >= bytes) return b.p;
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone) {
        dm_set_error("library scratch (slot %d) must grow to %zu bytes while the stream is being captured: run the same call once "
                     "before capture", slot, bytes);
        return nullptr;
    }
    void* p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess || cudaMemsetAsync(p, 0, bytes, st) != cudaSuccess) {
        dm_set_error("library scratch: cudaMalloc / memset of %zu bytes failed", bytes);
        return nullptr;
    }
    b.p = p; b.bytes = bytes;      // the old buffer (if any) stays allocated: a captured graph may still use it
    return p;
}
extern "C" int dm_version(void) { return 100; }

extern "C" int dm_device_check(int dev) {
    cudaDeviceProp p;
    DM_CHECK_CUDA(cudaGetDeviceProperties(&p, dev));
    if (p.major != 9 || p.minor != 0) {
        dm_set_error("device %d is sm_%d%d; this library only carries sm_90a code", dev, p.major, p.minor);
        return DM_EUNSUPPORTED;
    }
    return DM_OK;
}

namespace {

constexpr int CB = 1024;

__global__ void __launch_bounds__(CB) count_kernel(const uint8_t* __restrict__ mask, int64_t n, int32_t* __restrict__ counts) {
    __shared__ int s;
    if (threadIdx.x == 0) s = 0;
    __syncthreads();
    int64_t i = (int64_t)blockIdx.x * CB + threadIdx.x;
    int v = (i < n && mask[i]) ? 1 : 0;
    unsigned b = __ballot_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0) atomicAdd(&s, __popc(b));
    __syncthreads();
    if (threadIdx.x == 0) counts[blockIdx.x] = s;
}

__global__ void __launch_bounds__(CB) compact_kernel(const uint8_t* __restrict__ mask, int64_t n,
                                                     const int32_t* __restrict__ offsets, int32_t* __restrict__ idx) {
    __shared__ int warp_cnt[CB / 32];
    int64_t i = (int64_t)blockIdx.x * CB + threadIdx.x;
    int v = (i < n && mask[i]) ? 1 : 0;
    unsigned b = __ballot_sync(0xffffffffu, v);
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) warp_cnt[w] = __popc(b);
    __syncthreads();
    int base = offsets[blockIdx.x];
    for (int k = 0; k < w; ++k) base += warp_cnt[k];
    if (v) idx[base + __popc(b & ((1u << lane) - 1u))] = (int32_t)i;
}

__global__ void gather_rows_kernel(const float* __restrict__ src, const int32_t* __restrict__ idx, int64_t n, int c,
                                   float* __restrict__ dst) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * c) return;
    int64_t r = i / c; int k = (int)(i % c);
    dst[i] = src[(int64_t)idx[r] * c + k];
}

__global__ void scatter_rows_kernel(const float* __restrict__ src, const int32_t* __restrict__ idx, int64_t n, int c,
                                    float* __restrict__ dst) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * c) return;
    int64_t r = i / c; int k = (int)(i % c);
    dst[(int64_t)idx[r] * c + k] = src[i];
}

__global__ void fill_kernel(float* __restrict__ p, int64_t n, float v) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// depth: scratch2[0] = min, scratch2[1] = max of 1/(z/w+1e-6) over the mask (as ordered-int atomics)
__device__ __forceinline__ int f2ord(float f) { int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7fffffff; }
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

__global__ void depth_minmax_kernel(const float* __restrict__ rast, const uint8_t* __restrict__ mask, int64_t n, int* mm) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float lo = 3e38f, hi = -3e38f;
    if (i < n && mask[i]) { float d = 1.0f / (rast[4 * i + 2] + 1e-6f); lo = d; hi = d; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
    if ((threadIdx.x & 31) == 0 && hi >= lo) { atomicMin(mm, f2ord(lo)); atomicMax(mm + 1, f2ord(hi)); }
}
__global__ void depth_init_kernel(int* mm) { mm[0] = f2ord(3e38f); mm[1] = f2ord(-3e38f); }
__global__ void depth_apply_kernel(const float* __restrict__ rast, const uint8_t* __restrict__ mask, int64_t n,
                                   const int* __restrict__ mm, float* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float v = rast[4 * i + 2];
    if (mask[i]) {
        float lo = ord2f(mm[0]), hi = ord2f(mm[1]);
        float d = 1.0f / (v + 1e-6f);
        v = (1.0f - 0.3f) * (d - lo) / (hi - lo + 1e-6f) + 0.3f;
    }
    out[i] = v;
}

// torch.optim.Adam (no amsgrad, no weight decay):
//   m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ; p -= lr/bc1 * m / (sqrt(v)/sqrt(bc2) + eps)
__global__ void __launch_bounds__(256) adam_kernel(float4* __restrict__ p, const float4* __restrict__ g,
                                                   float4* __restrict__ m, float4* __restrict__ v, int64_t n4,
                                                   float* __restrict__ pt, const float* __restrict__ gt,
                                                   float* __restrict__ mt, float* __restrict__ vt, int tail,
                                                   float b1, float b2, float eps, float step_size, float inv_sqrt_bc2,
                                                   float gscale) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    auto upd = [&](float& pp, float gg, float& mm, float& vv) {
        gg *= gscale;
        mm = b1 * mm + (1.0f - b1) * gg;
        vv = b2 * vv + (1.0f - b2) * gg * gg;
        float denom = sqrtf(vv) * inv_sqrt_bc2 + eps;
        pp -= step_size * (mm / denom);
    };
    if (i < n4) {
        float4 P = p[i], G = g[i], M = m[i], V = v[i];
        upd(P.x, G.x, M.x, V.x); upd(P.y, G.y, M.y, V.y); upd(P.z, G.z, M.z, V.z); upd(P.w, G.w, M.w, V.w);
        p[i] = P; m[i] = M; v[i] = V;
    }
    if (i < tail) upd(pt[i], gt[i], mt[i], vt[i]);
}

// silhouette antialias as a cached sparse blend (see dreammat_b200/antialias.py): out[dst] += a * (in[src] - in[dst]).
// Deterministic for any pair order, O(k): each pair drops its index into a small bucket of its key pixel (library scratch:
// count[n_pix] + AA_CAP slots per pixel); the pair with the lowest index owns the pixel and sums the bucket's pairs in index
// order (a fuller bucket falls back to a scan of the list); a last pass clears the touched counts.  No fp32 atomics.
constexpr int AA_CAP = 8;
__global__ void aa_bucket_kernel(const int32_t* __restrict__ key, int64_t k, int32_t* __restrict__ cnt, int32_t* __restrict__ slot) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= k) return;
    const int64_t x = key[e];
    const int i = atomicAdd(cnt + x, 1);
    if (i < AA_CAP) slot[x * AA_CAP + i] = (int32_t)e;
}
__global__ void aa_clear_kernel(const int32_t* __restrict__ key, int64_t k, int32_t* __restrict__ cnt) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < k) cnt[key[e]] = 0;
}
// pairs of pixel key[e] in index order if e owns the pixel (returns their number; -1: e owns it but the bucket overflowed,
// scan the list from e), 0 if another pair owns it
__device__ __forceinline__ int aa_owned(const int32_t* __restrict__ key, int64_t e, const int32_t* __restrict__ cnt,
                                        const int32_t* __restrict__ slot, int32_t (&list)[AA_CAP]) {
    const int64_t x = key[e];
    const int c = cnt[x];
    if (c > AA_CAP) {
        for (int64_t j = 0; j < e; ++j) if (key[j] == x) return 0;
        return -1;
    }
    for (int i = 0; i < c; ++i) {
        const int32_t v = slot[x * AA_CAP + i];
        if (v < e) return 0;
        int p = i;                                  // insertion sort (c <= 8)
        while (p > 0 && list[p - 1] > v) { list[p] = list[p - 1]; --p; }
        list[p] = v;
    }
    return c;
}
__global__ void aa_fwd_kernel(const float* __restrict__ in, const int32_t* __restrict__ dst, const int32_t* __restrict__ src,
                              const float* __restrict__ alpha, int64_t k, int c, const int32_t* __restrict__ cnt,
                              const int32_t* __restrict__ slot, float* __restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= k) return;
    int32_t list[AA_CAP];
    const int m = aa_owned(dst, e, cnt, slot, list);
    if (m == 0) return;
    const int64_t d = dst[e];
    for (int ch = 0; ch < c; ++ch) {
        const float base = in[d * c + ch];
        float acc = 0.f;
        if (m > 0) {
            for (int i = 0; i < m; ++i) acc += alpha[list[i]] * (in[(int64_t)src[list[i]] * c + ch] - base);
        } else {
            for (int64_t j = e; j < k; ++j) if (dst[j] == d) acc += alpha[j] * (in[(int64_t)src[j] * c + ch] - base);
        }
        out[d * c + ch] = base + acc;
    }
}
// adjoint, pass 1 (destination side): din[dst] -= sum a * dout[dst]
__global__ void aa_bwd_dst_kernel(const float* __restrict__ dout, const int32_t* __restrict__ dst, const float* __restrict__ alpha,
                                  int64_t k, int c, const int32_t* __restrict__ cnt, const int32_t* __restrict__ slot,
                                  float* __restrict__ din) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= k) return;
    int32_t list[AA_CAP];
    const int m = aa_owned(dst, e, cnt, slot, list);
    if (m == 0) return;
    const int64_t d = dst[e];
    float a = 0.f;
    if (m > 0) { for (int i = 0; i < m; ++i) a += alpha[list[i]]; }
    else { for (int64_t j = e; j < k; ++j) if (dst[j] == d) a += alpha[j]; }
    for (int ch = 0; ch < c; ++ch) din[d * c + ch] -= a * dout[d * c + ch];
}
// adjoint, pass 2 (source side, after pass 1): din[src] += sum a * dout[dst]
__global__ void aa_bwd_src_kernel(const float* __restrict__ dout, const int32_t* __restrict__ dst, const int32_t* __restrict__ src,
                                  const float* __restrict__ alpha, int64_t k, int c, const int32_t* __restrict__ cnt,
                                  const int32_t* __restrict__ slot, float* __restrict__ din) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= k) return;
    int32_t list[AA_CAP];
    const int m = aa_owned(src, e, cnt, slot, list);
    if (m == 0) return;
    const int64_t s_ = src[e];
    for (int ch = 0; ch < c; ++ch) {
        float acc = 0.f;
        if (m > 0) {
            for (int i = 0; i < m; ++i) acc += alpha[list[i]] * dout[(int64_t)dst[list[i]] * c + ch];
        } else {
            for (int64_t j = e; j < k; ++j) if (src[j] == s_) acc += alpha[j] * dout[(int64_t)dst[j] * c + ch];
        }
        din[s_ * c + ch] += acc;
    }
}

// bucket scratch of one antialias call: count[n_pix] then AA_CAP slots per pixel (counts are zero between calls)
static int aa_scratch(int64_t n_pix, cudaStream_t st, int32_t** cnt, int32_t** slot) {
    void* p = dm_scratch(DM_SCRATCH_AA, (size_t)n_pix * (1 + AA_CAP) * sizeof(int32_t), st);
    if (!p) return DM_EDRIVER;
    *cnt = (int32_t*)p; *slot = *cnt + n_pix;
    return DM_OK;
}

// F.interpolate(mode="bilinear", align_corners=False) on NHWC fp32 (dreammat_guidance.py:507-513) and its adjoint
__device__ __forceinline__ void bil_src(int dst, float scale, int in_size, int& i0, int& i1, float& l) {
    float src = ((float)dst + 0.5f) * scale - 0.5f;
    src = src < 0.f ? 0.f : src;
    i0 = (int)src; if (i0 > in_size - 1) i0 = in_size - 1;
    i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
    l = src - (float)i0;
}
__global__ void resize_bilinear_kernel(const float* __restrict__ in, int n, int Hi, int Wi, int Ho, int Wo, int c,
                                       float* __restrict__ out, int adjoint) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t tot = (int64_t)n * Ho * Wo * c;
    if (i >= tot) return;
    int ch = (int)(i % c); int64_t r = i / c; int xo = (int)(r % Wo); r /= Wo; int yo = (int)(r % Ho); int b = (int)(r / Ho);
    int y0, y1, x0, x1; float ly, lx;
    bil_src(yo, (float)Hi / (float)Ho, Hi, y0, y1, ly);
    bil_src(xo, (float)Wi / (float)Wo, Wi, x0, x1, lx);
    const int64_t base = (int64_t)b * Hi * Wi;
    const int64_t a00 = ((base + (int64_t)y0 * Wi + x0) * c + ch), a01 = ((base + (int64_t)y0 * Wi + x1) * c + ch);
    const int64_t a10 = ((base + (int64_t)y1 * Wi + x0) * c + ch), a11 = ((base + (int64_t)y1 * Wi + x1) * c + ch);
    const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
    if (!adjoint) {
        out[i] = w00 * in[a00] + w01 * in[a01] + w10 * in[a10] + w11 * in[a11];
    } else {   // `in` is d(out) [n,Ho,Wo,c]; `out` is d(in) [n,Hi,Wi,c], pre-zeroed
        float g = in[i];
        atomicAdd(out + a00, w00 * g); atomicAdd(out + a01, w01 * g); atomicAdd(out + a10, w10 * g); atomicAdd(out + a11, w11 * g);
    }
}

// CSD combine (dreammat_guidance.py:475-481, 584-594) with the 10 diagnostic sums.
__global__ void __launch_bounds__(256) sds_kernel(const float* __restrict__ e, const float* __restrict__ noise,
                                                  const float* __restrict__ w, int B, int64_t chw, float ct, float cu,
                                                  float cn, float cs, float* __restrict__ grad,
                                                  float* __restrict__ dlat, float* __restrict__ norms) {
    __shared__ float s[10];
    if (threadIdx.x < 10) s[threadIdx.x] = 0.f;
    __syncthreads();
    int64_t total = (int64_t)B * chw;
    float acc[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int b = (int)(i / chw);
        float et = e[i], eu = e[total + i], en = e[2 * total + i], nz = noise[i];
        float g = w[b] * (ct * et + cu * eu + cn * en + cs * nz);
        // torch.nan_to_num: nan -> 0, +-inf -> +-float max
        if (isnan(g)) g = 0.f; else if (isinf(g)) g = g > 0 ? 3.4028234663852886e38f : -3.4028234663852886e38f;
        if (grad) grad[i] = g;
        if (dlat) dlat[i] = g / (float)B;
        acc[0] += 0.5f * g * g;            // loss_sds * B
        acc[1] += g * g;                   // grad_norm^2
        acc[2] += (eu - nz) * (eu - nz);
        acc[3] += (et - nz) * (et - nz);
        acc[4] += (et - eu) * (et - eu);
        acc[5] += (et - en) * (et - en);
        acc[6] += (en - eu) * (en - eu);
        acc[7] += nz * nz;
        acc[8] += eu * eu;
        acc[9] += et * et;
    }
#pragma unroll
    for (int k = 0; k < 10; ++k) {
        float v = warp_sum(acc[k]);
        if ((threadIdx.x & 31) == 0) atomicAdd(&s[k], v);
    }
    __syncthreads();
    if (threadIdx.x < 10 && norms) atomicAdd(norms + threadIdx.x, s[threadIdx.x]);
}

}  // namespace

extern "C" int dm_compact_mask(const uint8_t* mask, int64_t n, int32_t* idx_out, int64_t* count_host, void* stream) {
    DM_REQUIRE(mask && idx_out && count_host, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    int nb = (int)dm_ceil_div(n, CB);
    if (nb == 0) { *count_host = 0; return DM_OK; }
    int32_t* d_counts = nullptr;
    DM_CHECK_CUDA(cudaMalloc(&d_counts, sizeof(int32_t) * nb));
    count_kernel<<<nb, CB, 0, st>>>(mask, n, d_counts);
    std::vector<int32_t> h(nb);
    cudaError_t e = cudaMemcpyAsync(h.data(), d_counts, sizeof(int32_t) * nb, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { cudaFree(d_counts); dm_set_error("dm_compact_mask: %s", cudaGetErrorString(e)); return (int)e; }
    int64_t run = 0;
    for (int i = 0; i < nb; ++i) { int32_t c = h[i]; h[i] = (int32_t)run; run += c; }
    *count_host = run;
    e = cudaMemcpyAsync(d_counts, h.data(), sizeof(int32_t) * nb, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) { compact_kernel<<<nb, CB, 0, st>>>(mask, n, d_counts, idx_out); e = cudaStreamSynchronize(st); }
    cudaFree(d_counts);
    if (e != cudaSuccess) { dm_set_error("dm_compact_mask: %s", cudaGetErrorString(e)); return (int)e; }
    return DM_OK;
}

extern "C" int dm_gather_rows(const float* src, const int32_t* idx, int64_t n, int c, float* dst, void* stream) {
    if (n == 0) return DM_OK;
    DM_REQUIRE(src && idx && dst && c > 0, "bad args");
    gather_rows_kernel<<<(unsigned)dm_ceil_div(n * c, 256), 256, 0, (cudaStream_t)stream>>>(src, idx, n, c, dst);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_gather_canvas_grad(const float* dcanvas, const int32_t* pix, int64_t n, int c, float* dvalues, void* stream) {
    return dm_gather_rows(dcanvas, pix, n, c, dvalues, stream);
}

extern "C" int dm_scatter_canvas(const float* values, const int32_t* pix, int64_t n, int c, float* canvas, void* stream) {
    if (n == 0) return DM_OK;
    DM_REQUIRE(values && pix && canvas && c > 0, "bad args");
    scatter_rows_kernel<<<(unsigned)dm_ceil_div(n * c, 256), 256, 0, (cudaStream_t)stream>>>(values, pix, n, c, canvas);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_fill(float* p, int64_t n, float v, void* stream) {
    if (n == 0) return DM_OK;
    DM_REQUIRE(p, "null pointer");
    fill_kernel<<<(unsigned)dm_ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(p, n, v);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_antialias_fwd(const float* in, const int32_t* dst, const int32_t* src, const float* alpha, int64_t k,
                                int64_t n_pix, int c, float* out, void* stream) {
    DM_REQUIRE(in && out && c > 0, "bad args");
    cudaStream_t st = (cudaStream_t)stream;
    if (in != out) DM_CHECK_CUDA(cudaMemcpyAsync(out, in, sizeof(float) * n_pix * c, cudaMemcpyDeviceToDevice, st));
    if (k == 0) return DM_OK;
    DM_REQUIRE(dst && src && alpha && in != out, "null pointer / in-place with pairs");
    int32_t *cnt, *slot; int rc = aa_scratch(n_pix, st, &cnt, &slot); if (rc) return rc;
    const unsigned blocks = (unsigned)dm_ceil_div(k, 128);
    aa_bucket_kernel<<<blocks, 128, 0, st>>>(dst, k, cnt, slot);
    DM_CHECK_LAUNCH();
    aa_fwd_kernel<<<blocks, 128, 0, st>>>(in, dst, src, alpha, k, c, cnt, slot, out);
    DM_CHECK_LAUNCH();
    aa_clear_kernel<<<blocks, 128, 0, st>>>(dst, k, cnt);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_antialias_bwd(const float* dout, const int32_t* dst, const int32_t* src, const float* alpha, int64_t k,
                                int64_t n_pix, int c, float* din, void* stream) {
    DM_REQUIRE(dout && din && c > 0 && dout != din, "bad args");
    cudaStream_t st = (cudaStream_t)stream;
    DM_CHECK_CUDA(cudaMemcpyAsync(din, dout, sizeof(float) * n_pix * c, cudaMemcpyDeviceToDevice, st));
    if (k == 0) return DM_OK;
    DM_REQUIRE(dst && src && alpha, "null pointer");
    int32_t *cnt, *slot; int rc = aa_scratch(n_pix, st, &cnt, &slot); if (rc) return rc;
    const unsigned blocks = (unsigned)dm_ceil_div(k, 128);
    aa_bucket_kernel<<<blocks, 128, 0, st>>>(dst, k, cnt, slot);
    DM_CHECK_LAUNCH();
    aa_bwd_dst_kernel<<<blocks, 128, 0, st>>>(dout, dst, alpha, k, c, cnt, slot, din);
    DM_CHECK_LAUNCH();
    aa_clear_kernel<<<blocks, 128, 0, st>>>(dst, k, cnt);
    DM_CHECK_LAUNCH();
    aa_bucket_kernel<<<blocks, 128, 0, st>>>(src, k, cnt, slot);
    DM_CHECK_LAUNCH();
    aa_bwd_src_kernel<<<blocks, 128, 0, st>>>(dout, dst, src, alpha, k, c, cnt, slot, din);
    DM_CHECK_LAUNCH();
    aa_clear_kernel<<<blocks, 128, 0, st>>>(src, k, cnt);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_resize_bilinear(const float* in, int n, int Hi, int Wi, int Ho, int Wo, int c, float* out, int adjoint,
                                  void* stream) {
    DM_REQUIRE(in && out && n > 0 && c > 0, "bad args");
    cudaStream_t st = (cudaStream_t)stream;
    if (adjoint) DM_CHECK_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)n * Hi * Wi * c, st));
    int64_t tot = (int64_t)n * Ho * Wo * c;
    resize_bilinear_kernel<<<(unsigned)dm_ceil_div(tot, 256), 256, 0, st>>>(in, n, Hi, Wi, Ho, Wo, c, out, adjoint);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_depth_normalize(const float* rast, const uint8_t* mask, int64_t n_pix, float* depth_out, float* scratch2,
                                  void* stream) {
    if (n_pix == 0) return DM_OK;
    DM_REQUIRE(rast && mask && depth_out && scratch2, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    depth_init_kernel<<<1, 1, 0, st>>>((int*)scratch2);
    depth_minmax_kernel<<<(unsigned)dm_ceil_div(n_pix, 256), 256, 0, st>>>(rast, mask, n_pix, (int*)scratch2);
    depth_apply_kernel<<<(unsigned)dm_ceil_div(n_pix, 256), 256, 0, st>>>(rast, mask, n_pix, (const int*)scratch2, depth_out);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_adam_step(float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2,
                            float eps, int32_t step, float grad_scale, void* stream) {
    if (n == 0) return DM_OK;
    DM_REQUIRE(p && g && m && v && step >= 1, "bad args");
    DM_REQUIRE((((uintptr_t)p | (uintptr_t)g | (uintptr_t)m | (uintptr_t)v) & 15) == 0, "16-byte alignment");
    double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
    float step_size = (float)((double)lr / bc1), inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
    int64_t n4 = n / 4; int tail = (int)(n - 4 * n4);
    int64_t work = n4 > tail ? n4 : tail;
    adam_kernel<<<(unsigned)dm_ceil_div(work, 256), 256, 0, (cudaStream_t)stream>>>(
        (float4*)p, (const float4*)g, (float4*)m, (float4*)v, n4, p + 4 * n4, g + 4 * n4, m + 4 * n4, v + 4 * n4, tail, beta1,
        beta2, eps, step_size, inv_sqrt_bc2, grad_scale);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_sds_grad(const float* eps_pred, const float* noise, const float* w, int B, int64_t chw, float c_text,
                           float c_uncond, float c_null, float c_noise, float* grad, float* dlatents, float* norms,
                           void* stream) {
    DM_REQUIRE(eps_pred && noise && w && B > 0 && chw > 0, "bad args");
    int64_t total = (int64_t)B * chw;
    int blocks = (int)(dm_ceil_div(total, 256) < DM_NUM_SMS * 4 ? dm_ceil_div(total, 256) : DM_NUM_SMS * 4);
    sds_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(eps_pred, noise, w, B, chw, c_text, c_uncond, c_null, c_noise, grad,
                                                         dlatents, norms);
    DM_CHECK_LAUNCH();
    return DM_OK;
}
