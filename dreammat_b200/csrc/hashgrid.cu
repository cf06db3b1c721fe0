// hashgrid.cu -- fused multiresolution hash-grid encoding + bias-free 32->64->5 MLP, forward and
// backward (row a3 of SURVEY.md section 8).
//
// Replaces tcnn.Encoding("HashGrid") + VanillaMLP as called from
//   models/geometry/dreammat_mesh.py:239-254  (contract -> encoding -> feature_network)
//   models/networks.py:55-64 (TCNNEncoding, fp32 out), :150-187 (VanillaMLP, no bias, ReLU)
// Parameter layout is tiny-cuda-nn's (level-major, entry-major, features interleaved) so a
// reference checkpoint's `geometry.encoding.encoding.encoding.params` loads unchanged.
//
// Memory behaviour: the 50.4 MB table is about the size of the H100's 50 MB L2; each point does
// 16 levels x 8 corner float2 gathers.  One thread owns (point, 4 levels) in the gather phase
// so 32 independent 8-byte loads are in flight per thread; the MLP runs out of shared memory.
// Backward recomputes the forward (nothing saved) and is deterministic: the grid gradient is scattered as int64 fixed
// point into a library-owned accumulator (integer adds are associative, so the order in which warps arrive does not change
// the sum) with a power-of-two scale fixed per call from a bound on every finite contribution; one pass then adds it to
// dgrid in fp32.  Non-finite contributions go straight to dgrid (inf / nan results do not depend on the order).  The weight gradients
// stay in shared memory until the block retires and are written as per-block rows that are added in block order.
#include "common.cuh"

namespace {

constexpr int MAXL = 16;
constexpr int TILE = 64;       // points per tile
constexpr int NTHREADS = 256;  // 4 level-groups x 64 points
constexpr int ENC = 32;
constexpr int HID = 64;
constexpr int NOUT = 5;

constexpr int DW_ROW = HID * ENC + NOUT * HID;   // one block's dW1 | dW2 partial row
constexpr int BWD_MAX_BLOCKS = DM_NUM_SMS * 2;
constexpr int64_t HDR_BYTES = 256;

// Fixed-point scale 2^e of a backward call: every contribution is at most U = hdr[0]*hdr[1]*hdr[2] in magnitude and an
// entry receives at most 8 per point and level, so |sum| * 2^e < 8 n U 2^e <= 2^62 fits int64.
__device__ __forceinline__ double fixed_scale(const uint32_t* hdr, int64_t n) {
    const double U = (double)__uint_as_float(hdr[0]) * (double)__uint_as_float(hdr[1]) * (double)__uint_as_float(hdr[2]);
    if (!(U > 0.0) || !isfinite(U)) return 1.0;
    int eu, en;
    frexp(U, &eu);                       // U < 2^eu
    frexp((double)(8 * (n > 0 ? n : 1)), &en);
    return ldexp(1.0, 62 - eu - en);
}
__device__ __forceinline__ void fixed_add(unsigned long long* acc, float* dgrid, int64_t i, float v, double S) {
    if (v == 0.f) return;
    const double q = (double)v * S;
    if (isfinite(v) && fabs(q) < 4.6116860184273879e18)        // 2^62: inside the bound (always, for finite weights)
        atomicAdd(acc + i, (unsigned long long)__double2ll_rn(q));
    else
        atomicAdd(dgrid + i, v);
}

struct LevelMeta {
    float scale[MAXL];
    uint32_t res[MAXL];
    uint32_t size[MAXL];
    uint32_t offset[MAXL];
    uint32_t hashed[MAXL];
    int n_levels;
    float bmin, inv_ext;
};

int make_meta(const dm_hashgrid_cfg* c, LevelMeta& m, int64_t* total) {
    if (!c || c->n_levels < 1 || c->n_levels > MAXL || c->n_features != 2) {
        dm_set_error("hashgrid cfg: n_levels in [1,16] and n_features == 2 required");
        return DM_EINVAL;
    }
    uint64_t off = 0;
    const float l2 = log2f(c->per_level_scale);
    for (int l = 0; l < c->n_levels; ++l) {
        // tcnn: scale = exp2f(level * log2f(per_level_scale)) * base_resolution - 1.0f
        float s = exp2f((float)l * l2) * (float)c->base_resolution - 1.0f;
        uint32_t res = (uint32_t)ceilf(s) + 1u;
        uint64_t n = (uint64_t)res * res * res;
        n = ((n + 7) / 8) * 8;
        uint64_t cap = 1ull << c->log2_hashmap;
        if (n > cap) n = cap;
        m.scale[l] = s; m.res[l] = res; m.size[l] = (uint32_t)n; m.offset[l] = (uint32_t)off;
        m.hashed[l] = ((uint64_t)res * res * res > n) ? 1u : 0u;
        off += n;
    }
    m.n_levels = c->n_levels;
    m.bmin = c->bbox_min;
    m.inv_ext = 1.0f / (c->bbox_max - c->bbox_min);
    if (total) *total = (int64_t)off;
    return DM_OK;
}

__device__ __forceinline__ uint32_t grid_index(uint32_t x, uint32_t y, uint32_t z, uint32_t res, uint32_t size,
                                               uint32_t hashed) {
    uint32_t idx;
    if (hashed) idx = (x * 1u) ^ (y * 2654435761u) ^ (z * 805459861u);
    else idx = x + y * res + z * res * res;
    return idx % size;
}

// Encode 4 levels [l0, l0+4) of one point into enc[0..8)
struct Corner { uint32_t idx[8]; float w[8]; };

__device__ __forceinline__ void level_corners(const LevelMeta& m, int l, float x, float y, float z, Corner& c) {
    float s = m.scale[l];
    float px = fmaf(s, x, 0.5f), py = fmaf(s, y, 0.5f), pz = fmaf(s, z, 0.5f);
    float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
    uint32_t ix = (uint32_t)(int)fx, iy = (uint32_t)(int)fy, iz = (uint32_t)(int)fz;
    float wx = px - fx, wy = py - fy, wz = pz - fz;
    uint32_t res = m.res[l], size = m.size[l], hs = m.hashed[l], off = m.offset[l];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        uint32_t ox = k & 1, oy = (k >> 1) & 1, oz = (k >> 2) & 1;
        c.idx[k] = off + grid_index(ix + ox, iy + oy, iz + oz, res, size, hs);
        c.w[k] = (ox ? wx : 1.0f - wx) * (oy ? wy : 1.0f - wy) * (oz ? wz : 1.0f - wz);
    }
}

template <bool WITH_MLP>
__global__ void __launch_bounds__(NTHREADS) hashgrid_fwd_kernel(LevelMeta m, const float* __restrict__ points,
                                                                int64_t n, const float2* __restrict__ grid,
                                                                const float* __restrict__ W1,
                                                                const float* __restrict__ W2,
                                                                float* __restrict__ out) {
    __shared__ float s_enc[TILE][ENC + 1];
    __shared__ float s_w1[HID][ENC + 1];
    __shared__ float s_w2[NOUT][HID];
    __shared__ float s_part[4][TILE][NOUT];
    const int tid = threadIdx.x;
    if (WITH_MLP) {
        for (int i = tid; i < HID * ENC; i += NTHREADS) s_w1[i / ENC][i % ENC] = W1[i];
        for (int i = tid; i < NOUT * HID; i += NTHREADS) s_w2[i / HID][i % HID] = W2[i];
    }
    const int lp = tid % TILE;   // point within the tile
    const int lg = tid / TILE;   // level group (gather) / hidden group (MLP)
    const int64_t n_tiles = (n + TILE - 1) / TILE;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        int64_t p = tile * TILE + lp;
        __syncthreads();
        if (p < n) {
            float x = (points[3 * p] - m.bmin) * m.inv_ext;
            float y = (points[3 * p + 1] - m.bmin) * m.inv_ext;
            float z = (points[3 * p + 2] - m.bmin) * m.inv_ext;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int l = lg * 4 + j;
                float e0 = 0.f, e1 = 0.f;
                if (l < m.n_levels) {
                    Corner c;
                    level_corners(m, l, x, y, z, c);
                    float2 g[8];
#pragma unroll
                    for (int k = 0; k < 8; ++k) g[k] = __ldg(grid + c.idx[k]);
#pragma unroll
                    for (int k = 0; k < 8; ++k) { e0 = fmaf(c.w[k], g[k].x, e0); e1 = fmaf(c.w[k], g[k].y, e1); }
                }
                s_enc[lp][2 * l] = e0; s_enc[lp][2 * l + 1] = e1;
            }
        }
        __syncthreads();
        if (!WITH_MLP) {
            for (int i = tid; i < TILE * ENC; i += NTHREADS) {
                int64_t pp = tile * TILE + i / ENC;
                if (pp < n) out[pp * ENC + (i % ENC)] = s_enc[i / ENC][i % ENC];
            }
            continue;
        }
        // MLP: thread (lp, lg) computes hidden units [16*lg, 16*lg+16) of point lp
        float o[NOUT] = {0, 0, 0, 0, 0};
        {
            float e[ENC];
#pragma unroll
            for (int k = 0; k < ENC; ++k) e[k] = s_enc[lp][k];
#pragma unroll 4
            for (int hh = 0; hh < 16; ++hh) {
                int h = lg * 16 + hh;
                float a = 0.f;
#pragma unroll
                for (int k = 0; k < ENC; ++k) a = fmaf(e[k], s_w1[h][k], a);
                a = fmaxf(a, 0.f);
#pragma unroll
                for (int c = 0; c < NOUT; ++c) o[c] = fmaf(a, s_w2[c][h], o[c]);
            }
        }
#pragma unroll
        for (int c = 0; c < NOUT; ++c) s_part[lg][lp][c] = o[c];
        __syncthreads();
        for (int i = tid; i < TILE * NOUT; i += NTHREADS) {
            int q = i / NOUT, c = i % NOUT;
            int64_t pp = tile * TILE + q;
            if (pp < n) out[pp * NOUT + c] = (s_part[0][q][c] + s_part[1][q][c]) + (s_part[2][q][c] + s_part[3][q][c]);
        }
    }
}

__global__ void __launch_bounds__(NTHREADS) hashgrid_bwd_kernel(LevelMeta m, const float* __restrict__ points,
                                                                int64_t n, const float2* __restrict__ grid,
                                                                const float* __restrict__ W1,
                                                                const float* __restrict__ W2,
                                                                const float* __restrict__ dout,
                                                                const uint32_t* __restrict__ hdr,
                                                                unsigned long long* __restrict__ acc_grid,
                                                                float* __restrict__ dgrid, float* __restrict__ dw_part) {
    const double S = fixed_scale(hdr, n);
    __shared__ float s_enc[TILE][ENC + 1];
    __shared__ float s_w1[HID][ENC + 1];
    __shared__ float s_w2[NOUT][HID];
    __shared__ float s_dw1[HID][ENC + 1];
    __shared__ float s_dw2[NOUT][HID];
    __shared__ float s_hid[TILE][HID + 1];   // relu(h), later reused as dh
    __shared__ float s_do[TILE][NOUT];
    const int tid = threadIdx.x;
    for (int i = tid; i < HID * ENC; i += NTHREADS) { s_w1[i / ENC][i % ENC] = W1[i]; s_dw1[i / ENC][i % ENC] = 0.f; }
    for (int i = tid; i < NOUT * HID; i += NTHREADS) { s_w2[i / HID][i % HID] = W2[i]; s_dw2[i / HID][i % HID] = 0.f; }
    const int lp = tid % TILE, lg = tid / TILE;
    const int64_t n_tiles = (n + TILE - 1) / TILE;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        int64_t p = tile * TILE + lp;
        bool valid = p < n;
        float x = 0, y = 0, z = 0;
        __syncthreads();
        if (valid) {
            x = (points[3 * p] - m.bmin) * m.inv_ext;
            y = (points[3 * p + 1] - m.bmin) * m.inv_ext;
            z = (points[3 * p + 2] - m.bmin) * m.inv_ext;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int l = lg * 4 + j;
            float e0 = 0.f, e1 = 0.f;
            if (valid && l < m.n_levels) {
                Corner c;
                level_corners(m, l, x, y, z, c);
#pragma unroll
                for (int k = 0; k < 8; ++k) { float2 g = __ldg(grid + c.idx[k]); e0 = fmaf(c.w[k], g.x, e0); e1 = fmaf(c.w[k], g.y, e1); }
            }
            s_enc[lp][2 * l] = e0; s_enc[lp][2 * l + 1] = e1;
        }
        for (int i = tid; i < TILE * NOUT; i += NTHREADS) {
            int64_t pp = tile * TILE + i / NOUT;
            s_do[i / NOUT][i % NOUT] = (pp < n) ? dout[pp * NOUT + (i % NOUT)] : 0.f;
        }
        __syncthreads();
        // hidden activations relu(h) (kept in smem for dW2), dh computed in the next pass
        {
            float e[ENC];
#pragma unroll
            for (int k = 0; k < ENC; ++k) e[k] = s_enc[lp][k];
#pragma unroll 4
            for (int hh = 0; hh < 16; ++hh) {
                int h = lg * 16 + hh;
                float a = 0.f;
#pragma unroll
                for (int k = 0; k < ENC; ++k) a = fmaf(e[k], s_w1[h][k], a);
                s_hid[lp][h] = fmaxf(a, 0.f);
            }
        }
        __syncthreads();
        // dW2 += sum_p dout[p][c] * relu_h[p][h]   (320 outputs, 256 threads)
        for (int i = tid; i < NOUT * HID; i += NTHREADS) {
            int c = i / HID, h = i % HID;
            float acc = 0.f;
#pragma unroll 8
            for (int q = 0; q < TILE; ++q) acc = fmaf(s_do[q][c], s_hid[q][h], acc);
            s_dw2[c][h] += acc;
        }
        __syncthreads();
        // overwrite s_hid with dh
        {
            float d0 = s_do[lp][0], d1 = s_do[lp][1], d2 = s_do[lp][2], d3 = s_do[lp][3], d4 = s_do[lp][4];
#pragma unroll 4
            for (int hh = 0; hh < 16; ++hh) {
                int h = lg * 16 + hh;
                float r = s_hid[lp][h];
                float dh = (r > 0.f) ? (d0 * s_w2[0][h] + d1 * s_w2[1][h] + d2 * s_w2[2][h] + d3 * s_w2[3][h] + d4 * s_w2[4][h]) : 0.f;
                s_hid[lp][h] = dh;
            }
        }
        __syncthreads();
        // dW1[h][k] += sum_p dh[p][h] * enc[p][k]   (2048 outputs, 8 per thread)
        for (int i = tid; i < HID * ENC; i += NTHREADS) {
            int h = i / ENC, k = i % ENC;
            float acc = 0.f;
#pragma unroll 8
            for (int q = 0; q < TILE; ++q) acc = fmaf(s_hid[q][h], s_enc[q][k], acc);
            s_dw1[h][k] += acc;
        }
        // denc[p][k] = sum_h dh[p][h] * W1[h][k]; thread (lp, lg) -> k in [8*lg, 8*lg+8)
        {
            float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            for (int h = 0; h < HID; ++h) {
                float dh = s_hid[lp][h];
#pragma unroll
                for (int kk = 0; kk < 8; ++kk) acc[kk] = fmaf(dh, s_w1[h][lg * 8 + kk], acc[kk]);
            }
            // levels [4*lg, 4*lg+4) own encoding columns [8*lg, 8*lg+8): scatter directly
            if (lg < 2) {
                // Coarse levels (0-7): the 32 consecutive surface points of a warp fall into a handful of cells, so
                // plain atomics serialise on the same few addresses (level 0 has 4 913 vertices for ~10^5 points).
                // Runs of equal vertex index along the warp are summed with a segmented shuffle reduction and only the
                // head lane of each run issues the atomic.  (lg is warp-uniform: a warp is 32 points of one level group.)
                const int lane = tid & 31;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    int l = lg * 4 + j;
                    if (l < m.n_levels) {               // warp-uniform
                        Corner c;
                        if (valid) level_corners(m, l, x, y, z, c);
                        float g0 = acc[2 * j], g1 = acc[2 * j + 1];
#pragma unroll
                        for (int k = 0; k < 8; ++k) {
                            uint32_t idx = valid ? c.idx[k] : 0xffffffffu;
                            float v0 = valid ? c.w[k] * g0 : 0.f, v1 = valid ? c.w[k] * g1 : 0.f;
                            uint32_t prev = __shfl_up_sync(0xffffffffu, idx, 1);
                            const bool head = (lane == 0) || (idx != prev);
                            const unsigned heads = __ballot_sync(0xffffffffu, head);
                            const unsigned after = (lane == 31) ? 0u : (heads >> (lane + 1));   // heads at lane+1, lane+2, ...
#pragma unroll
                            for (int d = 1; d < 32; d <<= 1) {
                                float o0 = __shfl_down_sync(0xffffffffu, v0, d), o1 = __shfl_down_sync(0xffffffffu, v1, d);
                                // lane + d belongs to this lane's run iff no head lies in (lane, lane + d]
                                if (lane + d < 32 && (after & ((1u << d) - 1u)) == 0u) { v0 += o0; v1 += o1; }
                            }
                            if (head && idx != 0xffffffffu) { fixed_add(acc_grid, dgrid, 2 * (int64_t)idx, v0, S); fixed_add(acc_grid, dgrid, 2 * (int64_t)idx + 1, v1, S); }
                        }
                    }
                }
            } else if (valid) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    int l = lg * 4 + j;
                    if (l < m.n_levels) {
                        Corner c;
                        level_corners(m, l, x, y, z, c);
                        float g0 = acc[2 * j], g1 = acc[2 * j + 1];
#pragma unroll
                        for (int k = 0; k < 8; ++k) { fixed_add(acc_grid, dgrid, 2 * (int64_t)c.idx[k], c.w[k] * g0, S); fixed_add(acc_grid, dgrid, 2 * (int64_t)c.idx[k] + 1, c.w[k] * g1, S); }
                    }
                }
            }
        }
    }
    __syncthreads();
    float* row = dw_part + (int64_t)blockIdx.x * DW_ROW;
    for (int i = tid; i < HID * ENC; i += NTHREADS) row[i] = s_dw1[i / ENC][i % ENC];
    for (int i = tid; i < NOUT * HID; i += NTHREADS) row[HID * ENC + i] = s_dw2[i / HID][i % HID];
}

// bound of every finite grid-gradient contribution c.w * denc (c.w <= 1): |denc_k| <= |dout_p|_1 * max|W2| * sum_h |W1[h][k]|
// (non-finite entries are left out: their contributions take the direct path of fixed_add).
// hdr[0] = max_p |dout_p|_1, hdr[1] = max|W2|, hdr[2] = max_k sum_h |W1[h][k]| (float bits; non-negative floats order like
// their bit patterns, so atomicMax on them is exact and order-independent).  hdr[0] is zeroed by the host first.
__global__ void __launch_bounds__(256) hashgrid_bound_kernel(const float* __restrict__ dout, int64_t n, const float* __restrict__ W1,
                                                             const float* __restrict__ W2, uint32_t* __restrict__ hdr) {
    float mx = 0.f;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
        float a = 0.f;
#pragma unroll
        for (int c = 0; c < NOUT; ++c) { const float d = fabsf(dout[p * NOUT + c]); if (isfinite(d)) a += d; }
        if (isfinite(a)) mx = fmaxf(mx, a);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) atomicMax(hdr, __float_as_uint(mx));
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        float w2 = 0.f, w1 = 0.f;
        for (int i = 0; i < NOUT * HID; ++i) if (isfinite(W2[i])) w2 = fmaxf(w2, fabsf(W2[i]));
        for (int k = 0; k < ENC; ++k) {
            float c = 0.f;
            for (int h = 0; h < HID; ++h) if (isfinite(W1[h * ENC + k])) c += fabsf(W1[h * ENC + k]);
            if (isfinite(c)) w1 = fmaxf(w1, c);
        }
        hdr[1] = __float_as_uint(w2); hdr[2] = __float_as_uint(w1);
    }
}

// dgrid += fixed-point sums / S, and the accumulator goes back to zero for the next call
__global__ void __launch_bounds__(256) hashgrid_fixed_flush_kernel(const uint32_t* __restrict__ hdr, int64_t n, int64_t count,
                                                                   unsigned long long* __restrict__ acc_grid, float* __restrict__ dgrid) {
    const double inv = 1.0 / fixed_scale(hdr, n);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long v = acc_grid[i];
        if (v) { dgrid[i] += (float)((double)(long long)v * inv); acc_grid[i] = 0ull; }
    }
}

// dW1 | dW2 += the blocks' rows, in block order
__global__ void __launch_bounds__(256) hashgrid_dw_reduce_kernel(const float* __restrict__ dw_part, int blocks, float* __restrict__ dW1,
                                                                 float* __restrict__ dW2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= DW_ROW) return;
    float a = 0.f;
    for (int b = 0; b < blocks; ++b) a += dw_part[(int64_t)b * DW_ROW + i];
    if (i < HID * ENC) dW1[i] += a; else dW2[i - HID * ENC] += a;
}

}  // namespace

extern "C" int64_t dm_hashgrid_layout(const dm_hashgrid_cfg* cfg, uint32_t* offsets_host) {
    LevelMeta m; int64_t total = 0;
    if (make_meta(cfg, m, &total) != DM_OK) return -1;
    if (offsets_host) {
        for (int l = 0; l < m.n_levels; ++l) offsets_host[l] = m.offset[l];
        offsets_host[m.n_levels] = (uint32_t)total;
    }
    return total;
}

static int check_mlp(const dm_hashgrid_cfg* cfg) {
    if (cfg->n_levels * cfg->n_features != ENC || cfg->n_hidden != HID || cfg->n_out != NOUT) {
        dm_set_error("fused MLP supports 16x2 -> 64 -> 5 only (got %dx%d -> %d -> %d)", cfg->n_levels, cfg->n_features,
                     cfg->n_hidden, cfg->n_out);
        return DM_EUNSUPPORTED;
    }
    return DM_OK;
}

extern "C" int dm_hashgrid_mlp_fwd(const dm_hashgrid_cfg* cfg, const float* points, int64_t n, const float* grid,
                                   const float* W1, const float* W2, float* features, void* stream) {
    if (n == 0) return DM_OK;
    DM_REQUIRE(cfg && points && grid && W1 && W2 && features, "null pointer");
    LevelMeta m; int rc = make_meta(cfg, m, nullptr); if (rc) return rc;
    rc = check_mlp(cfg); if (rc) return rc;
    int64_t tiles = dm_ceil_div(n, TILE);
    int grid_dim = (int)(tiles < (int64_t)DM_NUM_SMS * 4 ? tiles : (int64_t)DM_NUM_SMS * 4);
    hashgrid_fwd_kernel<true><<<grid_dim, NTHREADS, 0, (cudaStream_t)stream>>>(m, points, n, (const float2*)grid, W1, W2, features);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_hashgrid_encode(const dm_hashgrid_cfg* cfg, const float* points, int64_t n, const float* grid,
                                  float* enc, void* stream) {
    if (n == 0) return DM_OK;
    DM_REQUIRE(cfg && points && grid && enc, "null pointer");
    LevelMeta m; int rc = make_meta(cfg, m, nullptr); if (rc) return rc;
    DM_REQUIRE(cfg->n_levels == 16, "encode-only path expects 16 levels");
    int64_t tiles = dm_ceil_div(n, TILE);
    int grid_dim = (int)(tiles < (int64_t)DM_NUM_SMS * 4 ? tiles : (int64_t)DM_NUM_SMS * 4);
    hashgrid_fwd_kernel<false><<<grid_dim, NTHREADS, 0, (cudaStream_t)stream>>>(m, points, n, (const float2*)grid, nullptr, nullptr, enc);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_hashgrid_mlp_bwd(const dm_hashgrid_cfg* cfg, const float* points, int64_t n, const float* grid,
                                   const float* W1, const float* W2, const float* dfeatures, float* dgrid, float* dW1,
                                   float* dW2, void* stream) {
    if (n == 0) return DM_OK;
    DM_REQUIRE(cfg && points && grid && W1 && W2 && dfeatures && dgrid && dW1 && dW2, "null pointer");
    LevelMeta m; int64_t total = 0; int rc = make_meta(cfg, m, &total); if (rc) return rc;
    rc = check_mlp(cfg); if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    // header | per-block weight-gradient rows | int64 accumulator [total * 2] (zero between calls: the flush re-zeroes it)
    void* scratch = dm_scratch(DM_SCRATCH_HASHGRID, (size_t)(HDR_BYTES + (int64_t)BWD_MAX_BLOCKS * DW_ROW * 4 + total * 2 * 8), st);
    if (!scratch) return DM_EDRIVER;
    uint32_t* hdr = (uint32_t*)scratch;
    float* dw_part = (float*)((char*)scratch + HDR_BYTES);
    unsigned long long* acc_grid = (unsigned long long*)((char*)scratch + HDR_BYTES + (int64_t)BWD_MAX_BLOCKS * DW_ROW * 4);
    int64_t tiles = dm_ceil_div(n, TILE);
    int grid_dim = (int)(tiles < (int64_t)BWD_MAX_BLOCKS ? tiles : (int64_t)BWD_MAX_BLOCKS);
    DM_CHECK_CUDA(cudaMemsetAsync(hdr, 0, 4, st));
    hashgrid_bound_kernel<<<(unsigned)(dm_ceil_div(n, 256) < DM_NUM_SMS * 4 ? dm_ceil_div(n, 256) : DM_NUM_SMS * 4), 256, 0, st>>>(dfeatures, n, W1, W2, hdr);
    DM_CHECK_LAUNCH();
    hashgrid_bwd_kernel<<<grid_dim, NTHREADS, 0, st>>>(m, points, n, (const float2*)grid, W1, W2, dfeatures, hdr, acc_grid, dgrid, dw_part);
    DM_CHECK_LAUNCH();
    hashgrid_dw_reduce_kernel<<<(unsigned)dm_ceil_div(DW_ROW, 256), 256, 0, st>>>(dw_part, grid_dim, dW1, dW2);
    DM_CHECK_LAUNCH();
    hashgrid_fixed_flush_kernel<<<DM_NUM_SMS * 8, 256, 0, st>>>(hdr, n, total * 2, acc_grid, dgrid);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

__global__ void jitter_kernel(const float* __restrict__ pos, const float* __restrict__ nrm,
                              const float* __restrict__ rand_ang, const float* __restrict__ normal_eps, int64_t n,
                              float* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    f3 nn = ld3(nrm, i);
    f3 x = ortho_dir(nn);
    f3 y = cross3(nn, x);
    float ang = rand_ang[i] * 3.14159265358979323846f * 2.0f;
    float s, c;
    sincosf(ang, &s, &c);
    f3 ch = (c * x + s * y) * normal_eps[i];
    st3(out, i, ld3(pos, i) + ch);
}

extern "C" int dm_jitter_positions(const float* pos, const float* nrm, const float* rand_ang, const float* normal_eps,
                                   int64_t n, float* out, void* stream) {
    if (n == 0) return DM_OK;
    DM_REQUIRE(pos && nrm && rand_ang && normal_eps && out, "null pointer");
    jitter_kernel<<<(unsigned)dm_ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(pos, nrm, rand_ang, normal_eps, n, out);
    DM_CHECK_LAUNCH();
    return DM_OK;
}
