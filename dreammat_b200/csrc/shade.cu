// shade.cu -- PBR fragment shading of the compacted G-buffer (rows a4, a5 of SURVEY.md section 8).
//
//   dm_shade_mc_fwd        models/materials/dreammat_material.py:615-677 (shade_raytracing), with
//                          :554-573 sample_diffuse_directions, :575-596 sample_specular_directions,
//                          :599-604 distribution_ggx, :519-530 geometry_schlick(_ggx),
//                          :509-517 fresnel_schlick(_directions), :490-507 get_lights,
//                          :439-455 get_envirmentlight_blender, :110-123 material_smoothness_grad
//   dm_shade_splitsum_fwd  dreammat_material.py:679-711 (shade_splitsum)
//   dm_shade_bwd           what torch autograd does for either branch, in closed form
//
// Design (GPU-first).  The reference materialises >= 40 tensors of shape [pn,328,{1,3}] per view
// and keeps them for autograd.  Here one WARP owns one covered pixel: lanes stride over the 328
// light samples, each lane builds its direction, evaluates the BRDF terms, walks the BVH for
// occlusion (any-hit) and fetches one env-map texel; partial sums are folded with warp
// shuffles.  The derivative of the colour w.r.t. the five material scalars is carried
// FORWARD through the same pass (dual numbers in the roughness `a`, which is the only input
// the sampled directions depend on), so the backward is a 9-float-per-pixel Jacobian product
// and no ray is traced twice.  HBM traffic per pixel: 56 B of G-buffer/feature reads (staged
// through shared memory with coalesced loads), 12-108 B of outputs, plus one 16 B texel per
// unoccluded sample out of a float4-padded lat-long map (one 32 B sector per fetch).
#include <math_constants.h>
#include "bvh.cuh"

namespace {

constexpr float PI_F = 3.14159265358979323846f;
constexpr float TWO_PI_F = 6.28318530717958647692f;

struct Dual {
    float v, d;
};
__device__ __forceinline__ Dual mkd(float v, float d = 0.f) { Dual r; r.v = v; r.d = d; return r; }
__device__ __forceinline__ Dual operator+(Dual a, Dual b) { return mkd(a.v + b.v, a.d + b.d); }
__device__ __forceinline__ Dual operator-(Dual a, Dual b) { return mkd(a.v - b.v, a.d - b.d); }
__device__ __forceinline__ Dual operator*(Dual a, Dual b) { return mkd(a.v * b.v, a.d * b.v + a.v * b.d); }
__device__ __forceinline__ Dual operator+(Dual a, float b) { return mkd(a.v + b, a.d); }
__device__ __forceinline__ Dual operator-(Dual a, float b) { return mkd(a.v - b, a.d); }
__device__ __forceinline__ Dual operator-(float a, Dual b) { return mkd(a - b.v, -b.d); }
__device__ __forceinline__ Dual operator*(Dual a, float b) { return mkd(a.v * b, a.d * b); }
__device__ __forceinline__ Dual operator*(float b, Dual a) { return mkd(a.v * b, a.d * b); }
__device__ __forceinline__ Dual operator/(Dual a, Dual b) {
    float q = a.v / b.v;
    return mkd(q, (a.d - q * b.d) / b.v);
}
__device__ __forceinline__ Dual operator/(Dual a, float b) { return mkd(a.v / b, a.d / b); }
__device__ __forceinline__ Dual dsqrt(Dual a) {
    float s = sqrtf(a.v);
    return mkd(s, s > 0.0f ? a.d / (2.0f * s) : 0.0f);
}
// torch.clamp(x, 0, 1): gradient passes where 0 <= x <= 1
__device__ __forceinline__ Dual dclamp01(Dual a) {
    bool in = (a.v >= 0.0f) && (a.v <= 1.0f);
    return mkd(fminf(fmaxf(a.v, 0.0f), 1.0f), in ? a.d : 0.0f);
}
__device__ __forceinline__ Dual dpow5(Dual a) {
    float a2 = a.v * a.v, a4 = a2 * a2;
    return mkd(a4 * a.v, 5.0f * a4 * a.d);
}
struct D3 {
    Dual x, y, z;
};
__device__ __forceinline__ Dual ddot(D3 a, f3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ Dual ddot(D3 a, D3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

// distribution_ggx (:599-604): a2 / (pi * (NoH^2 (a2-1) + 1)^2 + 1e-4)
__device__ __forceinline__ Dual ggx_D(Dual NoH, Dual a) {
    Dual a2 = a * a;
    Dual den = NoH * NoH * (a2 - 1.0f) + 1.0f;
    return a2 / (PI_F * (den * den) + 1e-4f);
}
// geometry_schlick_ggx (:519-525): c / (c (1-k) + k + 1e-5), k = a/2
__device__ __forceinline__ Dual ggx_G1(Dual c, Dual a) {
    Dual k = a * 0.5f;
    return c / (c * (1.0f - k) + k + 1e-5f);
}

// get_envirmentlight_blender (:439-455): nearest texel of the lat-long map
__device__ __forceinline__ float4 env_fetch(const float4* __restrict__ env, int H, int W, f3 d) {
    float inv = 1.0f / sqrtf(dot3(d, d));
    float x = d.x * inv, y = d.y * inv, z = d.z * inv;
    float theta = acosf(z);
    float phi = atan2f(y, x);
    phi = phi - floorf(phi / TWO_PI_F) * TWO_PI_F;  // torch.remainder(phi, 2 pi)
    float u = -phi / TWO_PI_F + 0.5f;
    float v = theta / PI_F;
    float fx = u * (float)W; fx = fx - floorf(fx / (float)W) * (float)W;
    float fy = v * (float)H; fy = fy - floorf(fy / (float)H) * (float)H;
    int ix = min(max((int)fx, 0), W - 1);
    int iy = min(max((int)fy, 0), H - 1);
    return __ldg(env + (int64_t)iy * W + ix);
}

struct PixelIn {
    f3 p, n, v;
    float m[5], mj[5];
};

constexpr int MC_WARPS = 8;   // warps (= pixels) per CTA of shade_mc_kernel

struct McParams {
    dm_material_cfg cfg;
    BvhView bvh;
    const float4* env; int envH, envW;
    const float* tab_d; const float* tab_s;
    const float *pts, *normals, *viewdirs, *features, *features_jitter, *rand_d, *rand_s;
    int64_t n;
    float *color, *jac, *reg_sums;
    float *albedo, *roughness, *metalness, *spec_light, *diff_light, *spec_color, *diff_color;
    uint32_t* hit_bits;
    int frontier;       // dm_tune "mc_frontier": 1 shared-origin traversal (see origin_frontier below) | 0 root traversal
};

// Per-pixel quantities are warp-uniform; they live in shared memory (one record per warp) instead of being
// replicated in 32 lanes' registers -- the traversal loop is latency-bound and wants occupancy.
struct PixState {
    float p[3], n[3], v[3], r[3], xd[3], yd[3], xs[3], ys[3];
    float a, NoV, rd, rs, g1v, g1d;
};

// specular sample direction about the reflection vector (value and d/da), dreammat_material.py:575-596
__device__ __forceinline__ D3 spec_direction(const PixState& px, float phi0, float ue) {
    float phi = phi0 + px.rs;
    phi = phi - floorf(phi / TWO_PI_F) * TWO_PI_F;
    float sn, cs;
    sincosf(phi, &sn, &cs);
    const Dual aD = mkd(px.a, 1.0f);
    // cos_theta = sqrt((1-el+1e-6)/(1+(a^2-1) el+1e-6)+1e-6) (:585)
    Dual den = (aD * aD - 1.0f) * ue + (1.0f + 1e-6f);
    Dual ct = dsqrt(mkd(1.0f - ue + 1e-6f) / den + 1e-6f);
    Dual st = dsqrt(1.0f - ct * ct + 1e-6f);
    Dual cx = st * cs, cy = st * sn;
    D3 d;
    d.x = cx * px.xs[0] + cy * px.ys[0] + ct * px.r[0];
    d.y = cx * px.xs[1] + cy * px.ys[1] + ct * px.r[1];
    d.z = cx * px.xs[2] + cy * px.ys[2] + ct * px.r[2];
    return d;
}

// ---- shared-origin traversal.  All 328 occlusion rays of a pixel start (to 1e-5) at the same surface point p, so the
// part of the BVH whose boxes CONTAIN p -- a connected piece T_p hanging off the root, ~2 x depth nodes -- passes the slab
// test of every one of them.  One lane walks T_p once per pixel and leaves in shared memory
//   * the leaves inside T_p (the triangles around p: every ray tests them), and
//   * the FRONTIER: children of T_p nodes whose box does not contain p (box + child code).
// Each ray then runs two warp-uniform loops (local triangles, frontier boxes: broadcast loads, all lanes busy, no stack)
// and only descends, divergently, into the frontier subtrees its own slab test hit.  The set of boxes / triangles a ray
// can reach is exactly that of a root traversal (a box containing the origin always passes slab2), so the any-hit result
// is bit-identical.
constexpr int FR_MAX = 64;        // frontier entries per pixel = bits of the per-ray hit mask (overflow -> plain root traversal)
constexpr int FR_LEAF_MAX = 12;   // leaves of T_p
constexpr float FR_INSIDE = 3e-5f;  // p must sit this far inside a box to count as contained (ray origins are p + 1e-5 d, |d| = 1)
struct FrontierList {
    float box[FR_MAX][6];
    int code[FR_MAX];
    int leaf[FR_LEAF_MAX];
    int nf, nl;                   // nf < 0: overflow
};

__device__ __forceinline__ void origin_frontier(const BvhView& bv, f3 p, FrontierList& F) {
    int nf = 0, nl = 0, sp = 0;
    bool ok = true;
    int stk[40];
    int cur = bv.root;
    if (cur < 0) { F.leaf[0] = cur; F.nf = 0; F.nl = 1; return; }
    auto child = [&](int code, float lx, float ly, float lz, float hx, float hy, float hz) {
        const bool inside = p.x > lx + FR_INSIDE && p.x < hx - FR_INSIDE && p.y > ly + FR_INSIDE && p.y < hy - FR_INSIDE &&
                            p.z > lz + FR_INSIDE && p.z < hz - FR_INSIDE;
        if (inside) {
            if (code < 0) { if (nl < FR_LEAF_MAX) F.leaf[nl++] = code; else ok = false; }
            else { if (sp < 40) stk[sp++] = code; else ok = false; }
        } else {
            if (nf < FR_MAX) {
                F.box[nf][0] = lx; F.box[nf][1] = ly; F.box[nf][2] = lz; F.box[nf][3] = hx; F.box[nf][4] = hy; F.box[nf][5] = hz;
                F.code[nf] = code; ++nf;
            } else ok = false;
        }
    };
    while (ok) {
        const float4* n = bv.nodes + (int64_t)cur * 4;
        const float4 n0 = __ldg(n), n1 = __ldg(n + 1), n2 = __ldg(n + 2), n3 = __ldg(n + 3);
        child(__float_as_int(n3.x), n0.x, n0.y, n0.z, n0.w, n1.x, n1.y);
        child(__float_as_int(n3.y), n1.z, n1.w, n2.x, n2.y, n2.z, n2.w);
        if (sp == 0) break;
        cur = stk[--sp];
    }
    F.nf = ok ? nf : -1;
    F.nl = nl;
}

// any-hit over the frontier subtrees selected by `mask` (bit i = F.code[i]); same node / leaf steps as bvh_trace<true>
__device__ __forceinline__ bool anyhit_subtrees(const BvhView& bv, const FrontierList& F, unsigned long long mask, f3 o, f3 d,
                                                f3 inv, f3 oi) {
    int stack[DM_BVH_STACK];
    int sp = 0, cur = 0;
    bool alive = mask != 0ull;
    if (alive) { const int i = __ffsll((long long)mask) - 1; mask &= mask - 1ull; cur = F.code[i]; }
    while (alive) {
        while (alive && cur >= 0) {
            const float4* n = bv.nodes + (int64_t)cur * 4;
            float4 n0 = __ldg(n), n1 = __ldg(n + 1), n2 = __ldg(n + 2), n3 = __ldg(n + 3);
            float tl, tr;
            bool hl = slab2(n0.x, n0.y, n0.z, n0.w, n1.x, n1.y, inv, oi, DM_RT_MAX_DIST, tl);
            bool hr = slab2(n1.z, n1.w, n2.x, n2.y, n2.z, n2.w, inv, oi, DM_RT_MAX_DIST, tr);
            int cl = __float_as_int(n3.x), cr = __float_as_int(n3.y);
            if (hl && hr) {
                bool lfirst = tl <= tr;
                if (sp < DM_BVH_STACK) stack[sp++] = lfirst ? cr : cl;
                cur = lfirst ? cl : cr;
            } else if (hl) cur = cl;
            else if (hr) cur = cr;
            else if (sp > 0) cur = stack[--sp];
            else if (mask) { const int i = __ffsll((long long)mask) - 1; mask &= mask - 1ull; cur = F.code[i]; }
            else alive = false;
        }
        if (!alive) break;
        {
            const int code = ~cur;
            const int first = code >> 2, cnt = (code & 3) + 1;
            for (int k = 0; k < cnt; ++k) {
                const float4* tp = bv.tris + (int64_t)(first + k) * 3;
                float4 A = __ldg(tp), B = __ldg(tp + 1), C = __ldg(tp + 2);
                float u, v;
                if (tri_hit_pre(o, d, A, B, C, u, v) < DM_RT_MAX_DIST) return true;
            }
        }
        if (sp > 0) cur = stack[--sp];
        else if (mask) { const int i = __ffsll((long long)mask) - 1; mask &= mask - 1ull; cur = F.code[i]; }
        else break;
    }
    return false;
}

// One warp per pixel.  4 CTAs (32 warps) resident per SM hold the allocation to 64 registers at the price of some spills;
// the traversal is latency-bound and gains more from the extra warps than it loses to the spills.
__global__ void __launch_bounds__(MC_WARPS * 32, 4) shade_mc_kernel(McParams P) {
    extern __shared__ float s_tab[];  // [nd*3 | ns*2]: (az0, sqrt(ue+1e-7), sqrt(1-ue+1e-7)) | (phi0, ue)
    __shared__ float s_in[MC_WARPS][20];
    __shared__ PixState s_px[MC_WARPS];
    __shared__ FrontierList s_fr[MC_WARPS];
    const int nd = P.cfg.n_diffuse, ns = P.cfg.n_specular, S = nd + ns;
    float* s_td = s_tab;
    float* s_ts = s_tab + 3 * nd;
    uint16_t* s_list = reinterpret_cast<uint16_t*>(s_tab + 3 * nd + 2 * ns);   // [MC_WARPS][S] compacted sample ids
    for (int i = threadIdx.x; i < nd; i += blockDim.x) {
        float ua = P.tab_d[2 * i], ue = P.tab_d[2 * i + 1];
        s_td[3 * i] = ua * PI_F * 2.0f;            // az = az * pi * 2 (:563)
        s_td[3 * i + 1] = sqrtf(ue + 1e-7f);       // el_sqrt (:564)
        s_td[3 * i + 2] = sqrtf(1.0f - ue + 1e-7f);  // coeff_z (:567)
    }
    for (int i = threadIdx.x; i < ns; i += blockDim.x) {
        s_ts[2 * i] = PI_F * 2.0f * P.tab_s[2 * i];  // phi = pi * 2 * az (:583)
        s_ts[2 * i + 1] = P.tab_s[2 * i + 1];
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t pix = (int64_t)blockIdx.x * MC_WARPS + warp;
    if (pix >= P.n) return;
    // coalesced staging of the 19 per-pixel input floats through shared memory
    if (lane < 3) s_in[warp][lane] = P.pts[3 * pix + lane];
    else if (lane < 6) s_in[warp][lane] = P.normals[3 * pix + lane - 3];
    else if (lane < 9) s_in[warp][lane] = P.viewdirs[3 * pix + lane - 6];
    else if (lane < 14) s_in[warp][lane] = P.features[5 * pix + lane - 9];
    else if (lane < 19) s_in[warp][lane] = P.features_jitter[5 * pix + lane - 14];
    __syncwarp();
    const float* si = s_in[warp];
    PixState& px = s_px[warp];
    if (lane == 0) {
        const f3 p = mk3(si[0], si[1], si[2]), n = mk3(si[3], si[4], si[5]), v = mk3(si[6], si[7], si[8]);
        const float a = sigmoidf_(si[13]) * (P.cfg.max_roughness - P.cfg.min_roughness) + P.cfg.min_roughness;
        const float ndv = dot3(v, n);
        const f3 r = (ndv * n) * 2.0f - v;  // reflections (:620)
        const f3 xd = ortho_dir(n), yd = cross3(n, xd), xs = ortho_dir(r), ys = cross3(r, xs);
        const float NoV = fminf(fmaxf(ndv, 0.f), 1.f);
        const Dual g1 = ggx_G1(mkd(NoV), mkd(a, 1.0f));
        px.p[0] = p.x; px.p[1] = p.y; px.p[2] = p.z; px.n[0] = n.x; px.n[1] = n.y; px.n[2] = n.z;
        px.v[0] = v.x; px.v[1] = v.y; px.v[2] = v.z; px.r[0] = r.x; px.r[1] = r.y; px.r[2] = r.z;
        px.xd[0] = xd.x; px.xd[1] = xd.y; px.xd[2] = xd.z; px.yd[0] = yd.x; px.yd[1] = yd.y; px.yd[2] = yd.z;
        px.xs[0] = xs.x; px.xs[1] = xs.y; px.xs[2] = xs.z; px.ys[0] = ys.x; px.ys[1] = ys.y; px.ys[2] = ys.z;
        px.a = a; px.NoV = NoV; px.g1v = g1.v; px.g1d = g1.d;
        px.rd = P.rand_d[pix] * PI_F * 2.0f; px.rs = P.rand_s[pix] * PI_F * 2.0f;
        if (P.frontier) origin_frontier(P.bvh, p, s_fr[warp]);
    }
    __syncwarp();
    const FrontierList& FR = s_fr[warp];
    const bool use_frontier = P.frontier && FR.nf >= 0;
    const float kd_pdf = (float)nd / (float)(ns + nd), ks_pdf = (float)ns / (float)(ns + nd);

    float Ld[3] = {0, 0, 0}, Ls[3] = {0, 0, 0};
    float U[3] = {0, 0, 0}, V[3] = {0, 0, 0};      // sum L*w, sum L*w*fh
    float Ud[3] = {0, 0, 0}, Vd[3] = {0, 0, 0};    // d/da of the above with fh held fixed
    float Wd[3] = {0, 0, 0};                       // sum L*w*dfh/da

    // ---- work list.  Specular samples whose direction falls below the horizon have NoL = 0 -> G = 0 -> weight and
    // d(weight)/da exactly 0; unless the aux light maps are requested their radiance is never used, so they are not
    // traced.  Instead of idling their lanes, the surviving sample ids are compacted (ballot + prefix count) behind the
    // diffuse ids, so every pass of the loop below runs with 32 live rays and there are fewer passes.
    uint16_t* list = s_list + warp * S;
    const bool compact = !P.spec_light && !P.hit_bits;
    int count;
    if (compact) {
        for (int i = lane; i < nd; i += 32) list[i] = (uint16_t)i;
        count = nd;
        for (int j0 = 0; j0 < ns; j0 += 32) {
            const int j = j0 + lane;
            bool act = false;
            if (j < ns) {
                D3 d = spec_direction(px, s_ts[2 * j], s_ts[2 * j + 1]);
                act = (d.x.v * px.n[0] + d.y.v * px.n[1] + d.z.v * px.n[2]) > 0.0f;
            }
            const unsigned bal = __ballot_sync(0xffffffffu, act);
            if (act) list[count + __popc(bal & ((1u << lane) - 1u))] = (uint16_t)(nd + j);
            count += __popc(bal);
        }
    } else {
        for (int i = lane; i < S; i += 32) list[i] = (uint16_t)i;
        count = S;
    }
    __syncwarp();
    auto sample_dir = [&](int s) -> D3 {                       // sample direction (value and d/da), :554-596
        D3 d;
        if (s < nd) {
            float az = s_td[3 * s] + px.rd;
            az = az - floorf(az / TWO_PI_F) * TWO_PI_F;  // % (2 pi)
            float sn, cs;
            sincosf(az, &sn, &cs);
            float cx = s_td[3 * s + 1] * cs, cy = s_td[3 * s + 1] * sn, cz = s_td[3 * s + 2];
            d.x = mkd(cx * px.xd[0] + cy * px.yd[0] + cz * px.n[0]);
            d.y = mkd(cx * px.xd[1] + cy * px.yd[1] + cz * px.n[1]);
            d.z = mkd(cx * px.xd[2] + cy * px.yd[2] + cz * px.n[2]);
        } else {
            const int j = s - nd;
            d = spec_direction(px, s_ts[2 * j], s_ts[2 * j + 1]);
        }
        return d;
    };
    auto shade_sample = [&](int s, const D3& d) {             // unoccluded sample: BRDF terms (value and d/da) + env texel (:615-677)
        const bool spec = s >= nd;
        const f3 dv = mk3(d.x.v, d.y.v, d.z.v);
        const f3 n = mk3(px.n[0], px.n[1], px.n[2]), v = mk3(px.v[0], px.v[1], px.v[2]);
        const Dual aD = mkd(px.a, 1.0f);
        D3 h; h.x = d.x + v.x; h.y = d.y + v.y; h.z = d.z + v.z;   // H = normalize(v + d) (:513-514)
        Dual hl = dsqrt(ddot(h, h));
        float hlc = fmaxf(hl.v, 1e-12f);
        Dual hinv = mkd(1.0f / hlc, (hl.v > 1e-12f) ? (-hl.d / (hlc * hlc)) : 0.0f);
        D3 Hh; Hh.x = h.x * hinv; Hh.y = h.y * hinv; Hh.z = h.z * hinv;
        Dual HoV = dclamp01(ddot(Hh, v));
        Dual fh = dpow5(dclamp01(1.0f - HoV));
        Dual NoL = dclamp01(ddot(d, n));
        Dual NoH = dclamp01(ddot(Hh, n));
        Dual Dg = ggx_D(NoH, aD);
        Dual G = mkd(px.g1v, px.g1d) * ggx_G1(NoL, aD);
        Dual pdf;
        if (!spec) pdf = mkd(NoL.v / PI_F * kd_pdf);
        else pdf = Dg * NoH / (4.0f * HoV + 1e-5f) * ks_pdf;
        Dual w = Dg * G / (4.0f * px.NoV * pdf + 1e-5f);
        float4 L4 = env_fetch(P.env, P.envH, P.envW, dv);
        const float L[3] = {L4.x, L4.y, L4.z};
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            if (!spec) Ld[c] += L[c]; else Ls[c] += L[c];
            float lw = L[c] * w.v;
            U[c] += lw; V[c] += lw * fh.v;
            float lwd = L[c] * w.d;
            Ud[c] += lwd; Vd[c] += lwd * fh.v;
            Wd[c] += lw * fh.d;
        }
    };
    auto mark_hit = [&](int s) {
        if (P.hit_bits) atomicOr(P.hit_bits + pix * ((S + 31) / 32) + (s >> 5), 1u << (s & 31));
    };
    // ---- lane = slot of the work list, all lanes in step.  Samples are visited in table order (Fibonacci points sorted
    // by elevation).  With the frontier, local triangles and frontier boxes are tested coherently and each ray descends
    // only into the frontier subtrees its slab test hit.
    for (int base = 0; base < count; base += 32) {
        const bool in_range = base + lane < count;
        const int s = in_range ? list[base + lane] : 0;
        const D3 d = sample_dir(s);
        const f3 dv = mk3(d.x.v, d.y.v, d.z.v);
        // a specular sample below the horizon has NoL = 0 -> G = 0 -> weight and d(weight)/da exactly 0: unless the
        // aux light maps are requested its radiance is never used, so the ray need not be traced
        const bool valid = in_range && !(compact && s >= nd && (dv.x * px.n[0] + dv.y * px.n[1] + dv.z * px.n[2]) <= 0.0f);
        // ---- occlusion first (:490-507): occluded samples contribute nothing, skip their BRDF math
        bool hit = false;
        const f3 o = mk3(px.p[0] + dv.x * 1e-5f, px.p[1] + dv.y * 1e-5f, px.p[2] + dv.z * 1e-5f);
        if (use_frontier) {
            // (1) the triangles around p: warp-uniform loop, broadcast loads
            for (int li = 0; li < FR.nl; ++li) {
                const int code = ~FR.leaf[li];
                const int first = code >> 2, cnt = (code & 3) + 1;
                for (int k = 0; k < cnt; ++k) {
                    const float4* tp = P.bvh.tris + (int64_t)(first + k) * 3;
                    const float4 A = __ldg(tp), B = __ldg(tp + 1), C = __ldg(tp + 2);
                    float u, v;
                    if (valid && !hit && tri_hit_pre(o, dv, A, B, C, u, v) < DM_RT_MAX_DIST) hit = true;
                }
            }
            // (2) frontier boxes: warp-uniform loop over shared memory
            const f3 inv = mk3(1.0f / dv.x, 1.0f / dv.y, 1.0f / dv.z);
            const f3 oi = mk3(o.x * inv.x, o.y * inv.y, o.z * inv.z);
            unsigned long long mask = 0ull;
            if (valid && !hit) {
                for (int i = 0; i < FR.nf; ++i) {
                    float tn;
                    if (slab2(FR.box[i][0], FR.box[i][1], FR.box[i][2], FR.box[i][3], FR.box[i][4], FR.box[i][5], inv, oi,
                              DM_RT_MAX_DIST, tn)) mask |= 1ull << i;
                }
            }
            // (3) divergent descent into the frontier subtrees this ray's slab test hit
            if (mask) hit = anyhit_subtrees(P.bvh, FR, mask, o, dv, inv, oi);
        } else if (valid) {
            float bt, bu, bvv; int bid;
            hit = bvh_trace<true>(P.bvh, o, dv, bt, bid, bu, bvv);
        }
        if (valid && hit) mark_hit(s);
        if (valid && !hit) shade_sample(s, d);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        Ld[c] = warp_sum(Ld[c]); Ls[c] = warp_sum(Ls[c]);
        U[c] = warp_sum(U[c]); V[c] = warp_sum(V[c]);
        Ud[c] = warp_sum(Ud[c]); Vd[c] = warp_sum(Vd[c]); Wd[c] = warp_sum(Wd[c]);
    }
    if (lane == 0) {
        float m[5], mj[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) { m[k] = sigmoidf_(si[9 + k]); mj[k] = sigmoidf_(si[14 + k]); }
        // material_smoothness_grad (:110-123)
        float k0 = fabsf(m[0] - mj[0]), k1 = fabsf(m[1] - mj[1]), k2 = fabsf(m[2] - mj[2]);
        const float reg_kd = ((k0 + k1 + k2) / 3.0f) * k2;
        const float reg_ks = fabsf(m[3] - mj[3]) * fabsf(m[4] - mj[4]);
        const float alb[3] = {fminf(fmaxf(m[0], 0.f), 1.f), fminf(fmaxf(m[1], 0.f), 1.f), fminf(fmaxf(m[2], 0.f), 1.f)};
        const float met = m[3] * (P.cfg.max_metallic - P.cfg.min_metallic) + P.cfg.min_metallic;
        const float a = px.a;
        const float invS = 1.0f / (float)S, invd = 1.0f / (float)nd, invs = 1.0f / (float)ns;
        float colv[3], specv[3], diffv[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float F0 = 0.04f * (1.0f - met) + met * alb[c];
            float spec = (F0 * (U[c] - V[c]) + V[c]) * invS;
            float diff = alb[c] * (Ld[c] * invd);
            float lin = diff + spec;
            float g = lin2srgb_grad(lin);
            float dS_dF0 = (U[c] - V[c]) * invS;
            float dS_da = (F0 * (Ud[c] - Vd[c]) + Vd[c] + (1.0f - F0) * Wd[c]) * invS;
            colv[c] = lin2srgb_f(lin); specv[c] = spec; diffv[c] = diff;
            P.jac[9 * pix + 3 * c + 0] = g * (Ld[c] * invd + dS_dF0 * met);          // d/d albedo_c
            P.jac[9 * pix + 3 * c + 1] = g * (dS_dF0 * (alb[c] - 0.04f));            // d/d metallic
            P.jac[9 * pix + 3 * c + 2] = g * dS_da;                                   // d/d a
        }
        st3(P.color, pix, mk3(colv[0], colv[1], colv[2]));
        if (P.albedo) st3(P.albedo, pix, mk3(lin2srgb_f(alb[0]), lin2srgb_f(alb[1]), lin2srgb_f(alb[2])));
        if (P.roughness) P.roughness[pix] = sqrtf(a + 1e-7f);
        if (P.metalness) P.metalness[pix] = met;
        if (P.spec_light) st3(P.spec_light, pix, mk3(lin2srgb_f(Ls[0] * invs), lin2srgb_f(Ls[1] * invs), lin2srgb_f(Ls[2] * invs)));
        if (P.diff_light) st3(P.diff_light, pix, mk3(lin2srgb_f(Ld[0] * invd), lin2srgb_f(Ld[1] * invd), lin2srgb_f(Ld[2] * invd)));
        if (P.spec_color) st3(P.spec_color, pix, mk3(lin2srgb_f(specv[0]), lin2srgb_f(specv[1]), lin2srgb_f(specv[2])));
        if (P.diff_color) st3(P.diff_color, pix, mk3(lin2srgb_f(diffv[0]), lin2srgb_f(diffv[1]), lin2srgb_f(diffv[2])));
        if (P.reg_sums && (reg_kd != 0.f || reg_ks != 0.f)) {
            atomicAdd(P.reg_sums, reg_kd);
            atomicAdd(P.reg_sums + 1, reg_ks);
        }
    }
}


// ------------------------------------------------------------------------------------------ split-sum

struct SsParams {
    dm_material_cfg cfg;
    const float* lut; int lut_res;
    const float* dcube; int dres; int dcube_smem;
    const float* mips[8]; int n_mips; int res0;
    const float *normals, *viewdirs, *features, *features_jitter;
    int64_t n;
    float *color, *jac, *reg_sums;
    float *albedo, *roughness, *metalness, *spec_light, *diff_light, *spec_color, *diff_color;
};

__device__ __forceinline__ f3 cube_dir(int s, float x, float y) {
    switch (s) {
        case 0: return mk3(1.f, -y, -x);
        case 1: return mk3(-1.f, -y, x);
        case 2: return mk3(x, 1.f, y);
        case 3: return mk3(x, -1.f, -y);
        case 4: return mk3(x, -y, 1.f);
        default: return mk3(-x, -y, -1.f);
    }
}
__device__ __forceinline__ void dir_cube(f3 d, int& face, float& s, float& t) {
    float ax = fabsf(d.x), ay = fabsf(d.y), az = fabsf(d.z);
    float ma;
    if (ax >= ay && ax >= az) { face = d.x >= 0 ? 0 : 1; ma = ax; }
    else if (ay >= az) { face = d.y >= 0 ? 2 : 3; ma = ay; }
    else { face = d.z >= 0 ? 4 : 5; ma = az; }
    float sv = (face == 0) ? -d.z : (face == 1) ? d.z : (face == 5) ? -d.x : d.x;
    float tv = (face == 2) ? d.z : (face == 3) ? -d.z : -d.y;
    s = sv / ma; t = tv / ma;
}
// seamless texel fetch (edge texels come from the neighbouring face, corner texels are dropped)
__device__ __forceinline__ bool cube_texel(const float* cube, int res, int face, int ix, int iy, f3& val) {
    bool inx = ix >= 0 && ix < res, iny = iy >= 0 && iy < res;
    if (!(inx || iny)) { val = mk3(0, 0, 0); return false; }
    if (!(inx && iny)) {
        float s = ((float)ix + 0.5f) / (float)res * 2.0f - 1.0f, t = ((float)iy + 0.5f) / (float)res * 2.0f - 1.0f;
        f3 d = cube_dir(face, s, t);
        float s2, t2;
        dir_cube(d, face, s2, t2);
        ix = min(max((int)floorf((s2 + 1.0f) * 0.5f * (float)res), 0), res - 1);
        iy = min(max((int)floorf((t2 + 1.0f) * 0.5f * (float)res), 0), res - 1);
    }
    const float* p = cube + (((int64_t)face * res + iy) * res + ix) * 3;   // global (L1-cached) or shared memory
    val = mk3(p[0], p[1], p[2]);
    return true;
}
__device__ __forceinline__ f3 cube_linear(const float* cube, int res, f3 d) {
    int face; float s, t;
    dir_cube(d, face, s, t);
    float x = (s + 1.0f) * 0.5f * (float)res - 0.5f, y = (t + 1.0f) * 0.5f * (float)res - 0.5f;
    float x0f = floorf(x), y0f = floorf(y);
    float fx = x - x0f, fy = y - y0f;
    int x0 = (int)x0f, y0 = (int)y0f;
    f3 acc = mk3(0, 0, 0); float ws = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        int dx = k & 1, dy = k >> 1;
        float w = (dx ? fx : 1.0f - fx) * (dy ? fy : 1.0f - fy);
        f3 val;
        if (cube_texel(cube, res, face, x0 + dx, y0 + dy, val)) { acc = acc + val * w; ws += w; }
    }
    return acc * (1.0f / ws);
}

// HBM-bound kernel (SURVEY.md section 8d: 124 B read+written per covered pixel forward, 200 B with the backward):
//   * persistent CTAs (grid = a multiple of the SM count) walk chunks of 128 pixels;
//   * the chunk's G-buffer rows (normal, view direction: 3 floats; features, jittered features: 5 floats) are dense
//     arrays, so the CTA moves them as 16-byte vectors (float4) into shared memory -- fully coalesced whatever the row
//     length -- and the colour / Jacobian rows leave the same way;
//   * the diffuse irradiance cube (6 x 16 x 16 x 3 floats = 18 KB) is staged in shared memory once per CTA; the specular
//     mips and the 512 KB FG LUT stay L1 / L2-resident (texture-like gathers, excluded from the algorithmic bytes).
constexpr int SS_CHUNK = 128;
__device__ __forceinline__ void ss_stage_in(const float* __restrict__ g, float* s, int64_t row0, int rows, int per, int tid) {
    const float* base = g + row0 * per;
    const int total = rows * per;
    if ((reinterpret_cast<uintptr_t>(base) & 15) == 0) {
        const int nv = total >> 2;
        for (int i = tid; i < nv; i += SS_CHUNK) reinterpret_cast<float4*>(s)[i] = __ldg(reinterpret_cast<const float4*>(base) + i);
        for (int i = (nv << 2) + tid; i < total; i += SS_CHUNK) s[i] = __ldg(base + i);
    } else {
        for (int i = tid; i < total; i += SS_CHUNK) s[i] = __ldg(base + i);
    }
}
__device__ __forceinline__ void ss_stage_out(float* __restrict__ g, const float* s, int64_t row0, int rows, int per, int tid) {
    float* base = g + row0 * per;
    const int total = rows * per;
    if ((reinterpret_cast<uintptr_t>(base) & 15) == 0) {
        const int nv = total >> 2;
        for (int i = tid; i < nv; i += SS_CHUNK) reinterpret_cast<float4*>(base)[i] = reinterpret_cast<const float4*>(s)[i];
        for (int i = (nv << 2) + tid; i < total; i += SS_CHUNK) base[i] = s[i];
    } else {
        for (int i = tid; i < total; i += SS_CHUNK) base[i] = s[i];
    }
}

__global__ void __launch_bounds__(SS_CHUNK) shade_splitsum_kernel(SsParams P) {
    __shared__ float s_reg[2];
    __shared__ __align__(16) float s_n[SS_CHUNK * 3], s_v[SS_CHUNK * 3], s_f[SS_CHUNK * 5], s_fj[SS_CHUNK * 5];
    __shared__ __align__(16) float s_col[SS_CHUNK * 3], s_jac[SS_CHUNK * 9];
    extern __shared__ float s_dcube[];      // [6 * dres * dres * 3] when P.dcube_smem, else unused
    if (threadIdx.x < 2) s_reg[threadIdx.x] = 0.f;
    const float* dcube = P.dcube;
    if (P.dcube_smem) {
        const int nd = 6 * P.dres * P.dres * 3;
        for (int i = threadIdx.x; i < nd; i += SS_CHUNK) s_dcube[i] = __ldg(P.dcube + i);
        dcube = s_dcube;
    }
    __syncthreads();
    float reg_kd = 0.f, reg_ks = 0.f;
    const int64_t n_chunks = (P.n + SS_CHUNK - 1) / SS_CHUNK;
    for (int64_t chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
        const int64_t row0 = chunk * SS_CHUNK;
        const int rows = (int)((P.n - row0) < SS_CHUNK ? (P.n - row0) : SS_CHUNK);
        __syncthreads();                      // previous chunk's staged outputs have been written out
        ss_stage_in(P.normals, s_n, row0, rows, 3, threadIdx.x);
        ss_stage_in(P.viewdirs, s_v, row0, rows, 3, threadIdx.x);
        ss_stage_in(P.features, s_f, row0, rows, 5, threadIdx.x);
        ss_stage_in(P.features_jitter, s_fj, row0, rows, 5, threadIdx.x);
        __syncthreads();
        const int lp = threadIdx.x;
        const int64_t pix = row0 + lp;
        if (lp < rows) {
        f3 n = mk3(s_n[3 * lp], s_n[3 * lp + 1], s_n[3 * lp + 2]), v = mk3(s_v[3 * lp], s_v[3 * lp + 1], s_v[3 * lp + 2]);
        float m[5], mj[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) { m[k] = sigmoidf_(s_f[5 * lp + k]); mj[k] = sigmoidf_(s_fj[5 * lp + k]); }
        float k0 = fabsf(m[0] - mj[0]), k1 = fabsf(m[1] - mj[1]), k2 = fabsf(m[2] - mj[2]);
        reg_kd += ((k0 + k1 + k2) / 3.0f) * k2;
        reg_ks += fabsf(m[3] - mj[3]) * fabsf(m[4] - mj[4]);
        float alb[3] = {fminf(fmaxf(m[0], 0.f), 1.f), fminf(fmaxf(m[1], 0.f), 1.f), fminf(fmaxf(m[2], 0.f), 1.f)};
        float met = m[3] * (P.cfg.max_metallic - P.cfg.min_metallic) + P.cfg.min_metallic;
        float rough = m[4] * (P.cfg.max_roughness - P.cfg.min_roughness) + P.cfg.min_roughness;
        float ndv = dot3(n, v);
        f3 refl = (ndv * n) * 2.0f - v;
        // FG LUT, bilinear, clamp (:686-692); d fg / d rough kept for the Jacobian
        float fg0, fg1, dfg0, dfg1;
        {
            int R = P.lut_res;
            float x = fminf(fmaxf(ndv, 0.f), 1.f) * R - 0.5f, y = fminf(fmaxf(rough, 0.f), 1.f) * R - 0.5f;
            float x0f = floorf(x), y0f = floorf(y);
            float fx = x - x0f, fy = y - y0f;
            int x0 = min(max((int)x0f, 0), R - 1), x1 = min(max((int)x0f + 1, 0), R - 1);
            int y0 = min(max((int)y0f, 0), R - 1), y1 = min(max((int)y0f + 1, 0), R - 1);
            const float2* L = reinterpret_cast<const float2*>(P.lut);
            float2 a00 = __ldg(L + y0 * R + x0), a01 = __ldg(L + y0 * R + x1), a10 = __ldg(L + y1 * R + x0), a11 = __ldg(L + y1 * R + x1);
            float t0x = a00.x * (1 - fx) + a01.x * fx, t1x = a10.x * (1 - fx) + a11.x * fx;
            float t0y = a00.y * (1 - fx) + a01.y * fx, t1y = a10.y * (1 - fx) + a11.y * fx;
            fg0 = t0x * (1 - fy) + t1x * fy; fg1 = t0y * (1 - fy) + t1y * fy;
            bool rin = rough >= 0.f && rough <= 1.f;
            dfg0 = rin ? (t1x - t0x) * R : 0.f; dfg1 = rin ? (t1y - t0y) * R : 0.f;
        }
        f3 dl = cube_linear(dcube, P.dres, n);
        // envlight.get_mip + trilinear mip blend; d/d rough through the level
        float lvl, dlvl;
        {
            const float mn = 0.08f, mx = 0.5f; int nm = P.n_mips;
            if (rough < mx) { float rc = fminf(fmaxf(rough, mn), mx); lvl = (rc - mn) / (mx - mn) * (nm - 2); dlvl = (rough >= mn && rough <= mx) ? (nm - 2) / (mx - mn) : 0.f; }
            else { float rc = fminf(fmaxf(rough, mx), 1.0f); lvl = (rc - mx) / (1.0f - mx) + nm - 2; dlvl = (rough >= mx && rough <= 1.0f) ? 1.0f / (1.0f - mx) : 0.f; }
        }
        float lc = fminf(fmaxf(lvl, 0.f), (float)(P.n_mips - 1));
        int l0 = min((int)floorf(lc), P.n_mips - 1), l1 = min(l0 + 1, P.n_mips - 1);
        float fl = lc - (float)l0;
        f3 s0 = cube_linear(P.mips[l0], P.res0 >> l0, refl);
        f3 s1 = cube_linear(P.mips[l1], P.res0 >> l1, refl);
        f3 sl = s0 * (1.0f - fl) + s1 * fl;
        f3 dsl = (lvl >= 0.f && lvl <= (float)(P.n_mips - 1)) ? (s1 - s0) * dlvl : mk3(0, 0, 0);
        const float dlv[3] = {dl.x, dl.y, dl.z}, slv[3] = {sl.x, sl.y, sl.z}, dslv[3] = {dsl.x, dsl.y, dsl.z};
        float colv[3], sa[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float F0 = (1.0f - met) * 0.04f + met * alb[c];
            sa[c] = F0 * fg0 + fg1;
            float lin = alb[c] * dlv[c] + sa[c] * slv[c];
            float g = (lin >= 0.f && lin <= 1.f) ? 1.f : 0.f;
            colv[c] = fminf(fmaxf(lin, 0.f), 1.f);
            s_jac[9 * lp + 3 * c + 0] = g * (dlv[c] + met * fg0 * slv[c]);
            s_jac[9 * lp + 3 * c + 1] = g * ((alb[c] - 0.04f) * fg0 * slv[c]);
            s_jac[9 * lp + 3 * c + 2] = g * ((F0 * dfg0 + dfg1) * slv[c] + sa[c] * dslv[c]);
            s_col[3 * lp + c] = colv[c];
        }
        if (P.albedo) st3(P.albedo, pix, mk3(alb[0], alb[1], alb[2]));
        if (P.roughness) P.roughness[pix] = rough;
        if (P.metalness) P.metalness[pix] = met;
        if (P.spec_light) st3(P.spec_light, pix, mk3(lin2srgb_f(sl.x), lin2srgb_f(sl.y), lin2srgb_f(sl.z)));
        if (P.diff_light) st3(P.diff_light, pix, mk3(lin2srgb_f(dl.x), lin2srgb_f(dl.y), lin2srgb_f(dl.z)));
        if (P.spec_color) st3(P.spec_color, pix, mk3(lin2srgb_f(sa[0]), lin2srgb_f(sa[1]), lin2srgb_f(sa[2])));
        if (P.diff_color) st3(P.diff_color, pix, mk3(lin2srgb_f(alb[0]), lin2srgb_f(alb[1]), lin2srgb_f(alb[2])));
        }
        __syncthreads();
        ss_stage_out(P.color, s_col, row0, rows, 3, threadIdx.x);
        ss_stage_out(P.jac, s_jac, row0, rows, 9, threadIdx.x);
    }
    reg_kd = warp_sum(reg_kd); reg_ks = warp_sum(reg_ks);
    if ((threadIdx.x & 31) == 0) { atomicAdd(&s_reg[0], reg_kd); atomicAdd(&s_reg[1], reg_ks); }
    __syncthreads();
    if (threadIdx.x < 2 && P.reg_sums) atomicAdd(P.reg_sums + threadIdx.x, s_reg[threadIdx.x]);
}

// ------------------------------------------------------------------------------------------ backward
// dfeatures = sigmoid'(f) * [ J^T dcolor (through the range maps) + d reg / d m ],  dfeatures_jitter = sigmoid'(fj) * d reg / d mj
__global__ void __launch_bounds__(256) shade_bwd_kernel(dm_material_cfg cfg, const float* __restrict__ features,
                                                        const float* __restrict__ features_jitter,
                                                        const float* __restrict__ dcolor,
                                                        const float* __restrict__ jac, float dreg_kd, float dreg_ks,
                                                        int64_t n, float* __restrict__ df, float* __restrict__ dfj) {
    const int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= n) return;
    float m[5], mj[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) { m[k] = sigmoidf_(features[5 * pix + k]); mj[k] = sigmoidf_(features_jitter[5 * pix + k]); }
    float dm[5] = {0, 0, 0, 0, 0}, dmj[5] = {0, 0, 0, 0, 0};
    const float* J = jac + 9 * pix;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float g = dcolor[3 * pix + c];
        dm[c] += g * J[3 * c + 0];  // albedo clamp(0,1) of a sigmoid is the identity with unit slope
        dm[3] += g * J[3 * c + 1] * (cfg.max_metallic - cfg.min_metallic);
        dm[4] += g * J[3 * c + 2] * (cfg.max_roughness - cfg.min_roughness);
    }
    // smoothness regulariser: kd = |m-mj|[0:3], ks = |m-mj|[3:5]; sign(0) = 0 as in torch.abs backward
    {
        float d[5], sg[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) { float x = m[k] - mj[k]; d[k] = fabsf(x); sg[k] = (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f); }
        float luma = (d[0] + d[1] + d[2]) / 3.0f;
        float gk[5];
        gk[0] = dreg_kd * d[2] / 3.0f;
        gk[1] = dreg_kd * d[2] / 3.0f;
        gk[2] = dreg_kd * (d[2] / 3.0f + luma);
        gk[3] = dreg_ks * d[4];
        gk[4] = dreg_ks * d[3];
#pragma unroll
        for (int k = 0; k < 5; ++k) { dm[k] += gk[k] * sg[k]; dmj[k] -= gk[k] * sg[k]; }
    }
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        df[5 * pix + k] = dm[k] * m[k] * (1.0f - m[k]);
        dfj[5 * pix + k] = dmj[k] * mj[k] * (1.0f - mj[k]);
    }
}

__global__ void envmap_pack_kernel(const float* __restrict__ rgb, int64_t n, float4* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = make_float4(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2], 0.f);
}

}  // namespace

static int g_mc_frontier = 1;     // dm_tune "mc_frontier": 1 shared-origin frontier traversal | 0 root traversal

/* run-time switches: "mc_frontier" (MC shader traversal, 0 | 1), "pdl" (programmatic dependent launch of the dense kernels) */
extern "C" int dm_tune(const char* key, int value) {
    if (!key) return DM_EINVAL;
    if (!strcmp(key, "mc_frontier")) {
        if (value != 0 && value != 1) { dm_set_error("dm_tune mc_frontier: 0 or 1"); return DM_EINVAL; }
        g_mc_frontier = value;
    }
    else if (!strcmp(key, "pdl")) g_dm_pdl = value ? 1 : 0;
    else { dm_set_error("dm_tune: unknown key %s", key); return DM_EINVAL; }
    return DM_OK;
}

extern "C" int dm_shade_mc_fwd(const dm_material_cfg* cfg, const dm_bvh* bvh, const float* env_rgba, int envH, int envW,
                               const float* tab_d, const float* tab_s, const float* pts, const float* normals,
                               const float* viewdirs, const float* features, const float* features_jitter,
                               const float* rand_d, const float* rand_s, int64_t n, float* color, float* jac,
                               float* reg_sums, float* albedo, float* roughness, float* metalness, float* spec_light,
                               float* diff_light, float* spec_color, float* diff_color, uint32_t* hit_bits, void* stream) {
    if (n == 0) return DM_OK;
    DM_REQUIRE(cfg && bvh && env_rgba && tab_d && tab_s && pts && normals && viewdirs && features && features_jitter &&
                   rand_d && rand_s && color && jac, "null pointer");
    DM_REQUIRE(cfg->n_diffuse > 0 && cfg->n_specular > 0 && cfg->n_diffuse + cfg->n_specular <= 4096, "sample counts");
    McParams P;
    P.cfg = *cfg; P.bvh = BvhView{bvh->nodes, bvh->tris, bvh->ids, bvh->root};
    P.env = (const float4*)env_rgba; P.envH = envH; P.envW = envW; P.tab_d = tab_d; P.tab_s = tab_s;
    P.pts = pts; P.normals = normals; P.viewdirs = viewdirs; P.features = features; P.features_jitter = features_jitter;
    P.rand_d = rand_d; P.rand_s = rand_s; P.n = n; P.color = color; P.jac = jac; P.reg_sums = reg_sums;
    P.albedo = albedo; P.roughness = roughness; P.metalness = metalness; P.spec_light = spec_light;
    P.diff_light = diff_light; P.spec_color = spec_color; P.diff_color = diff_color; P.hit_bits = hit_bits;
    P.frontier = g_mc_frontier;
    // direction tables + one compacted sample-id list per warp
    const size_t smem = (size_t)(3 * cfg->n_diffuse + 2 * cfg->n_specular) * sizeof(float) +
                        (size_t)MC_WARPS * (cfg->n_diffuse + cfg->n_specular) * sizeof(uint16_t);
    static size_t smem_configured = 0;
    if (smem > smem_configured) {
        DM_CHECK_CUDA(cudaFuncSetAttribute(shade_mc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        smem_configured = smem;
    }
    shade_mc_kernel<<<(unsigned)dm_ceil_div(n, MC_WARPS), MC_WARPS * 32, smem, (cudaStream_t)stream>>>(P);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_shade_splitsum_fwd(const dm_material_cfg* cfg, const float* fg_lut, int lut_res,
                                     const float* diffuse_cube, int diff_res, const float* const* spec_mips_host,
                                     int n_mips, int spec_res0, const float* normals, const float* viewdirs,
                                     const float* features, const float* features_jitter, int64_t n, float* color,
                                     float* jac, float* reg_sums, float* albedo, float* roughness, float* metalness,
                                     float* spec_light, float* diff_light, float* spec_color, float* diff_color,
                                     void* stream) {
    if (n == 0) return DM_OK;
    DM_REQUIRE(cfg && fg_lut && diffuse_cube && spec_mips_host && normals && viewdirs && features && features_jitter &&
                   color && jac, "null pointer");
    DM_REQUIRE(n_mips >= 2 && n_mips <= 8, "2..8 specular mips");
    SsParams P;
    P.cfg = *cfg; P.lut = fg_lut; P.lut_res = lut_res; P.dcube = diffuse_cube; P.dres = diff_res;
    for (int i = 0; i < 8; ++i) P.mips[i] = i < n_mips ? spec_mips_host[i] : nullptr;
    P.n_mips = n_mips; P.res0 = spec_res0;
    P.normals = normals; P.viewdirs = viewdirs; P.features = features; P.features_jitter = features_jitter; P.n = n;
    P.color = color; P.jac = jac; P.reg_sums = reg_sums; P.albedo = albedo; P.roughness = roughness;
    P.metalness = metalness; P.spec_light = spec_light; P.diff_light = diff_light; P.spec_color = spec_color;
    P.diff_color = diff_color;
    // persistent CTAs: 8 per SM (128 threads, ~10 KB static + the staged diffuse cube), grid = a multiple of the SM count
    const size_t cube_bytes = (size_t)6 * diff_res * diff_res * 3 * sizeof(float);
    P.dcube_smem = cube_bytes <= 24 * 1024 ? 1 : 0;
    const size_t smem = P.dcube_smem ? cube_bytes : 0;
    const int64_t chunks = dm_ceil_div(n, SS_CHUNK);
    const int64_t grid = chunks < (int64_t)DM_NUM_SMS * 6 ? chunks : (int64_t)DM_NUM_SMS * 6;
    shade_splitsum_kernel<<<(unsigned)grid, SS_CHUNK, smem, (cudaStream_t)stream>>>(P);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_shade_bwd(const dm_material_cfg* cfg, const float* features, const float* features_jitter,
                            const float* dcolor, const float* jac, float dreg_kd, float dreg_ks, int64_t n,
                            float* dfeatures, float* dfeatures_jitter, void* stream) {
    if (n == 0) return DM_OK;
    DM_REQUIRE(cfg && features && features_jitter && dcolor && jac && dfeatures && dfeatures_jitter, "null pointer");
    shade_bwd_kernel<<<(unsigned)dm_ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(*cfg, features, features_jitter, dcolor,
                                                                                   jac, dreg_kd, dreg_ks, n, dfeatures,
                                                                                   dfeatures_jitter);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

extern "C" int dm_envmap_pack(const float* rgb, int64_t n_texels, float* rgba, void* stream) {
    if (n_texels == 0) return DM_OK;
    DM_REQUIRE(rgb && rgba, "null pointer");
    envmap_pack_kernel<<<(unsigned)dm_ceil_div(n_texels, 256), 256, 0, (cudaStream_t)stream>>>(rgb, n_texels, (float4*)rgba);
    DM_CHECK_LAUNCH();
    return DM_OK;
}
