// bvh.cuh -- device-side BVH2 traversal (closest-hit and any-hit) over the layout built in bvh.cu.
//
// Replaces the `_raytracing` extension the reference calls at
// models/renderers/raytracing_renderer.py:31,61 (semantics: closest hit with t initialised to
// 10; `depth >= 10` is a miss, :322).  Triangle test = the determinant form the published
// instant-ngp / ashawkey-raytracing BVH uses (no culling, u,v in [0,1], u+v<=1, t>=0).
//
// Node = 4 x float4 (64 B): both child boxes live in the parent, so one node fetch (two 32 B
// sectors) decides both children; boxes are widened by 1e-6 at build time so that a hit exactly on a
// box face is never culled.  Leaves hold <= 4 triangles stored as 3 x float4 = (a, e1 = b-a, e2 = c-a,
// n = e1 x e2), precomputed on the host in fp32; original triangle ids live in a side array.
#pragma once
#include "common.cuh"

#define DM_RT_MAX_DIST 10.0f
#define DM_BVH_STACK 48

struct dm_bvh {
    float4* nodes;   // [n_nodes*4]
    float4* tris;    // [n_tris*3]   leaf order
    int32_t* ids;    // [n_tris]     leaf order -> original triangle id
    int32_t n_nodes;
    int32_t n_tris;
    int32_t root;    // child code of the root (>=0 node, <0 leaf)
};

struct BvhView {
    const float4* __restrict__ nodes;
    const float4* __restrict__ tris;
    const int32_t* __restrict__ ids;
    int32_t root;
};

// same determinant-form test with the edge vectors / normal precomputed; the reciprocal is the fast MUFU one
// (<= 2 ulp), which can only move rays that graze an edge within rounding
__device__ __forceinline__ float tri_hit_pre(f3 o, f3 d, float4 A, float4 B, float4 C, float& u, float& v) {
    f3 r = mk3(o.x - A.x, o.y - A.y, o.z - A.z);
    f3 e1 = mk3(A.w, B.x, B.y), e2 = mk3(B.z, B.w, C.x), n = mk3(C.y, C.z, C.w);
    f3 q = cross3(r, d);
    float inv = __fdividef(1.0f, dot3(d, n));
    u = inv * -dot3(q, e2);
    v = inv * dot3(q, e1);
    float t = inv * -dot3(n, r);
    if (!(u >= 0.0f) || u > 1.0f || !(v >= 0.0f) || (u + v) > 1.0f || !(t >= 0.0f)) return 3.0e38f;
    return t;
}

// slab test against a pre-widened box; oi = o * inv
__device__ __forceinline__ bool slab2(float lox, float loy, float loz, float hix, float hiy, float hiz, f3 inv, f3 oi,
                                      float tmax, float& tn) {
    float ax = fmaf(lox, inv.x, -oi.x), bx = fmaf(hix, inv.x, -oi.x);
    float ay = fmaf(loy, inv.y, -oi.y), by = fmaf(hiy, inv.y, -oi.y);
    float az = fmaf(loz, inv.z, -oi.z), bz = fmaf(hiz, inv.z, -oi.z);
    float t0 = fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fmaxf(fminf(az, bz), 0.0f));
    float t1 = fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fminf(fmaxf(az, bz), tmax));
    tn = t0;
    return t0 <= t1;
}

// ANY=true : returns as soon as some triangle is hit with t < tmax (occlusion rays)
// ANY=false: closest hit; ties go to the lowest original triangle id (matches the oracle's scan order)
template <bool ANY>
__device__ __forceinline__ bool bvh_trace(const BvhView& bv, f3 o, f3 d, float& best_t, int& best_id, float& bu,
                                          float& bvv) {
    f3 inv = mk3(1.0f / d.x, 1.0f / d.y, 1.0f / d.z);
    f3 oi = mk3(o.x * inv.x, o.y * inv.y, o.z * inv.z);
    int stack[DM_BVH_STACK];
    int sp = 0;
    int cur = bv.root;
    best_t = DM_RT_MAX_DIST;
    best_id = -1;
    bu = bvv = 0.0f;
    bool alive = true;
    // "while-while" traversal: every lane first descends through internal nodes until it holds a leaf (or has
    // nothing left); the warp reconverges there, so the expensive triangle tests run with all leaf-holding lanes
    // active instead of the few an interleaved node/leaf loop leaves.
    while (alive) {
        while (alive && cur >= 0) {
            const float4* n = bv.nodes + (int64_t)cur * 4;
            float4 n0 = __ldg(n), n1 = __ldg(n + 1), n2 = __ldg(n + 2), n3 = __ldg(n + 3);
            float tl, tr;
            bool hl = slab2(n0.x, n0.y, n0.z, n0.w, n1.x, n1.y, inv, oi, best_t, tl);
            bool hr = slab2(n1.z, n1.w, n2.x, n2.y, n2.z, n2.w, inv, oi, best_t, tr);
            int cl = __float_as_int(n3.x), cr = __float_as_int(n3.y);
            if (hl && hr) {
                bool lfirst = tl <= tr;      // near child first
                if (sp < DM_BVH_STACK) stack[sp++] = lfirst ? cr : cl;
                cur = lfirst ? cl : cr;
            } else if (hl) cur = cl;
            else if (hr) cur = cr;
            else if (sp == 0) alive = false;
            else cur = stack[--sp];
        }
        if (!alive) break;
        {
            int code = ~cur;
            int first = code >> 2, cnt = (code & 3) + 1;
            for (int k = 0; k < cnt; ++k) {
                const float4* tp = bv.tris + (int64_t)(first + k) * 3;
                float4 A = __ldg(tp), B = __ldg(tp + 1), C = __ldg(tp + 2);
                float u, v;
                float t = tri_hit_pre(o, d, A, B, C, u, v);
                if (ANY) {
                    if (t < best_t) { best_t = t; best_id = 0; return true; }
                } else {
                    int id = __ldg(bv.ids + first + k);
                    if (t < best_t || (t == best_t && best_id >= 0 && id < best_id)) {
                        best_t = t; best_id = id; bu = u; bvv = v;
                    }
                }
            }
        }
        if (sp == 0) break;
        cur = stack[--sp];
    }
    return best_id >= 0;
}
