// bvh.cu -- host-side binned-SAH BVH2 build, device upload, closest-hit trace and the
// G-buffer producer (replaces _raytracing + dr.rasterize/dr.interpolate; see bvh.cuh, dreammat_b200.h).
#include <algorithm>
#include <vector>
#include <cmath>
#include "bvh.cuh"

namespace {

constexpr int BVH_LEAF_MAX = 4;   // triangles per leaf: the leaf code stores cnt - 1 in 2 bits

struct Box {
    float lo[3], hi[3];
    void init() { for (int k = 0; k < 3; ++k) { lo[k] = 3e38f; hi[k] = -3e38f; } }
    void grow(const Box& b) { for (int k = 0; k < 3; ++k) { lo[k] = std::min(lo[k], b.lo[k]); hi[k] = std::max(hi[k], b.hi[k]); } }
    void grow(const float* p) { for (int k = 0; k < 3; ++k) { lo[k] = std::min(lo[k], p[k]); hi[k] = std::max(hi[k], p[k]); } }
    float area() const {
        float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        if (dx < 0 || dy < 0 || dz < 0) return 0.f;
        return 2.f * (dx * dy + dy * dz + dz * dx);
    }
};

struct Builder {
    const float* v; const int32_t* t; int64_t nt;
    std::vector<Box> tb; std::vector<float> cent; std::vector<int32_t> perm;
    std::vector<float4> nodes;  // 4 per node
    std::vector<int32_t> leaf_order;  // triangles in leaf order

    // returns child code: >=0 node index, <0 leaf code ~((first<<2)|(cnt-1)); fills `box`
    int32_t build(int32_t first, int32_t count, Box& box) {
        box.init();
        Box cb; cb.init();
        for (int32_t i = first; i < first + count; ++i) { box.grow(tb[perm[i]]); cb.grow(&cent[3 * (size_t)perm[i]]); }
        if (count <= BVH_LEAF_MAX) {
            int32_t lf = (int32_t)leaf_order.size();
            for (int32_t i = first; i < first + count; ++i) leaf_order.push_back(perm[i]);
            return ~((lf << 2) | (count - 1));
        }
        // binned SAH over the 3 axes
        const int NB = 16;
        float best_cost = 3e38f; int best_axis = -1, best_bin = -1;
        for (int ax = 0; ax < 3; ++ax) {
            float lo = cb.lo[ax], ext = cb.hi[ax] - lo;
            if (!(ext > 1e-12f)) continue;
            Box bb[NB]; int bc[NB];
            for (int b = 0; b < NB; ++b) { bb[b].init(); bc[b] = 0; }
            float sc = NB / ext;
            for (int32_t i = first; i < first + count; ++i) {
                int b = std::min(NB - 1, std::max(0, (int)((cent[3 * (size_t)perm[i] + ax] - lo) * sc)));
                bb[b].grow(tb[perm[i]]); bc[b]++;
            }
            float ra[NB]; int rc[NB]; Box acc; acc.init(); int c = 0;
            for (int b = NB - 1; b > 0; --b) { acc.grow(bb[b]); c += bc[b]; ra[b] = acc.area(); rc[b] = c; }
            acc.init(); c = 0;
            for (int b = 0; b < NB - 1; ++b) {
                acc.grow(bb[b]); c += bc[b];
                if (c == 0 || rc[b + 1] == 0) continue;
                float cost = acc.area() * c + ra[b + 1] * rc[b + 1];
                if (cost < best_cost) { best_cost = cost; best_axis = ax; best_bin = b; }
            }
        }
        int32_t mid;
        if (best_axis < 0) {
            mid = first + count / 2;  // degenerate: all centroids coincide
        } else {
            float lo = cb.lo[best_axis], sc = NB / (cb.hi[best_axis] - lo);
            int ax = best_axis, bbn = best_bin;
            auto it = std::partition(perm.begin() + first, perm.begin() + first + count, [&](int32_t f) {
                int b = std::min(NB - 1, std::max(0, (int)((cent[3 * (size_t)f + ax] - lo) * sc)));
                return b <= bbn;
            });
            mid = (int32_t)(it - perm.begin());
            if (mid == first || mid == first + count) mid = first + count / 2;
        }
        int32_t id = (int32_t)(nodes.size() / 4);
        nodes.resize(nodes.size() + 4);
        Box lb, rb;
        int32_t cl = build(first, mid - first, lb);
        int32_t cr = build(mid, first + count - mid, rb);
        const float W = 1e-6f;   // pre-widened slabs (see bvh.cuh)
        float4 n0 = make_float4(lb.lo[0] - W, lb.lo[1] - W, lb.lo[2] - W, lb.hi[0] + W);
        float4 n1 = make_float4(lb.hi[1] + W, lb.hi[2] + W, rb.lo[0] - W, rb.lo[1] - W);
        float4 n2 = make_float4(rb.lo[2] - W, rb.hi[0] + W, rb.hi[1] + W, rb.hi[2] + W);
        float4 n3; int32_t z = 0;
        memcpy(&n3.x, &cl, 4); memcpy(&n3.y, &cr, 4); memcpy(&n3.z, &z, 4); memcpy(&n3.w, &z, 4);
        nodes[4 * (size_t)id] = n0; nodes[4 * (size_t)id + 1] = n1; nodes[4 * (size_t)id + 2] = n2; nodes[4 * (size_t)id + 3] = n3;
        return id;
    }
};

}  // namespace

extern "C" int dm_bvh_build(const float* verts_host, int64_t n_verts, const int32_t* tris_host, int64_t n_tris,
                            dm_bvh** out) {
    DM_REQUIRE(verts_host && tris_host && out, "null pointer");
    DM_REQUIRE(n_tris > 0 && n_tris < (1 << 29), "triangle count");
    Builder b; b.v = verts_host; b.t = tris_host; b.nt = n_tris;
    b.tb.resize(n_tris); b.cent.resize(3 * n_tris); b.perm.resize(n_tris);
    for (int64_t f = 0; f < n_tris; ++f) {
        b.perm[f] = (int32_t)f; b.tb[f].init();
        for (int j = 0; j < 3; ++j) {
            int32_t vi = tris_host[3 * f + j];
            DM_REQUIRE(vi >= 0 && vi < n_verts, "triangle index out of range");
            b.tb[f].grow(verts_host + 3 * (size_t)vi);
        }
        for (int k = 0; k < 3; ++k) b.cent[3 * f + k] = 0.5f * (b.tb[f].lo[k] + b.tb[f].hi[k]);
    }
    b.nodes.reserve(4 * (size_t)n_tris);
    Box root;
    int32_t rc = b.build(0, (int32_t)n_tris, root);
    std::vector<float4> tr(3 * (size_t)n_tris);
    for (int64_t i = 0; i < n_tris; ++i) {
        int32_t f = b.leaf_order[i];
        const float* a = verts_host + 3 * (size_t)tris_host[3 * f];
        const float* bb = verts_host + 3 * (size_t)tris_host[3 * f + 1];
        const float* c = verts_host + 3 * (size_t)tris_host[3 * f + 2];
        float e1[3], e2[3];
        for (int k = 0; k < 3; ++k) { e1[k] = bb[k] - a[k]; e2[k] = c[k] - a[k]; }
        float nx = e1[1] * e2[2] - e1[2] * e2[1], ny = e1[2] * e2[0] - e1[0] * e2[2], nz = e1[0] * e2[1] - e1[1] * e2[0];
        tr[3 * i] = make_float4(a[0], a[1], a[2], e1[0]);
        tr[3 * i + 1] = make_float4(e1[1], e1[2], e2[0], e2[1]);
        tr[3 * i + 2] = make_float4(e2[2], nx, ny, nz);
    }
    dm_bvh* h = new dm_bvh();
    h->n_nodes = (int32_t)(b.nodes.size() / 4); h->n_tris = (int32_t)n_tris; h->root = rc;
    h->nodes = nullptr; h->tris = nullptr; h->ids = nullptr;
    size_t nb = std::max<size_t>(b.nodes.size(), 4) * sizeof(float4);
    cudaError_t e = cudaMalloc(&h->nodes, nb);
    if (e == cudaSuccess) e = cudaMalloc(&h->tris, tr.size() * sizeof(float4));
    if (e == cudaSuccess && !b.nodes.empty()) e = cudaMemcpy(h->nodes, b.nodes.data(), b.nodes.size() * sizeof(float4), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(h->tris, tr.data(), tr.size() * sizeof(float4), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMalloc(&h->ids, sizeof(int32_t) * (size_t)n_tris);
    if (e == cudaSuccess) e = cudaMemcpy(h->ids, b.leaf_order.data(), sizeof(int32_t) * (size_t)n_tris, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        dm_set_error("dm_bvh_build: %s", cudaGetErrorString(e));
        if (h->nodes) cudaFree(h->nodes);
        if (h->tris) cudaFree(h->tris);
        if (h->ids) cudaFree(h->ids);
        delete h;
        return (int)e;
    }
    *out = h;
    return DM_OK;
}

extern "C" void dm_bvh_free(dm_bvh* bvh) {
    if (!bvh) return;
    cudaFree(bvh->nodes); cudaFree(bvh->tris); cudaFree(bvh->ids);
    delete bvh;
}

extern "C" int64_t dm_bvh_num_nodes(const dm_bvh* bvh) { return bvh ? bvh->n_nodes : 0; }

__global__ void __launch_bounds__(128) bvh_trace_kernel(BvhView bv, const float* __restrict__ ro,
                                                        const float* __restrict__ rd, int64_t n,
                                                        float* __restrict__ t_out, int32_t* __restrict__ tri_out,
                                                        float* __restrict__ uv_out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    f3 o = ld3(ro, i), d = ld3(rd, i);
    float t, u, v; int id;
    bvh_trace<false>(bv, o, d, t, id, u, v);
    t_out[i] = t; tri_out[i] = id;
    if (uv_out) { uv_out[2 * i] = u; uv_out[2 * i + 1] = v; }
}

extern "C" int dm_bvh_trace(const dm_bvh* bvh, const float* rays_o, const float* rays_d, int64_t n, float* t,
                            int32_t* tri, float* uv, void* stream) {
    if (n == 0) return DM_OK;
    DM_REQUIRE(bvh && rays_o && rays_d && t && tri, "null pointer");
    BvhView bv{bvh->nodes, bvh->tris, bvh->ids, bvh->root};
    bvh_trace_kernel<<<(unsigned)dm_ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(bv, rays_o, rays_d, n, t, tri, uv);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

// ---------------------------------------------------------------------------------------------
// G-buffer: one thread per pixel.  raytracing_renderer.py:122-159 (+ :326-331 view normals).
__global__ void __launch_bounds__(128) gbuffer_kernel(BvhView bv, const float* __restrict__ v_pos,
                                                      const float* __restrict__ v_nrm,
                                                      const int32_t* __restrict__ tris,
                                                      const float* __restrict__ rays_o,
                                                      const float* __restrict__ rays_d,
                                                      const float* __restrict__ mvp, const float* __restrict__ w2c,
                                                      int B, int64_t HW, float* __restrict__ rast,
                                                      float* __restrict__ gb_pos, float* __restrict__ gb_nrm,
                                                      uint8_t* __restrict__ mask, float* __restrict__ comp_normal) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)B * HW) return;
    int b = (int)(i / HW);
    f3 o = ld3(rays_o, i), d = ld3(rays_d, i);
    float t, u, v; int id;
    bool hit = bvh_trace<false>(bv, o, d, t, id, u, v);
    f3 P = mk3(0, 0, 0), N = mk3(0, 0, 0);
    float4 r = make_float4(0, 0, 0, 0);
    f3 cn = mk3(0.5f, 0.5f, 1.0f);
    if (hit) {
        int i0 = tris[3 * (int64_t)id], i1 = tris[3 * (int64_t)id + 1], i2 = tris[3 * (int64_t)id + 2];
        float b0 = 1.0f - u - v;
        P = ld3(v_pos, i0) * b0 + ld3(v_pos, i1) * u + ld3(v_pos, i2) * v;
        N = normalize3(ld3(v_nrm, i0) * b0 + ld3(v_nrm, i1) * u + ld3(v_nrm, i2) * v);
        const float* M = mvp + 16 * b;
        float cz = M[8] * P.x + M[9] * P.y + M[10] * P.z + M[11];
        float cw = M[12] * P.x + M[13] * P.y + M[14] * P.z + M[15];
        r = make_float4(b0, u, cz / cw, (float)(id + 1));
        const float* Wm = w2c + 16 * b;
        f3 nv = normalize3(mk3(Wm[0] * N.x + Wm[1] * N.y + Wm[2] * N.z, Wm[4] * N.x + Wm[5] * N.y + Wm[6] * N.z,
                               Wm[8] * N.x + Wm[9] * N.y + Wm[10] * N.z));
        cn = mk3(1.0f - 0.5f * (nv.x + 1.0f), 0.5f * (nv.y + 1.0f), 0.5f * (nv.z + 1.0f));
    }
    if (rast) reinterpret_cast<float4*>(rast)[i] = r;
    if (gb_pos) st3(gb_pos, i, P);
    if (gb_nrm) st3(gb_nrm, i, N);
    if (mask) mask[i] = hit ? 1 : 0;
    if (comp_normal) st3(comp_normal, i, cn);
}

extern "C" int dm_raster_gbuffer(const dm_bvh* bvh, const float* v_pos, const float* v_nrm, const int32_t* tris,
                                 const float* rays_o, const float* rays_d, const float* mvp, const float* w2c, int B,
                                 int H, int W, float* rast, float* gb_pos, float* gb_nrm, uint8_t* mask,
                                 float* comp_normal, void* stream) {
    if ((int64_t)B * H * W == 0) return DM_OK;
    DM_REQUIRE(bvh && v_pos && v_nrm && tris && rays_o && rays_d && mvp && w2c, "null pointer");
    int64_t n = (int64_t)B * H * W;
    BvhView bv{bvh->nodes, bvh->tris, bvh->ids, bvh->root};
    gbuffer_kernel<<<(unsigned)dm_ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(
        bv, v_pos, v_nrm, tris, rays_o, rays_d, mvp, w2c, B, (int64_t)H * W, rast, gb_pos, gb_nrm, mask, comp_normal);
    DM_CHECK_LAUNCH();
    return DM_OK;
}
