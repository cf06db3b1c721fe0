// envlight.cu -- device-side build of the split-sum environment lights (row a5 / N4 of SURVEY.md section 8).
//
// The reference builds one `envlight.EnvLight(path, scale)` per environment map at start-up
// (models/materials/dreammat_material.py:379-386; ashawkey/envlight, an un-vendored dependency that wraps
// nvdiffrec's renderutils): lat-long HDR -> cube map (128^2 per face) -> 2x2-average mip chain down to 16^2 ->
// GGX-prefiltered specular mips (roughness 0.08 .. 0.5 linearly over the chain, 1.0 for the last) and a
// cosine-convolved diffuse cube at 16^2.  `shade_splitsum` (:679-711) then needs only three texture lookups per pixel.
// Here the same construction runs as four small kernels (fp32, brute-force texel-pair sums: 6*128^2 squared is 9.7e9
// pairs, tens of milliseconds on the GPU); dreammat_b200/envlight.py drives them and caches the result on disk.
#include "common.cuh"

namespace {

constexpr float PI_F = 3.14159265358979323846f;

__device__ __forceinline__ f3 cube_dir_e(int s, float x, float y) {
    switch (s) {
        case 0: return mk3(1.f, -y, -x);
        case 1: return mk3(-1.f, -y, x);
        case 2: return mk3(x, 1.f, y);
        case 3: return mk3(x, -1.f, -y);
        case 4: return mk3(x, -y, 1.f);
        default: return mk3(-x, -y, -1.f);
    }
}

// latlong_to_cubemap: texel centres at linspace(-1 + 1/res, 1 - 1/res), bilinear lookup with wrap in both axes
__global__ void __launch_bounds__(256) latlong_to_cube_kernel(const float* __restrict__ ll, int H, int W, float scale, int res,
                                                              float* __restrict__ cube) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 6 * res * res) return;
    const int s = i / (res * res), r = i - s * res * res, iy = r / res, ix = r - iy * res;
    const float step = res > 1 ? (2.0f - 2.0f / res) / (float)(res - 1) : 0.f;
    const float gx = -1.0f + 1.0f / res + step * ix, gy = -1.0f + 1.0f / res + step * iy;
    const f3 v = normalize3(cube_dir_e(s, gx, gy));
    const float tu = atan2f(v.x, -v.z) / (2.0f * PI_F) + 0.5f;
    const float tv = acosf(fminf(fmaxf(v.y, -1.0f), 1.0f)) / PI_F;
    const float x = tu * W - 0.5f, y = tv * H - 0.5f;
    const float x0f = floorf(x), y0f = floorf(y);
    const float fx = x - x0f, fy = y - y0f;
    int x0 = (int)x0f, y0 = (int)y0f;
    int x1 = x0 + 1, y1 = y0 + 1;
    x0 = ((x0 % W) + W) % W; x1 = ((x1 % W) + W) % W; y0 = ((y0 % H) + H) % H; y1 = ((y1 % H) + H) % H;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float a = ll[((int64_t)y0 * W + x0) * 3 + c], b = ll[((int64_t)y0 * W + x1) * 3 + c];
        const float d = ll[((int64_t)y1 * W + x0) * 3 + c], e = ll[((int64_t)y1 * W + x1) * 3 + c];
        cube[(int64_t)i * 3 + c] = scale * (a * (1 - fx) * (1 - fy) + b * fx * (1 - fy) + d * (1 - fx) * fy + e * fx * fy);
    }
}

// F.avg_pool2d(., 2) per face
__global__ void __launch_bounds__(256) cube_downsample_kernel(const float* __restrict__ in, int res_in, float* __restrict__ out) {
    const int ro = res_in / 2;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 6 * ro * ro * 3) return;
    const int c = i % 3, t = i / 3, s = t / (ro * ro), r = t - s * ro * ro, y = r / ro, x = r - y * ro;
    const float* p = in + ((int64_t)s * res_in * res_in) * 3 + c;
    out[i] = 0.25f * (p[((2 * y) * res_in + 2 * x) * 3] + p[((2 * y) * res_in + 2 * x + 1) * 3] +
                      p[((2 * y + 1) * res_in + 2 * x) * 3] + p[((2 * y + 1) * res_in + 2 * x + 1) * 3]);
}

// direction of texel centre (i + 0.5) / res * 2 - 1 and its solid angle (difference of atan2(xy, sqrt(x^2+y^2+1)) corners)
__device__ __forceinline__ float corner_area(float x, float y) { return atan2f(x * y, sqrtf(x * x + y * y + 1.0f)); }
__device__ __forceinline__ void texel_dir_area(int res, int idx, f3& d, float& sa) {
    const int s = idx / (res * res), r = idx - s * res * res, iy = r / res, ix = r - iy * res;
    const float gx = ((float)ix + 0.5f) / res * 2.0f - 1.0f, gy = ((float)iy + 0.5f) / res * 2.0f - 1.0f;
    d = normalize3(cube_dir_e(s, gx, gy));
    const float h = 1.0f / res;
    sa = corner_area(gx - h, gy - h) - corner_area(gx - h, gy + h) - corner_area(gx + h, gy - h) + corner_area(gx + h, gy + h);
}

// mode 0 diffuse: w = clamp(N.L, 0, 0.999) * sa / 3.141592, out = sum w L
// mode 1 specular: w = max(N.L, 0) * D_ggx(a2, N.H) * sa / 4 over texels with N.L >= cos_cutoff, out = sum w L / sum w
// One block per output texel, threads stride over the input texels (direction + area recomputed: cheaper than a table).
__global__ void __launch_bounds__(256) cube_filter_kernel(const float* __restrict__ cube, int res, int mode, float a2, float cos_cutoff,
                                                          float* __restrict__ out) {
    __shared__ float red[4][8];
    const int o = blockIdx.x;
    f3 N; float sa_o;
    texel_dir_area(res, o, N, sa_o);
    const int n_in = 6 * res * res;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int j = threadIdx.x; j < n_in; j += blockDim.x) {
        f3 L; float sa;
        texel_dir_area(res, j, L, sa);
        const float ldn = dot3(N, L);
        float w;
        if (mode == 0) {
            w = fminf(fmaxf(ldn, 0.0f), 0.999f) * sa / 3.141592f;
        } else {
            if (ldn < cos_cutoff) continue;
            const f3 Hh = normalize3(N + L);
            const float noh = fmaxf(dot3(Hh, N), 0.0f);
            const float dd = (noh * a2 - noh) * noh + 1.0f;
            w = fmaxf(ldn, 0.0f) * (a2 / (dd * dd * PI_F)) * sa * 0.25f;
        }
        acc[0] += w * cube[(int64_t)j * 3]; acc[1] += w * cube[(int64_t)j * 3 + 1]; acc[2] += w * cube[(int64_t)j * 3 + 2];
        acc[3] += w;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float v = warp_sum(acc[k]);
        if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = v;
    }
    __syncthreads();
    if (threadIdx.x < 4) {
        float v = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v += red[threadIdx.x][w];
        red[threadIdx.x][0] = v;
    }
    __syncthreads();
    if (threadIdx.x < 3) out[(int64_t)o * 3 + threadIdx.x] = mode == 0 ? red[threadIdx.x][0] : red[threadIdx.x][0] / red[3][0];
}

}  // namespace

// lat-long [H,W,3] (* scale) -> cube [6,res,res,3]   (envlight utils.latlong_to_cubemap; dreammat_material.py:383)
extern "C" int dm_envlight_latlong_to_cube(const float* latlong, int H, int W, float scale, int res, float* cube, void* stream) {
    DM_REQUIRE(latlong && cube && H > 0 && W > 0 && res > 0, "bad args");
    latlong_to_cube_kernel<<<(unsigned)dm_ceil_div(6 * res * res, 256), 256, 0, (cudaStream_t)stream>>>(latlong, H, W, scale, res, cube);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

// [6,res,res,3] -> [6,res/2,res/2,3], 2x2 average
extern "C" int dm_envlight_downsample(const float* cube, int res, float* out, void* stream) {
    DM_REQUIRE(cube && out && res >= 2 && res % 2 == 0, "bad args");
    cube_downsample_kernel<<<(unsigned)dm_ceil_div(6 * (res / 2) * (res / 2) * 3, 256), 256, 0, (cudaStream_t)stream>>>(cube, res, out);
    DM_CHECK_LAUNCH();
    return DM_OK;
}

// diffuse (mode 0) or GGX-prefiltered specular (mode 1, alpha^2 = roughness^4, N.L >= cos_cutoff) convolution at equal resolution
extern "C" int dm_envlight_filter(const float* cube, int res, int mode, float roughness, float cos_cutoff, float* out, void* stream) {
    DM_REQUIRE(cube && out && res > 0 && (mode == 0 || mode == 1), "bad args");
    const float a = roughness * roughness;
    cube_filter_kernel<<<(unsigned)(6 * res * res), 256, 0, (cudaStream_t)stream>>>(cube, res, mode, a * a, cos_cutoff, out);
    DM_CHECK_LAUNCH();
    return DM_OK;
}
