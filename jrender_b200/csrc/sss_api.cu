// sss_api.cu -- texture-space subsurface scattering (jrender/renderer/lighting/lighting.py:86-156, SSS).
//
//   b200r_sss_stretch        <-  computeStretchMap (renderer/utils/ToStretchMap.py:5-13) of `7 * Worldcoord_Map` and the
//                                two clamps to [0, 1] (lighting.py:109-111)
//   b200r_sss_blur_pyramid   <-  the per-channel loop of lighting.py:133-150: three levels of gaussian_blur
//                                (renderer/utils/gaussian_blur.py:4-21, kernels gaussain_blur_{x,y}_Kernel :33-164) on the
//                                stretch maps and the irradiance, the weighted sum of the levels, `* irradiance`,
//                                `+ specular` and the vertical flip
//
// Maps are float32 [H, W] planes, row 0 = the top row of the SoftRas image they were rasterized into; the multi-channel
// inputs are [3, H, W] planar (the first three planes of the rasterizer's [4, H, W] soft_colors).
//
// The reference blurs each colour channel separately and recomputes the two stretch chains for each of them.  The chains
// do not depend on the channel, so here they are computed once, and one launch per pass and level does everything that
// pass needs: the x pass of level i blurs stretchU_{i-1} into stretchU_i at its pixel and uses that value at once as the
// modulation of the three irradiance channels' x blurs; the y pass does the same with stretchV and also adds the level
// into the weighted sum.  The last y pass multiplies by the unblurred irradiance, adds the specular map and writes the
// row flipped, in [H, W, 3], ready for the bake.  Three levels are six launches.
//
// Taps are read through the read-only data cache, not staged in shared memory: a tap's position depends on the centre
// pixel's own stretch value (and can extrapolate past it, see sss_blur_1d), so a tile's halo has no fixed bound, while
// neighbouring pixels' taps fall on the same few cache lines.  DESIGN.md section 11 gives the bytes each pass moves.
//
// Arithmetic is the reference kernels' float32 expressions unfused (-fmad=false), in their order; oracle/sss.py restates
// them in numpy and the two agree bit for bit.
#include <math.h>

#include "../../include/b200raster.h"
#include "api_util.cuh"
#include "sss_common.cuh"

namespace {

using namespace b200r_sss;

// One blurred value of gaussain_blur_{x,y}_Kernel (gaussian_blur.py:43-97, 109-164) for a single-channel map: `p` points
// at the line through the pixel (its row for x, its column for y, `stride` apart), `c` is the pixel's index on that line
// and `bound` the last index the reference clamps to (w - 1 in both kernels: the y kernel clamps rows against the width).
// The quirks are the reference's: int() truncates toward zero, so a tap in (-1, 0) gets x1 = 0, x2 = 1 and extrapolates;
// a tap wholly past an edge has x1 == x2 and contributes (x - c) v + (c - x) v = 0; a neighbour <= 1e-6 (compared in
// double) is replaced by the centre value; a centre value <= 0 gives 0.  The reference's centre test reads channel `l`
// of the pixel with `l` uninitialised; every SSS map has one channel, and the reference build reads channel 0.
__device__ __forceinline__ float sss_blur_1d(const float* __restrict__ p, int stride, int c, int bound, float mod,
                                             const SssPass& P) {
    const float centre = __ldg(p + (size_t)c * stride);
    if (!(centre > 0.f)) return 0.f;
    const float step = P.width * mod;
    float x = (float)c - step * (float)(kTaps - 1) / 2.f;
    float v = 0.f;
#pragma unroll
    for (int k = 0; k < kTaps; k++) {
        int x1 = (int)x;
        int x2 = (int)x + 1;
        x1 = x1 < 0 ? 0 : (x1 > bound ? bound : x1);
        x2 = x2 < 0 ? 0 : (x2 > bound ? bound : x2);
        float v1 = __ldg(p + (size_t)x1 * stride);
        v1 = (double)v1 > 1e-6 ? v1 : centre;
        float v2 = __ldg(p + (size_t)x2 * stride);
        v2 = (double)v2 > 1e-6 ? v2 : centre;
        const float interpolation = (x - (float)x1) * v2 + ((float)x2 - x) * v1;
        v = v + interpolation * P.taps[k];
        x = x + step;
    }
    return v;
}

// stretchU / stretchV of 7 * world (ToStretchMap.py:8-12, replicate padding of the last column / row), clamped to [0, 1]
// the way jt.clamp / np.clip do (NaN passes through).
__global__ void __launch_bounds__(256)
k_sss_stretch(const float* __restrict__ world, float* __restrict__ su, float* __restrict__ sv, int H, int W) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    const size_t hw = (size_t)H * W, id = (size_t)y * W + x;
    const size_t right = (size_t)y * W + (x + 1 < W ? x + 1 : x), down = (size_t)(y + 1 < H ? y + 1 : y) * W + x;
    float du = 0.f, dv = 0.f;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float* m = world + c * hw;
        const float a = __ldg(m + id) * 7.f;
        const float b = a - __ldg(m + right) * 7.f;
        const float d = a - __ldg(m + down) * 7.f;
        du = c == 0 ? b * b : du + b * b;
        dv = c == 0 ? d * d : dv + d * d;
    }
    float u = 1.f / sqrtf(du), v = 1.f / sqrtf(dv);
    u = u < 0.f ? 0.f : (u > 1.f ? 1.f : u);
    v = v < 0.f ? 0.f : (v > 1.f ? 1.f : v);
    su[id] = u;
    sv[id] = v;
}

// x pass of one level: stretchU_i = blur_x(stretchU_{i-1}, mod = stretchU_{i-1}) at the pixel, then
// irr_c = blur_x(irr_c, mod = stretchU_i) for the three channels (lighting.py:139-140).
__global__ void __launch_bounds__(kBlockX * kBlockY) k_sss_blur_x(const SssPass P) {
    const int x = blockIdx.x * kBlockX + threadIdx.x, y = blockIdx.y * kBlockY + threadIdx.y;
    if (x >= P.W || y >= P.H) return;
    const size_t hw = (size_t)P.H * P.W, row = (size_t)y * P.W, id = row + x;
    const float mod = __ldg(P.s_in + id);
    const float s = sss_blur_1d(P.s_in + row, 1, x, P.W - 1, mod, P);
    if (P.s_out) P.s_out[id] = s;
#pragma unroll
    for (int c = 0; c < 3; c++) P.irr_out[c * hw + id] = sss_blur_1d(P.irr_in + c * hw + row, 1, x, P.W - 1, s, P);
}

// y pass of one level: stretchV_i = blur_y(stretchV_{i-1}, mod = stretchV_{i-1}), irr_c = blur_y(irr_c, mod =
// stretchV_i) (lighting.py:141-142), then final_c += w_c,i * irr_c (:144-145, final starts at 0).  The last level goes on
// with final *= irradiance, final += specular (:147-148) and writes row H - 1 - y (:150) of out [H, W, 3].
__global__ void __launch_bounds__(kBlockX * kBlockY) k_sss_blur_y(const SssPass P) {
    const int x = blockIdx.x * kBlockX + threadIdx.x, y = blockIdx.y * kBlockY + threadIdx.y;
    if (x >= P.W || y >= P.H) return;
    const size_t hw = (size_t)P.H * P.W, id = (size_t)y * P.W + x;
    const float mod = __ldg(P.s_in + id);
    const float s = sss_blur_1d(P.s_in + x, P.W, y, P.W - 1, mod, P);
    if (P.s_out) P.s_out[id] = s;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float b = sss_blur_1d(P.irr_in + c * hw + x, P.W, y, P.W - 1, s, P);
        if (P.irr_out) P.irr_out[c * hw + id] = b;
        float f = P.first ? 0.f + P.weight[c] * b : P.acc[c * hw + id] + P.weight[c] * b;
        if (P.last) {
            f = f * __ldg(P.irr0 + c * hw + id);
            f = f + __ldg(P.spec + c * hw + id);
            P.out[((size_t)(P.H - 1 - y) * P.W + x) * 3 + c] = f;
        } else {
            P.acc[c * hw + id] = f;
        }
    }
}

// workspace: stretchU and stretchV ping-pong planes (2 + 2), the irradiance after the x pass and after the y pass (3 + 3),
// the running weighted sum (3)
constexpr int kPlanes = 13;

}  // namespace

void b200r_sss::forward_kernels(PassKernel* x_pass, PassKernel* y_pass) {
    *x_pass = k_sss_blur_x;
    *y_pass = k_sss_blur_y;
}

extern "C" size_t b200r_sss_workspace_bytes(int height, int width) {
    if (height <= 0 || width <= 0) return 0;
    return (size_t)kPlanes * height * width * sizeof(float);
}

extern "C" int b200r_sss_stretch(const float* world_map, float* stretch_u, float* stretch_v, int height, int width,
                                 void* stream) {
    if (!world_map || !stretch_u || !stretch_v) return b200r_fail(B200R_EINVAL, "b200r_sss_stretch: NULL pointer argument");
    if (height <= 0 || width <= 0 || height > 65535) return b200r_fail(B200R_EINVAL, "b200r_sss_stretch: map size %d x %d", height, width);
    return b200r_launch("k_sss_stretch", B200R_K_SSS, k_sss_stretch, dim3((width + 255) / 256, height), dim3(256), 0,
                        (cudaStream_t)stream, world_map, stretch_u, stretch_v, height, width);
}

extern "C" int b200r_sss_blur_pyramid(const float* stretch_u, const float* stretch_v, const float* irradiance_map,
                                      const float* specular_map, float* out_map, void* workspace, size_t workspace_bytes,
                                      const float* taps, const float* tap_widths, const float* weights, int num_levels,
                                      int height, int width, void* stream) {
    if (!stretch_u || !stretch_v || !irradiance_map || !specular_map || !out_map || !workspace || !taps || !tap_widths || !weights)
        return b200r_fail(B200R_EINVAL, "b200r_sss_blur_pyramid: NULL pointer argument");
    if (height <= 0 || width <= 0 || height != width || height > 65535 * kBlockY)
        return b200r_fail(B200R_EINVAL, "b200r_sss_blur_pyramid: map size %d x %d (the maps must be square)", height, width);
    if (num_levels < 1 || num_levels > kMaxLevels)
        return b200r_fail(B200R_EINVAL, "b200r_sss_blur_pyramid: num_levels %d outside [1, %d]", num_levels, kMaxLevels);
    if (workspace_bytes < b200r_sss_workspace_bytes(height, width))
        return b200r_fail(B200R_EWORKSPACE, "b200r_sss_blur_pyramid: workspace of %zu bytes, %zu needed", workspace_bytes,
                          b200r_sss_workspace_bytes(height, width));
    const size_t hw = (size_t)height * width;   // the kernels address channel c of a group at c * H * W
    float* ws = (float*)workspace;
    float* su[2] = {ws, ws + hw};
    float* sv[2] = {ws + 2 * hw, ws + 3 * hw};
    float* irr_x = ws + 4 * hw;
    float* irr_y = ws + 7 * hw;
    float* acc = ws + 10 * hw;
    const dim3 grid((width + kBlockX - 1) / kBlockX, (height + kBlockY - 1) / kBlockY), block(kBlockX, kBlockY);
    cudaStream_t st = (cudaStream_t)stream;
    const float* s_u = stretch_u;
    const float* s_v = stretch_v;
    const float* irr = irradiance_map;
    for (int i = 0; i < num_levels; i++) {
        const bool last = i == num_levels - 1;
        SssPass P = {};
        for (int k = 0; k < kTaps; k++) P.taps[k] = taps[i * kTaps + k];
        P.width = tap_widths[i];
        P.H = height;
        P.W = width;
        P.first = i == 0;
        P.last = last;
        P.s_in = s_u;
        P.s_out = last ? nullptr : su[i & 1];
        P.irr_in = irr;
        P.irr_out = irr_x;
        int rc = b200r_launch("k_sss_blur_x", B200R_K_SSS, k_sss_blur_x, grid, block, 0, st, P);
        if (rc) return rc;
        s_u = P.s_out;
        P.s_in = s_v;
        P.s_out = last ? nullptr : sv[i & 1];
        P.irr_in = irr_x;
        P.irr_out = last ? nullptr : irr_y;
        P.acc = acc;
        for (int c = 0; c < 3; c++) P.weight[c] = weights[c * num_levels + i];
        if (last) {
            P.irr0 = irradiance_map;
            P.spec = specular_map;
            P.out = out_map;
        }
        rc = b200r_launch("k_sss_blur_y", B200R_K_SSS, k_sss_blur_y, grid, block, 0, st, P);
        if (rc) return rc;
        s_v = P.s_out;
        irr = irr_y;
    }
    return 0;
}
