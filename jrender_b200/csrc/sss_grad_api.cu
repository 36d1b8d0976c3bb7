// sss_grad_api.cu -- gradients of the texture-space subsurface scattering (Lighting.sss_grad): the adjoints of
// b200r_sss_stretch and b200r_sss_blur_pyramid (sss_api.cu).  DESIGN.md section 11, "Gradients".
//
// Arithmetic is float32 unfused (-fmad=false); oracle/sss_grad.py mirrors it in float64 and bounds the difference.
#include <math.h>

#include "../../include/b200raster.h"
#include "api_util.cuh"
#include "sss_common.cuh"

namespace {

using namespace b200r_sss;

// ---------------------------------------------------------------------------------------------------
// The backward recomputes every level's stretch maps and pass inputs with the forward kernels (into its own workspace),
// then walks the levels in reverse: k_sss_bwd_y is the transpose of level i's y pass, k_sss_bwd_x of its x pass.
//
// A y pass's taps stay in the pixel's column and an x pass's in its row.  k_sss_bwd_x gives a whole row to one block
// and accumulates the row's gradients in shared memory, so it writes each gradient once, without global atomics.
// k_sss_bwd_y keeps the forward's 32 x 8 pixel blocks and adds into zeroed planes with global atomics: a column does not
// fit a block's shared memory.

constexpr int kBwdThreads = 256;
constexpr int kMaxBwdWidth = 8192;    // k_sss_bwd_x keeps 4 rows of the map in shared memory: 128 KB at 8192

struct SssBwdPass {
    const float* s_in;      // the stretch map this pass blurs: level i - 1's (the input stretch map at level 0)
    const float* s_cur;     // level i's blurred stretch map: the irradiance blurs' modulation
    const float* irr_in;    // [3, H, W]: this pass's irradiance input
    float* g_cur;           // x: [3, H, W] gradient of this pass's irradiance output (zeroed after reading)
    float* g_in;            // [3, H, W] gradient of irr_in: y adds into it (atomics), x overwrites it
    float* g_s_cur;         // gradient of s_cur from level i + 1 (NULL at the last level); y zeroes it after reading
    float* g_s_in;          // gradient of s_in, or NULL when no stretch gradient is wanted; y adds, x overwrites
    const float* g_next;    // y: [3, H, W] gradient of this level's output as level i + 1's input, or NULL
    const float* grad_out;  // [H, W, 3], rows flipped
    const float* irr0;      // [3, H, W] the unblurred irradiance map
    const float* acc;       // x at level 0: [3, H, W] the weighted sum of the levels
    float* grad_irr0;       // x at level 0: overwritten with the full gradient of irr0 (else NULL)
    float* grad_spec;       // y at the last level: overwritten with grad_out unflipped, planar (else NULL)
    float taps[kTaps];
    float width;
    float weight[3];
    int H, W;
};

// Adjoint of sss_blur_1d at the forward's decisions.  G is the gradient of the blurred value; each tap sends
// G taps[k] (x - x1) to x2 and G taps[k] (x2 - x) to x1 through add(index on the line, value), a replaced neighbour's
// share to the centre.  A tap whose clamped pair is one pixel (x1 == x2) contributes exactly 0 forward and backward, and
// a centre <= 0 nothing.  Returns G d blur / d mod = G width sum_k taps[k] (k - 3) (v2 - v1) when MOD, else 0.
template <bool MOD, class Add>
__device__ __forceinline__ float sss_blur_1d_adjoint(const float* __restrict__ p, int stride, int c, int bound, float mod,
                                                     float G, const SssBwdPass& P, Add add) {
    const float centre = __ldg(p + (size_t)c * stride);
    if (!(centre > 0.f) || G == 0.f) return 0.f;
    const float step = P.width * mod;
    float x = (float)c - step * (float)(kTaps - 1) / 2.f;
    float dmod = 0.f;
#pragma unroll
    for (int k = 0; k < kTaps; k++) {
        int x1 = (int)x;
        int x2 = (int)x + 1;
        x1 = x1 < 0 ? 0 : (x1 > bound ? bound : x1);
        x2 = x2 < 0 ? 0 : (x2 > bound ? bound : x2);
        if (x1 != x2) {
            float v1 = __ldg(p + (size_t)x1 * stride);
            const bool r1 = !((double)v1 > 1e-6);
            float v2 = __ldg(p + (size_t)x2 * stride);
            const bool r2 = !((double)v2 > 1e-6);
            const float gt = G * P.taps[k];
            add(r2 ? c : x2, gt * (x - (float)x1));
            add(r1 ? c : x1, gt * ((float)x2 - x));
            if (MOD) {
                v1 = r1 ? centre : v1;
                v2 = r2 ? centre : v2;
                dmod = dmod + P.taps[k] * (float)(k - 3) * (v2 - v1);
            }
        }
        x = x + step;
    }
    return MOD ? G * P.width * dmod : 0.f;
}

// Transpose of level i's y pass, one thread per pixel.  The gradient of the level's blurred irradiance is its share of
// the composition, w_c,i irr0 g, plus what level i + 1's x pass sent back; it scatters down the pixel's column into
// g_in.  With stretch gradients, the pixel's stretchV_i gradient (from level i + 1, plus the modulation term of the
// three irradiance blurs) goes on through stretchV_i = blur_y(stretchV_{i-1}, mod = stretchV_{i-1}): the image part
// down the column, the modulation part to the pixel itself.
template <bool STRETCH>
__global__ void __launch_bounds__(kBlockX * kBlockY) k_sss_bwd_y(const SssBwdPass P) {
    const int x = blockIdx.x * kBlockX + threadIdx.x, y = blockIdx.y * kBlockY + threadIdx.y;
    if (x >= P.W || y >= P.H) return;
    const size_t hw = (size_t)P.H * P.W, id = (size_t)y * P.W + x;
    const float* g = P.grad_out + ((size_t)(P.H - 1 - y) * P.W + x) * 3;
    const float s = __ldg(P.s_cur + id);
    float gs = 0.f;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float gc = __ldg(g + c);
        if (P.grad_spec) P.grad_spec[c * hw + id] = gc;
        float G = P.weight[c] * __ldg(P.irr0 + c * hw + id) * gc;
        if (P.g_next) G = G + P.g_next[c * hw + id];
        float* gi = P.g_in + c * hw + x;
        gs = gs + sss_blur_1d_adjoint<STRETCH>(P.irr_in + c * hw + x, P.W, y, P.W - 1, s, G, P,
                                                [gi, W = P.W](int j, float v) { atomicAdd(gi + (size_t)j * W, v); });
    }
    if (STRETCH) {
        if (P.g_s_cur) {
            gs = gs + P.g_s_cur[id];
            P.g_s_cur[id] = 0.f;   // ready for level i - 2's atomics
        }
        float* gi = P.g_s_in + x;
        const float m = __ldg(P.s_in + id);
        const float gm = sss_blur_1d_adjoint<true>(P.s_in + x, P.W, y, P.W - 1, m, gs, P,
                                                   [gi, W = P.W](int j, float v) { atomicAdd(gi + (size_t)j * W, v); });
        atomicAdd(P.g_s_in + id, gm);
    }
}

// Transpose of level i's x pass, one block per row: the row's gradients of irr_in (3 channels) and of stretchU_{i-1}
// are accumulated in shared memory and written once.  At level 0 the composition's g * sum_i w_i b_i joins the
// irradiance gradient, which is then the full gradient of the irradiance map.
template <bool STRETCH>
__global__ void __launch_bounds__(kBwdThreads, 2) k_sss_bwd_x(const SssBwdPass P) {
    extern __shared__ float row_grad[];   // [3 + STRETCH][W]
    const int y = blockIdx.x, W = P.W;
    const size_t hw = (size_t)P.H * W, row = (size_t)y * W;
    for (int x = threadIdx.x; x < (3 + STRETCH) * W; x += blockDim.x) row_grad[x] = 0.f;
    __syncthreads();
    for (int x = threadIdx.x; x < W; x += blockDim.x) {
        const size_t id = row + x;
        const float s = __ldg(P.s_cur + id);
        float gs = 0.f;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            float* gc = P.g_cur + c * hw + id;
            const float G = *gc;
            *gc = 0.f;                                  // ready for level i - 1's y pass atomics
            float* sm = row_grad + c * W;
            gs = gs + sss_blur_1d_adjoint<STRETCH>(P.irr_in + c * hw + row, 1, x, W - 1, s, G, P,
                                                    [sm](int j, float v) { atomicAdd(sm + j, v); });
        }
        if (STRETCH) {
            if (P.g_s_cur) gs = gs + P.g_s_cur[id];
            float* sm = row_grad + 3 * W;
            const float m = __ldg(P.s_in + id);
            const float gm = sss_blur_1d_adjoint<true>(P.s_in + row, 1, x, W - 1, m, gs, P,
                                                       [sm](int j, float v) { atomicAdd(sm + j, v); });
            atomicAdd(sm + x, gm);
        }
    }
    __syncthreads();
    for (int x = threadIdx.x; x < W; x += blockDim.x) {
        const size_t id = row + x;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            float v = row_grad[c * W + x];
            if (P.grad_irr0) v = v + __ldg(P.grad_out + ((size_t)(P.H - 1 - y) * W + x) * 3 + c) * __ldg(P.acc + c * hw + id);
            (P.grad_irr0 ? P.grad_irr0 : P.g_in)[c * hw + id] = v;
        }
        if (STRETCH) P.g_s_in[id] = row_grad[3 * W + x];
    }
}

// One term of the stretch map's gradient: for the pixel q and its neighbour nb (right for u, below for v), the
// derivative of clamp(1 / sqrt(sum_c (7 w_c(q) - 7 w_c(nb))^2), 0, 1) with respect to w_c(q) is -7 u^3 d_c with
// d_c = 7 w_c(q) - 7 w_c(nb) where the clamp passes u through (0 < u < 1), and 0 where it is active (this includes every
// face's inside, where d = 0 and u = inf).  Returns g -7 u^3 (0 where clamped) and d in d[].
__device__ __forceinline__ float stretch_term(const float* __restrict__ world, size_t hw, size_t q, size_t nb, float g,
                                              float d[3]) {
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float a = __ldg(world + c * hw + q) * 7.f;
        d[c] = a - __ldg(world + c * hw + nb) * 7.f;
        s = c == 0 ? d[c] * d[c] : s + d[c] * d[c];
    }
    const float u = 1.f / sqrtf(s);
    return (u > 0.f && u < 1.f) ? g * -7.f * (u * u * u) : 0.f;
}

// grad_world [3, H, W] from the gradients of the clamped stretch maps: each pixel gathers its own two terms (as w(q)) and
// those of its left neighbour's u and its upper neighbour's v (as w(nb)).  No atomics.
__global__ void __launch_bounds__(256)
k_sss_stretch_bwd(const float* __restrict__ world, const float* __restrict__ gu, const float* __restrict__ gv,
                  float* __restrict__ grad_world, int H, int W) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    const size_t hw = (size_t)H * W, id = (size_t)y * W + x;
    float d[3], acc[3];
    float k = stretch_term(world, hw, id, (size_t)y * W + (x + 1 < W ? x + 1 : x), __ldg(gu + id), d);
#pragma unroll
    for (int c = 0; c < 3; c++) acc[c] = k * d[c];
    k = stretch_term(world, hw, id, (size_t)(y + 1 < H ? y + 1 : y) * W + x, __ldg(gv + id), d);
#pragma unroll
    for (int c = 0; c < 3; c++) acc[c] = acc[c] + k * d[c];
    if (x > 0) {
        k = stretch_term(world, hw, id - 1, id, __ldg(gu + id - 1), d);
#pragma unroll
        for (int c = 0; c < 3; c++) acc[c] = acc[c] - k * d[c];
    }
    if (y > 0) {
        k = stretch_term(world, hw, id - W, id, __ldg(gv + id - W), d);
#pragma unroll
        for (int c = 0; c < 3; c++) acc[c] = acc[c] - k * d[c];
    }
#pragma unroll
    for (int c = 0; c < 3; c++) grad_world[c * hw + id] = acc[c];
}

// backward workspace planes: 2L stretch maps (levels 0 .. L-1), 3L x-pass outputs, 3(L - 1) y-pass outputs that feed
// the next level, the weighted sum (3), the y passes' gradient planes (3), the x passes' (3), and two ping-pong planes
// each for the stretchU and stretchV gradients
inline size_t sss_bwd_planes(int L) { return (size_t)8 * L + 10; }

}  // namespace

extern "C" size_t b200r_sss_backward_workspace_bytes(int height, int width, int num_levels) {
    if (height <= 0 || width <= 0 || num_levels < 1 || num_levels > kMaxLevels) return 0;
    return sss_bwd_planes(num_levels) * height * width * sizeof(float);
}

extern "C" int b200r_sss_stretch_backward(const float* world_map, const float* grad_stretch_u, const float* grad_stretch_v,
                                          float* grad_world_map, int height, int width, void* stream) {
    if (!world_map || !grad_stretch_u || !grad_stretch_v || !grad_world_map)
        return b200r_fail(B200R_EINVAL, "b200r_sss_stretch_backward: NULL pointer argument");
    if (height <= 0 || width <= 0 || height > 65535)
        return b200r_fail(B200R_EINVAL, "b200r_sss_stretch_backward: map size %d x %d", height, width);
    return b200r_launch("k_sss_stretch_bwd", B200R_K_SSS, k_sss_stretch_bwd, dim3((width + 255) / 256, height), dim3(256),
                        0, (cudaStream_t)stream, world_map, grad_stretch_u, grad_stretch_v, grad_world_map, height, width);
}

extern "C" int b200r_sss_blur_pyramid_backward(const float* stretch_u, const float* stretch_v, const float* irradiance_map,
                                               const float* grad_out, float* grad_irradiance_map, float* grad_specular_map,
                                               float* grad_stretch_u, float* grad_stretch_v, void* workspace,
                                               size_t workspace_bytes, const float* taps, const float* tap_widths,
                                               const float* weights, int num_levels, int height, int width, void* stream) {
    if (!stretch_u || !stretch_v || !irradiance_map || !grad_out || !grad_irradiance_map || !grad_specular_map || !workspace ||
        !taps || !tap_widths || !weights)
        return b200r_fail(B200R_EINVAL, "b200r_sss_blur_pyramid_backward: NULL pointer argument");
    if (!grad_stretch_u != !grad_stretch_v)
        return b200r_fail(B200R_EINVAL, "b200r_sss_blur_pyramid_backward: grad_stretch_u and grad_stretch_v must both be NULL or both set");
    if (height <= 0 || width <= 0 || height != width || width > kMaxBwdWidth)
        return b200r_fail(B200R_EINVAL, "b200r_sss_blur_pyramid_backward: map size %d x %d (the maps must be square, at most %d)",
                          height, width, kMaxBwdWidth);
    if (num_levels < 1 || num_levels > kMaxLevels)
        return b200r_fail(B200R_EINVAL, "b200r_sss_blur_pyramid_backward: num_levels %d outside [1, %d]", num_levels, kMaxLevels);
    const size_t need = b200r_sss_backward_workspace_bytes(height, width, num_levels);
    if (workspace_bytes < need)
        return b200r_fail(B200R_EWORKSPACE, "b200r_sss_blur_pyramid_backward: workspace of %zu bytes, %zu needed",
                          workspace_bytes, need);
    const int L = num_levels;
    const size_t hw = (size_t)height * width;
    float* ws = (float*)workspace;
    float* su = ws;                       // [L][H, W]
    float* sv = su + L * hw;              // [L][H, W]
    float* irr_x = sv + L * hw;           // [L][3, H, W]
    float* irr_y = irr_x + 3 * L * hw;    // [L - 1][3, H, W]
    float* acc = irr_y + 3 * (L - 1) * hw;
    float* g_y = acc + 3 * hw;            // gradient of the x-pass outputs, added into by the y passes
    float* g_x = g_y + 3 * hw;            // gradient of the x-pass inputs, written by the x passes
    float* g_su[2] = {g_x + 3 * hw, g_x + 4 * hw};
    float* g_sv[2] = {g_x + 5 * hw, g_x + 6 * hw};
    const bool stretch = grad_stretch_u != nullptr;
    const dim3 grid((width + kBlockX - 1) / kBlockX, (height + kBlockY - 1) / kBlockY), block(kBlockX, kBlockY);
    cudaStream_t st = (cudaStream_t)stream;

    // the forward's passes again, keeping every level's stretch maps and pass outputs
    PassKernel fwd_x, fwd_y;
    forward_kernels(&fwd_x, &fwd_y);
    for (int i = 0; i < L; i++) {
        SssPass P = {};
        for (int k = 0; k < kTaps; k++) P.taps[k] = taps[i * kTaps + k];
        P.width = tap_widths[i];
        P.H = height;
        P.W = width;
        P.first = i == 0;
        P.s_in = i == 0 ? stretch_u : su + (i - 1) * hw;
        P.s_out = su + i * hw;
        P.irr_in = i == 0 ? irradiance_map : irr_y + 3 * (i - 1) * hw;
        P.irr_out = irr_x + 3 * i * hw;
        int rc = b200r_launch("k_sss_blur_x", B200R_K_SSS, fwd_x, grid, block, 0, st, P);
        if (rc) return rc;
        P.s_in = i == 0 ? stretch_v : sv + (i - 1) * hw;
        P.s_out = sv + i * hw;
        P.irr_in = irr_x + 3 * i * hw;
        P.irr_out = i == L - 1 ? nullptr : irr_y + 3 * i * hw;
        P.acc = acc;
        for (int c = 0; c < 3; c++) P.weight[c] = weights[c * L + i];
        rc = b200r_launch("k_sss_blur_y", B200R_K_SSS, fwd_y, grid, block, 0, st, P);
        if (rc) return rc;
    }

    int rc = b200r_zero(g_y, 3 * hw * sizeof(float), st, "b200r_sss_blur_pyramid_backward");
    if (!rc && stretch) rc = b200r_zero(g_sv[0], 2 * hw * sizeof(float), st, "b200r_sss_blur_pyramid_backward");
    if (!rc && stretch) rc = b200r_zero(grad_stretch_v, hw * sizeof(float), st, "b200r_sss_blur_pyramid_backward");
    if (rc) return rc;
    const size_t smem = (size_t)(3 + (stretch ? 1 : 0)) * width * sizeof(float);
    auto bwd_x = stretch ? k_sss_bwd_x<true> : k_sss_bwd_x<false>;
    auto bwd_y = stretch ? k_sss_bwd_y<true> : k_sss_bwd_y<false>;
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(bwd_x, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return b200r_cuda_fail(e, "k_sss_bwd_x (shared memory)");
    }
    for (int i = L - 1; i >= 0; i--) {
        SssBwdPass B = {};
        for (int k = 0; k < kTaps; k++) B.taps[k] = taps[i * kTaps + k];
        B.width = tap_widths[i];
        for (int c = 0; c < 3; c++) B.weight[c] = weights[c * L + i];
        B.H = height;
        B.W = width;
        B.grad_out = grad_out;
        B.irr0 = irradiance_map;
        // y pass: stretchV_{i-1} -> stretchV_i, irr_x_i -> irr_y_i
        B.s_in = i == 0 ? stretch_v : sv + (i - 1) * hw;
        B.s_cur = sv + i * hw;
        B.irr_in = irr_x + 3 * i * hw;
        B.g_in = g_y;
        B.g_next = i == L - 1 ? nullptr : g_x;
        B.grad_spec = i == L - 1 ? grad_specular_map : nullptr;
        if (stretch) {
            B.g_s_cur = i == L - 1 ? nullptr : g_sv[(L - 1 - i) & 1];
            B.g_s_in = i == 0 ? grad_stretch_v : g_sv[(L - i) & 1];
        }
        rc = b200r_launch("k_sss_bwd_y", B200R_K_SSS, bwd_y, grid, block, 0, st, B);
        if (rc) return rc;
        // x pass: stretchU_{i-1} -> stretchU_i, irr_in_i -> irr_x_i
        B.s_in = i == 0 ? stretch_u : su + (i - 1) * hw;
        B.s_cur = su + i * hw;
        B.irr_in = i == 0 ? irradiance_map : irr_y + 3 * (i - 1) * hw;
        B.g_cur = g_y;
        B.g_in = g_x;
        B.g_next = nullptr;
        B.grad_spec = nullptr;
        B.acc = acc;
        B.grad_irr0 = i == 0 ? grad_irradiance_map : nullptr;
        B.g_s_cur = nullptr;
        B.g_s_in = nullptr;
        if (stretch) {
            B.g_s_cur = i == L - 1 ? nullptr : g_su[(L - 1 - i) & 1];
            B.g_s_in = i == 0 ? grad_stretch_u : g_su[(L - i) & 1];
        }
        rc = b200r_launch("k_sss_bwd_x", B200R_K_SSS, bwd_x, dim3(height), dim3(kBwdThreads), smem, st, B);
        if (rc) return rc;
    }
    return 0;
}
