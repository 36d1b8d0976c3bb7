// bake_api.cu -- texture baking (SURVEY.md section 8f rank 3).
//
//   b200r_bake_textures_softras  <-  _load_textures_for_softras / load_textures_cuda_kernel,
//                                    jrender/io/utils/load_textures.py:3-101
//   b200r_bake_textures_n3mr     <-  _load_textures_for_n3mr / load_textures_cuda_kernel,
//                                    jrender/io/utils/load_textures.py:103-246
//
// One thread per texel of [nf, R*R, 3]: the texel's barycentric sample point (two triangles of R x R cells per face,
// :29-37), its position in the texture image through the face's UVs (:42-45) and a bilinear fetch (:46-58).  The
// reference kernel promotes through double literals (`1. / 3.`, `1. - w0 - w1`) and narrows to float on assignment;
// the same promotions are made here.  Deviation, documented: the reference reads the image without bounds checks (a UV
// of exactly 1 reads one texel past the row / the image); out-of-image taps are clamped to the last valid element here.
#include "../../include/b200raster.h"
#include "api_util.cuh"

namespace {

__global__ void __launch_bounds__(256)
k_bake_textures_softras(const float* __restrict__ image, const float* __restrict__ faces_uv, const int32_t* __restrict__ is_update,
                        float* __restrict__ textures, long ntexels, int R, int H, int W) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ntexels) return;
    const int fn = (int)(i / (R * R));
    if (__ldg(is_update + fn) == 0) return;                    // :41
    const int w_y = (int)(i % (R * R)) / R, w_x = (int)(i % R);
    float w0, w1, w2;
    if (w_x + w_y < R) {                                       // :29-37
        w0 = (float)((w_x + 1. / 3.) / R);
        w1 = (float)((w_y + 1. / 3.) / R);
    } else {
        w0 = (float)(((R - 1. - w_x) + 2. / 3.) / R);
        w1 = (float)(((R - 1. - w_y) + 2. / 3.) / R);
    }
    w2 = (float)(1. - (double)w0 - (double)w1);
    const float* face = faces_uv + (size_t)fn * 6;
    const float pos_x = (__ldg(face + 0) * w0 + __ldg(face + 2) * w1 + __ldg(face + 4) * w2) * (float)(W - 1);   // :42-43
    const float pos_y = (__ldg(face + 1) * w0 + __ldg(face + 3) * w1 + __ldg(face + 5) * w2) * (float)(H - 1);   // :44-45
    const float weight_x1 = pos_x - (int)pos_x, weight_x0 = 1 - weight_x1;
    const float weight_y1 = pos_y - (int)pos_y, weight_y0 = 1 - weight_y1;
    const long n = (long)H * W;
    const long i00 = (long)(int)pos_y * W + (int)pos_x, i10 = (long)(int)(pos_y + 1) * W + (int)pos_x;
    const long i01 = i00 + 1, i11 = i10 + 1;
    auto px = [&](long j, int k) { return __ldg(image + (j < 0 ? 0 : (j >= n ? n - 1 : j)) * 3 + k); };
    float* texture = textures + i * 3;
#pragma unroll
    for (int k = 0; k < 3; k++) {                              // :50-57, same accumulation order
        float c = 0;
        c += px(i00, k) * (weight_x0 * weight_y0);
        c += px(i10, k) * (weight_x0 * weight_y1);
        c += px(i01, k) * (weight_x1 * weight_y0);
        c += px(i11, k) * (weight_x1 * weight_y1);
        texture[k] = c;
    }
}

// Adjoint of k_bake_textures_softras: every texel of a face with is_update != 0 adds its gradient times the forward's
// four bilinear weights (same promotions) into the same clamped pixels the forward read.  grad_image is zeroed first.
__global__ void __launch_bounds__(256)
k_bake_textures_softras_bwd(const float* __restrict__ grad_textures, const float* __restrict__ faces_uv,
                            const int32_t* __restrict__ is_update, float* __restrict__ grad_image, long ntexels, int R, int H,
                            int W) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ntexels) return;
    const int fn = (int)(i / (R * R));
    if (__ldg(is_update + fn) == 0) return;
    const int w_y = (int)(i % (R * R)) / R, w_x = (int)(i % R);
    float w0, w1, w2;
    if (w_x + w_y < R) {
        w0 = (float)((w_x + 1. / 3.) / R);
        w1 = (float)((w_y + 1. / 3.) / R);
    } else {
        w0 = (float)(((R - 1. - w_x) + 2. / 3.) / R);
        w1 = (float)(((R - 1. - w_y) + 2. / 3.) / R);
    }
    w2 = (float)(1. - (double)w0 - (double)w1);
    const float* face = faces_uv + (size_t)fn * 6;
    const float pos_x = (__ldg(face + 0) * w0 + __ldg(face + 2) * w1 + __ldg(face + 4) * w2) * (float)(W - 1);
    const float pos_y = (__ldg(face + 1) * w0 + __ldg(face + 3) * w1 + __ldg(face + 5) * w2) * (float)(H - 1);
    const float weight_x1 = pos_x - (int)pos_x, weight_x0 = 1 - weight_x1;
    const float weight_y1 = pos_y - (int)pos_y, weight_y0 = 1 - weight_y1;
    const long n = (long)H * W;
    const long i00 = (long)(int)pos_y * W + (int)pos_x, i10 = (long)(int)(pos_y + 1) * W + (int)pos_x;
    const long idx[4] = {i00, i10, i00 + 1, i10 + 1};
    const float wt[4] = {weight_x0 * weight_y0, weight_x0 * weight_y1, weight_x1 * weight_y0, weight_x1 * weight_y1};
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float g = __ldg(grad_textures + i * 3 + k);
#pragma unroll
        for (int j = 0; j < 4; j++) atomicAdd(grad_image + (idx[j] < 0 ? 0 : (idx[j] >= n ? n - 1 : idx[j])) * 3 + k, g * wt[j]);
    }
}

// fmod-based wrap of the reference (:112-119): x > 0 -> fmod(x, y), else y + fmod(x, y)
__device__ __forceinline__ float ref_mod(float x, float y) { return x > 0.f ? fmodf(x, y) : y + fmodf(x, y); }

// NMR textures [nf, ts, ts, ts, 3]: texel (a, b, c) of a face samples the texture image at the barycentric point
// (a, b, c) / (ts - 1), normalised to sum 1 (:138-146).  One thread per texel.  The reference kernel wraps the face's UVs
// IN PLACE from every one of the face's ts^3 threads (a race whose outcome depends on the interleaving when a wrapped
// value is not a fixed point of the wrap, e.g. UV == 0 under REPEAT); here every thread wraps the ORIGINAL UVs once and
// faces_uv is read-only.  Same float / double promotions as the reference (`/ (ts - 1.)` is a double division narrowed
// to float, the sums are float).
template <int WRAP, bool BILINEAR>
__global__ void __launch_bounds__(256)
k_bake_textures_n3mr(const float* __restrict__ image, const float* __restrict__ faces_uv, const int32_t* __restrict__ is_update,
                     float* __restrict__ textures, long ntexels, int ts, int H, int W) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ntexels) return;
    const int fn = (int)(i / ((long)ts * ts * ts));
    if (__ldg(is_update + fn) == 0) return;                    // :150
    float dim0 = (float)(((i / ((long)ts * ts)) % ts) / (ts - 1.));   // :138-140
    float dim1 = (float)(((i / ts) % ts) / (ts - 1.));
    float dim2 = (float)((i % ts) / (ts - 1.));
    if (0 < dim0 + dim1 + dim2) {                              // :141-146
        const float sum = dim0 + dim1 + dim2;
        dim0 /= sum;
        dim1 /= sum;
        dim2 /= sum;
    }
    float face[6];
#pragma unroll
    for (int k = 0; k < 6; k++) {
        float v = __ldg(faces_uv + (size_t)fn * 6 + k);
        if (WRAP == 0) v = ref_mod(v, 1.f);                                            // REPEAT :151-156
        else if (WRAP == 1) v = ref_mod(v, 2.f) < 1.f ? ref_mod(v, 1.f) : 1.f - ref_mod(v, 1.f);   // MIRRORED_REPEAT :157-167
        // CLAMP_TO_EDGE :168-173.  fminf(NaN, 1) is 1; spelled out because nvcc lowers the clamp to a saturating add,
        // which takes NaN to 0
        else if (WRAP == 2) v = v != v ? 1.f : fmaxf(fminf(v, 1.f), 0.f);
        face[k] = v;
    }
    float* texture = textures + i * 3;
    if (WRAP == 3) {                                           // CLAMP_TO_BORDER: the reference writes zeros (:192-194, :205-207)
        texture[0] = texture[1] = texture[2] = 0.f;
        return;
    }
    const float pos_x = (face[0] * dim0 + face[2] * dim1 + face[4] * dim2) * (float)(W - 1);   // :174-175
    const float pos_y = (face[1] * dim0 + face[3] * dim1 + face[5] * dim2) * (float)(H - 1);   // :176-177
    if (BILINEAR) {                                            // :178-195
        const float weight_x1 = pos_x - (int)pos_x, weight_x0 = 1 - weight_x1;
        const float weight_y1 = pos_y - (int)pos_y, weight_y0 = 1 - weight_y1;
        // wrapped UVs lie in [0, 1], so (int)pos is inside the image; the +1 taps are clamped by the reference itself
        const int x0 = min(max((int)pos_x, 0), W - 1), y0 = min(max((int)pos_y, 0), H - 1);
        const int x1 = min((int)pos_x + 1, W - 1), y1 = min((int)(pos_y + 1), H - 1);
#pragma unroll
        for (int k = 0; k < 3; k++) {
            float c = 0;
            c += __ldg(image + ((size_t)y0 * W + x0) * 3 + k) * (weight_x0 * weight_y0);
            c += __ldg(image + ((size_t)y1 * W + x0) * 3 + k) * (weight_x0 * weight_y1);
            c += __ldg(image + ((size_t)y0 * W + x1) * 3 + k) * (weight_x1 * weight_y0);
            c += __ldg(image + ((size_t)y1 * W + x1) * 3 + k) * (weight_x1 * weight_y1);
            texture[k] = c;
        }
    } else {                                                   // nearest neighbour :196-208 (round() on the double promotion)
        const int pos_xi = min(max((int)round((double)pos_x), 0), W - 1);
        const int pos_yi = min(max((int)round((double)pos_y), 0), H - 1);
#pragma unroll
        for (int k = 0; k < 3; k++) texture[k] = __ldg(image + ((size_t)pos_yi * W + pos_xi) * 3 + k);
    }
}

}  // namespace

extern "C" int b200r_bake_textures_n3mr(const float* image, const float* faces_uv, const int32_t* is_update, float* textures,
                                        int nf, int texture_size, int image_height, int image_width, int texture_wrapping,
                                        int use_bilinear, void* stream) {
    if (!image || !faces_uv || !is_update || !textures) return b200r_fail(B200R_EINVAL, "b200r_bake_textures_n3mr: NULL pointer argument");
    if (nf <= 0 || image_height <= 0 || image_width <= 0) return b200r_fail(B200R_EINVAL, "b200r_bake_textures_n3mr: non-positive size");
    if (texture_size < 2)   // the reference divides by (texture_size - 1.): 0 / 0 sample points for texture_size 1
        return b200r_fail(B200R_EINVAL, "b200r_bake_textures_n3mr: texture_size %d < 2", texture_size);
    if (texture_wrapping < 0 || texture_wrapping > 3) return b200r_fail(B200R_EINVAL, "b200r_bake_textures_n3mr: texture_wrapping %d outside [0, 3]", texture_wrapping);
    cudaStream_t st = (cudaStream_t)stream;
    const long ntexels = (long)nf * texture_size * texture_size * texture_size;
    // indexed by texture_wrapping * 2 + use_bilinear
    static constexpr decltype(&k_bake_textures_n3mr<0, false>) kernels[8] = {
        k_bake_textures_n3mr<0, false>, k_bake_textures_n3mr<0, true>, k_bake_textures_n3mr<1, false>, k_bake_textures_n3mr<1, true>,
        k_bake_textures_n3mr<2, false>, k_bake_textures_n3mr<2, true>, k_bake_textures_n3mr<3, false>, k_bake_textures_n3mr<3, true>};
    return b200r_launch("k_bake_textures_n3mr", B200R_K_BAKE, kernels[texture_wrapping * 2 + (use_bilinear ? 1 : 0)],
                        (unsigned)((ntexels + 255) / 256), 256, 0, st, image, faces_uv, is_update, textures, ntexels, texture_size,
                        image_height, image_width);
}

extern "C" int b200r_bake_textures_softras(const float* image, const float* faces_uv, const int32_t* is_update, float* textures,
                                           int nf, int texture_res, int image_height, int image_width, void* stream) {
    if (!image || !faces_uv || !is_update || !textures) return b200r_fail(B200R_EINVAL, "b200r_bake_textures_softras: NULL pointer argument");
    if (nf <= 0 || texture_res <= 0 || image_height <= 0 || image_width <= 0)
        return b200r_fail(B200R_EINVAL, "b200r_bake_textures_softras: non-positive size");
    cudaStream_t st = (cudaStream_t)stream;
    const long ntexels = (long)nf * texture_res * texture_res;
    return b200r_launch("k_bake_textures_softras", B200R_K_BAKE, k_bake_textures_softras, (unsigned)((ntexels + 255) / 256), 256, 0, st,
                        image, faces_uv, is_update, textures, ntexels, texture_res, image_height, image_width);
}

extern "C" int b200r_bake_textures_softras_backward(const float* grad_textures, const float* faces_uv, const int32_t* is_update,
                                                    float* grad_image, int nf, int texture_res, int image_height,
                                                    int image_width, void* stream) {
    if (!grad_textures || !faces_uv || !is_update || !grad_image)
        return b200r_fail(B200R_EINVAL, "b200r_bake_textures_softras_backward: NULL pointer argument");
    if (nf <= 0 || texture_res <= 0 || image_height <= 0 || image_width <= 0)
        return b200r_fail(B200R_EINVAL, "b200r_bake_textures_softras_backward: non-positive size");
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = b200r_zero(grad_image, (size_t)image_height * image_width * 3 * sizeof(float), st,
                            "b200r_bake_textures_softras_backward"))
        return rc;
    const long ntexels = (long)nf * texture_res * texture_res;
    return b200r_launch("k_bake_textures_softras_bwd", B200R_K_BAKE, k_bake_textures_softras_bwd,
                        (unsigned)((ntexels + 255) / 256), 256, 0, st, grad_textures, faces_uv, is_update, grad_image, ntexels,
                        texture_res, image_height, image_width);
}
