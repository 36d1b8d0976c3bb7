// texture_atlas_api.cu -- texture-atlas export, the inverse of the bake in bake_api.cu.
//
//   b200r_texture_atlas_softras  <-  create_texture_image_cuda_kernel, jrender/io/utils/create_texture_image.py:3-104,
//                                    called from create_texture_image, jrender/io/save_obj.py:7-29
//   b200r_texture_atlas_n3mr     <-  no reference counterpart (the reference cannot export NMR textures)
//
// One thread per atlas pixel (x, y) of image [H, W, 3].  Face fn = x / R_out + (y / R_out) * tile_width owns the
// R_out x R_out tile the pixel lies in (:25-29); pixels of tiles past the last face are set to 1, the value the reference
// starts its image from (jt.ones, save_obj.py:11), so the kernel writes the whole image.  The pixel's barycentric weights
// in the face's tile triangle (tile_vertices [nf, 3, 2], pixel units) are the reference's (:42-62): face_inv divided by
// (den + eps), w_k = inv . (x, y, 1), clamped to [0, 1] through double literals (`max(min(w, 1.), 0.)`, narrowed to
// float on assignment), then divided by (sum + eps); eps = 1e-5 as save_obj.py:22 passes it.
//
// SoftRas textures [nf, R*R, 3] (:64-72): the weights pick one texel, the inverse of the bake's sample points
// (load_textures.py:29-37): w_x = (int)(w0 R), w_y = (int)(w1 R); texel w_y R + w_x in the lower triangle of the cell,
// (R-1-w_y) R + (R-1-w_x) in the upper one.  A pure copy.  Deviation, documented: the reference indexes the face's
// texels without a bounds check (w0 or w1 rounding up to R, or a NaN weight from degenerate tile vertices, would read
// another face's texels or past the tensor); the texel index is clamped to [0, R*R) here.
//
// NMR textures [nf, ts, ts, ts, 3]: the face's volume is sampled trilinearly at p_k = clamp(w_k (ts-1), 0, ts-1-1e-3),
// with the corner order, index (i0 ts^2 + i1 ts + i2) and weight products of the NMR forward sampler
// (jrender/renderer/dr/n3mr/cuda/rasterize.py:227-298, SURVEY.md Appendix B.2, K8) at depth / z_k = 1 and the
// Renderer's default eps 1e-3.  Same float / double promotions (`max(tif, 0.)`).  This inverts
// b200r_bake_textures_n3mr, which fills texel (a, b, c) from the image at the barycentric point (a, b, c) / (ts-1)
// normalised to sum 1: every texel of a face is baked from a point of the face's triangle, but the atlas keeps only the
// slice a + b + c = ts - 1 of the volume (the weights sum to 1), so what lies off that slice is lost on export.
#include "../../include/b200raster.h"
#include "api_util.cuh"

namespace {

constexpr float kAtlasEps = 1e-5f;   // save_obj.py:22
constexpr float kNmrTexEps = 1e-3f;  // the NMR sampler's clamp eps (rasterize.py:269) at the Renderer's default, renderer.py:12

// :42-62.  Same operand order as the reference; no a*b+c contraction (-fmad=false, build.py).
__device__ __forceinline__ void atlas_weights(const float* __restrict__ tri, int x, int y, float w[3]) {
    const float p0x = __ldg(tri + 0), p0y = __ldg(tri + 1);
    const float p1x = __ldg(tri + 2), p1y = __ldg(tri + 3);
    const float p2x = __ldg(tri + 4), p2y = __ldg(tri + 5);
    float face_inv[9] = {p1y - p2y, p2x - p1x, p1x * p2y - p2x * p1y,
                         p2y - p0y, p0x - p2x, p2x * p0y - p0x * p2y,
                         p0y - p1y, p1x - p0x, p0x * p1y - p1x * p0y};
    const float den = p2x * (p0y - p1y) + p0x * (p1y - p2y) + p1x * (p2y - p0y);
#pragma unroll
    for (int k = 0; k < 9; k++) face_inv[k] /= (den + kAtlasEps);
    float w_sum = 0;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        w[k] = face_inv[3 * k + 0] * (float)x + face_inv[3 * k + 1] * (float)y + face_inv[3 * k + 2];
        // fmin(NaN, 1.) is 1 (a degenerate tile divides by zero); spelled out because nvcc lowers the clamp to a
        // saturate, which takes NaN to 0
        w[k] = w[k] != w[k] ? 1.f : (float)fmax(fmin((double)w[k], 1.), 0.);
        w_sum += w[k];
    }
#pragma unroll
    for (int k = 0; k < 3; k++) w[k] /= (w_sum + kAtlasEps);
}

__global__ void __launch_bounds__(256)
k_texture_atlas_softras(const float* __restrict__ tile_vertices, const float* __restrict__ textures, float* __restrict__ image,
                        int nf, int R, int R_out, int tile_width, long npix, int W) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const int x = (int)(i % W), y = (int)(i / W);
    const long fn = (long)(x / R_out) + (long)(y / R_out) * tile_width;
    float* px = image + i * 3;
    if (fn >= nf) {
        px[0] = px[1] = px[2] = 1.f;
        return;
    }
    float w[3];
    atlas_weights(tile_vertices + fn * 6, x, y, w);
    const int w_x = (int)(w[0] * R), w_y = (int)(w[1] * R);
    int t = ((w[0] + w[1]) * R - w_x - w_y <= 1) ? w_y * R + w_x : (R - 1 - w_y) * R + (R - 1 - w_x);
    t = min(max(t, 0), R * R - 1);
    const float* texel = textures + (fn * R * R + t) * 3;
#pragma unroll
    for (int k = 0; k < 3; k++) px[k] = __ldg(texel + k);
}

__global__ void __launch_bounds__(256)
k_texture_atlas_n3mr(const float* __restrict__ tile_vertices, const float* __restrict__ textures, float* __restrict__ image,
                     int nf, int ts, int R_out, int tile_width, long npix, int W) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const int x = (int)(i % W), y = (int)(i / W);
    const long fn = (long)(x / R_out) + (long)(y / R_out) * tile_width;
    float* px = image + i * 3;
    if (fn >= nf) {
        px[0] = px[1] = px[2] = 1.f;
        return;
    }
    float w[3];
    atlas_weights(tile_vertices + fn * 6, x, y, w);
    float tif[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {                              // rasterize.py:267-270 with depth / z_k = 1
        float t = w[k] * (ts - 1);
        t = (float)fmax((double)t, 0.);
        tif[k] = fminf(t, ts - 1 - kNmrTexEps);
    }
    const float* texture = textures + fn * ts * ts * ts * 3;
    float c[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int pn = 0; pn < 8; pn++) {                           // rasterize.py:274-293, same corner and accumulation order
        float wt = 1;
        int ti[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            if ((pn >> k) % 2 == 0) {
                wt *= 1 - (tif[k] - (int)tif[k]);
                ti[k] = (int)tif[k];
            } else {
                wt *= tif[k] - (int)tif[k];
                ti[k] = (int)tif[k] + 1;
            }
        }
        const int isc = ti[0] * ts * ts + ti[1] * ts + ti[2];
#pragma unroll
        for (int k = 0; k < 3; k++) c[k] += wt * __ldg(texture + isc * 3 + k);
    }
#pragma unroll
    for (int k = 0; k < 3; k++) px[k] = c[k];
}

int check_atlas_args(const char* what, const float* tile_vertices, const float* textures, const float* image, int nf,
                     int texture_res_out, int tile_width, int H, int W) {
    if (!tile_vertices || !textures || !image) return b200r_fail(B200R_EINVAL, "%s: NULL pointer argument", what);
    if (nf < 1) return b200r_fail(B200R_EINVAL, "%s: nf %d < 1", what, nf);
    // texture_res_out 3 puts all three tile vertices on one row (r R + 1 == (r + 1) R - 2): a degenerate triangle
    if (texture_res_out < 2 || texture_res_out == 3)
        return b200r_fail(B200R_EINVAL, "%s: texture_res_out %d (must be 2 or >= 4)", what, texture_res_out);
    if (tile_width < 1 || H < 1 || (long)W != (long)tile_width * texture_res_out)
        return b200r_fail(B200R_EINVAL, "%s: image %d x %d does not hold tiles of %d pixels, %d per row", what, H, W,
                          texture_res_out, tile_width);
    return 0;
}

}  // namespace

extern "C" int b200r_texture_atlas_softras(const float* tile_vertices, const float* textures, float* image, int nf,
                                           int texture_res, int texture_res_out, int tile_width, int image_height,
                                           int image_width, void* stream) {
    if (int rc = check_atlas_args("b200r_texture_atlas_softras", tile_vertices, textures, image, nf, texture_res_out, tile_width,
                                  image_height, image_width))
        return rc;
    if (texture_res < 1) return b200r_fail(B200R_EINVAL, "b200r_texture_atlas_softras: texture_res %d < 1", texture_res);
    cudaStream_t st = (cudaStream_t)stream;
    const long npix = (long)image_height * image_width;
    return b200r_launch("k_texture_atlas_softras", B200R_K_ATLAS, k_texture_atlas_softras, (unsigned)((npix + 255) / 256), 256, 0, st,
                        tile_vertices, textures, image, nf, texture_res, texture_res_out, tile_width, npix, image_width);
}

extern "C" int b200r_texture_atlas_n3mr(const float* tile_vertices, const float* textures, float* image, int nf,
                                        int texture_size, int texture_res_out, int tile_width, int image_height,
                                        int image_width, void* stream) {
    if (int rc = check_atlas_args("b200r_texture_atlas_n3mr", tile_vertices, textures, image, nf, texture_res_out, tile_width,
                                  image_height, image_width))
        return rc;
    if (texture_size < 2)   // the sample points are w_k (ts - 1): one texel per face has no interior to sample
        return b200r_fail(B200R_EINVAL, "b200r_texture_atlas_n3mr: texture_size %d < 2", texture_size);
    cudaStream_t st = (cudaStream_t)stream;
    const long npix = (long)image_height * image_width;
    return b200r_launch("k_texture_atlas_n3mr", B200R_K_ATLAS, k_texture_atlas_n3mr, (unsigned)((npix + 255) / 256), 256, 0, st,
                        tile_vertices, textures, image, nf, texture_size, texture_res_out, tile_width, npix, image_width);
}
