// nmr_api.cu -- C ABI entry points for the NMR (dr_type='n3mr') path (see include/b200raster.h).
#include <atomic>
#include <cmath>
#include <cstring>

#include "../../include/b200raster.h"
#include "api_util.cuh"
#include "nmr_kernels.cuh"

using namespace b200r;

// K9's two kernels and its packed record width (floats) per MODE (1: rgb, 2: alpha, 3: both)
struct K9Kernels { decltype(&k_nmr_pack<1>) pack; decltype(&k_nmr_backward_pixel_map<1>) pixel_map; size_t fl; };
template <int MODE>
static constexpr K9Kernels kK9 = {&k_nmr_pack<MODE>, &k_nmr_backward_pixel_map<MODE>, K9Rec<MODE>::FL};

extern "C" {

size_t b200r_nmr_workspace_bytes(int batch_size, int num_faces, int image_size) {
    if (batch_size <= 0 || num_faces <= 0 || image_size <= 0) return 0;
    return (size_t)batch_size * image_size * image_size * sizeof(unsigned long long);   // the (depth, face id) z-buffer
}

int b200r_nmr_forward(const float* faces, const float* textures, int32_t* face_index_map, float* weight_map,
                      float* depth_map, float* rgb_map, float* alpha_map, int32_t* sampling_index_map,
                      float* sampling_weight_map, float* face_inv_map, void* workspace, size_t workspace_bytes,
                      int B, int nf, int texture_size, int is, float near_, float far_, float eps,
                      const float* background_rgb, int return_rgb, int return_alpha, int return_depth, void* stream) {
    if (B <= 0 || nf <= 0 || is <= 0) return b200r_fail(B200R_EINVAL, "b200r_nmr_forward: non-positive size (B=%d nf=%d image_size=%d)", B, nf, is);
    if (is > 4096) return b200r_fail(B200R_EUNSUPPORTED, "b200r_nmr_forward: image_size %d > 4096", is);
    if (!faces || !face_index_map || !weight_map || !depth_map || !workspace)
        return b200r_fail(B200R_EINVAL, "b200r_nmr_forward: NULL pointer argument");
    if (return_rgb && (!textures || !rgb_map || !sampling_index_map || !sampling_weight_map || texture_size <= 0))
        return b200r_fail(B200R_EINVAL, "b200r_nmr_forward: return_rgb needs textures, rgb_map, sampling maps and texture_size > 0");
    if (return_alpha && !alpha_map) return b200r_fail(B200R_EINVAL, "b200r_nmr_forward: return_alpha needs alpha_map");
    if (return_depth && !face_inv_map) return b200r_fail(B200R_EINVAL, "b200r_nmr_forward: return_depth needs face_inv_map");
    const size_t need = b200r_nmr_workspace_bytes(B, nf, is);
    if (workspace_bytes < need)
        return b200r_fail(B200R_EWORKSPACE, "b200r_nmr_forward: workspace %zu < required %zu bytes", workspace_bytes, need);
    NmrParams P;
    P.B = B; P.nf = nf; P.ts = texture_size; P.is = is; P.near_ = near_; P.far_ = far_; P.eps = eps;
    for (int k = 0; k < 3; k++) P.bg[k] = background_rgb ? background_rgb[k] : 0.f;
    P.return_rgb = return_rgb ? 1 : 0; P.return_alpha = return_alpha ? 1 : 0; P.return_depth = return_depth ? 1 : 0;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long* zbuf = reinterpret_cast<unsigned long long*>(workspace);
    cudaError_t e = cudaMemsetAsync(zbuf, 0xFF, need, st);   // every pixel: "no face yet"
    if (e != cudaSuccess) return b200r_cuda_fail(e, "memset z-buffer");
    const long nfaces = (long)B * nf;
    if (int rc = b200r_launch("k_nmr_zbuffer", B200R_K_NMR_SETUP, k_nmr_zbuffer, (unsigned)((nfaces + 255) / 256), 256, 0, st,
                              faces, zbuf, B, nf, is, near_, far_))
        return rc;
    const size_t npix = (size_t)B * is * is;
    return b200r_launch("k_nmr_resolve", B200R_K_NMR_FWD, k_nmr_resolve, (unsigned)((npix + 255) / 256), 256, 0, st, P, zbuf, faces,
                        textures, face_index_map, weight_map, depth_map, rgb_map, alpha_map, sampling_index_map,
                        sampling_weight_map, face_inv_map);
}

size_t b200r_nmr_backward_scratch_bytes(int batch_size, int image_size) {
    if (batch_size <= 0 || image_size <= 0) return 0;
    return 2 * (size_t)batch_size * image_size * image_size * 32;  // row-major + column-major packed pixel records
}

int b200r_nmr_backward(const float* faces, const int32_t* face_index_map, const float* weight_map,
                       const float* depth_map, const float* rgb_map, const float* alpha_map,
                       const int32_t* sampling_index_map, const float* sampling_weight_map,
                       const float* face_inv_map, const float* grad_rgb_map, const float* grad_alpha_map,
                       const float* grad_depth_map, float* grad_faces, float* grad_textures, void* scratch,
                       size_t scratch_bytes, int B, int nf, int texture_size, int is, float eps, int return_rgb,
                       int return_alpha, int return_depth, void* stream) {
    if (B <= 0 || nf <= 0 || is <= 0) return b200r_fail(B200R_EINVAL, "b200r_nmr_backward: non-positive size");
    if (!faces || !face_index_map || !grad_faces) return b200r_fail(B200R_EINVAL, "b200r_nmr_backward: NULL pointer argument");
    if (return_rgb && (!rgb_map || !grad_rgb_map || !sampling_index_map || !sampling_weight_map || !grad_textures || texture_size <= 0))
        return b200r_fail(B200R_EINVAL, "b200r_nmr_backward: return_rgb needs rgb_map, grad_rgb_map, sampling maps, grad_textures");
    if (return_alpha && (!alpha_map || !grad_alpha_map)) return b200r_fail(B200R_EINVAL, "b200r_nmr_backward: return_alpha needs alpha_map and grad_alpha_map");
    if (return_depth && (!depth_map || !weight_map || !face_inv_map || !grad_depth_map))
        return b200r_fail(B200R_EINVAL, "b200r_nmr_backward: return_depth needs depth_map, weight_map, face_inv_map, grad_depth_map");
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = b200r_zero(grad_faces, sizeof(float) * 9 * (size_t)B * nf, st, "memset grad_faces")) return rc;   // rasterize.py:623
    if (return_rgb) {
        const size_t bytes = sizeof(float) * 3 * (size_t)texture_size * texture_size * texture_size * B * nf;
        if (int rc = b200r_zero(grad_textures, bytes, st, "memset grad_textures")) return rc;   // :705
    }
    if (return_rgb || return_alpha) {  // n3mr.py:150-154
        const size_t need = b200r_nmr_backward_scratch_bytes(B, is);
        if (!scratch || scratch_bytes < need)
            return b200r_fail(B200R_EWORKSPACE, "b200r_nmr_backward: scratch %zu < required %zu bytes", scratch_bytes, need);
        const int mode = (return_rgb ? 1 : 0) | (return_alpha ? 2 : 0);
        const K9Kernels k9 = mode == 1 ? kK9<1> : mode == 2 ? kK9<2> : kK9<3>;
        float* ph = reinterpret_cast<float*>(scratch);
        float* pv = ph + (size_t)B * is * is * k9.fl;
        const long warps = (long)B * nf;
        if (int rc = b200r_launch("k_nmr_pack", B200R_K_NMR_PACK, k9.pack, dim3((is + 31) / 32, (is + 31) / 32, B), 256, 0, st,
                                  rgb_map, alpha_map, grad_rgb_map, grad_alpha_map, ph, pv, is))
            return rc;
        if (int rc = b200r_launch("k_nmr_backward_pixel_map", B200R_K_NMR_BWD_PIXEL, k9.pixel_map, (unsigned)((warps + 7) / 8), 256,
                                  0, st, faces, face_index_map, rgb_map, alpha_map, ph, pv, grad_faces, B, nf, is, eps))
            return rc;
    }
    if (!return_rgb && !return_depth) return 0;
    const size_t npix = (size_t)B * is * is;
    return b200r_launch("k_nmr_backward_maps", B200R_K_NMR_BWD_MAPS, k_nmr_backward_maps, (unsigned)((npix + 255) / 256), 256, 0, st,
                        faces, face_index_map, weight_map, depth_map, face_inv_map, sampling_index_map, sampling_weight_map,
                        grad_rgb_map, grad_depth_map, grad_faces, grad_textures, B, nf, is, texture_size, return_rgb ? 1 : 0,
                        return_depth ? 1 : 0);
}

}  // extern "C"
