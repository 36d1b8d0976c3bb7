// softras_api.cu -- C ABI entry points for the SoftRas path (see include/b200raster.h).
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>

#include "../../include/b200raster.h"
#include "api_util.cuh"
#include "softras_launch.cuh"
#include "softras_setup.cuh"

using namespace b200r;

namespace {

std::atomic<int> g_exact_tail{0};      // 1: reference's double-precision sigmoid / alpha tails bit for bit; 0: fp32 tails (<= 1 ulp)
std::atomic<int> g_pool_cap{-1};       // >= 0: cap on the coarse-list chunk pool (tests of the pool-exhausted path); -1: the carved size
}  // namespace

namespace {

int validate(const char* fn, int B, int nf, int T, int is, int K, int dist, int rgb, int alpha, int tex,
             float sigma, float gamma) {
    if (B <= 0 || nf <= 0 || T <= 0 || is <= 0) return b200r_fail(B200R_EINVAL, "%s: non-positive size (B=%d nf=%d T=%d image_size=%d)", fn, B, nf, T, is);
    if (is > 4096) return b200r_fail(B200R_EUNSUPPORTED, "%s: image_size %d > 4096", fn, is);
    if (K <= 0 || K > B200R_MAX_FACES_PER_PIXEL)
        return b200r_fail(B200R_EINVAL, "%s: max_faces_per_pixel %d outside [1, %d] (reference kMaxPointsPerPixel)", fn, K, B200R_MAX_FACES_PER_PIXEL);
    if (dist < 0 || dist > 2 || rgb < 0 || rgb > 2 || alpha < 0 || alpha > 2 || tex < 0 || tex > 1)
        return b200r_fail(B200R_EINVAL, "%s: enum out of range (dist=%d rgb=%d alpha=%d tex=%d)", fn, dist, rgb, alpha, tex);
    if (tex == 1 && T != 3) return b200r_fail(B200R_EINVAL, "%s: vertex textures need texture_size 3, got %d", fn, T);
    if (tex == 0) {
        const int R = (int)std::sqrt((double)T);
        if (R * R != T) return b200r_fail(B200R_EINVAL, "%s: surface texture_size %d is not a square", fn, T);
    }
    if (!(sigma != 0.f) || !(gamma != 0.f)) return b200r_fail(B200R_EINVAL, "%s: sigma_val/gamma_val must be non-zero", fn);
    return 0;
}

SoftRasParams make_params(int B, int nf, int T, int is, int K, float near_, float far_, float eps, float sigma,
                          float gamma, float dist_eps, int dist, int rgb, int alpha, int tex, int double_side) {
    SoftRasParams P;
    P.B = B; P.nf = nf; P.T = T; P.R = (int)std::sqrt((double)T); P.is = is; P.K = K;
    P.near_ = near_; P.far_ = far_; P.eps = eps; P.sigma = sigma; P.gamma = gamma; P.dist_eps = dist_eps;
    P.dist_func = dist; P.rgb_func = rgb; P.alpha_func = alpha; P.tex_type = tex; P.double_side = double_side ? 1 : 0;
    b200r_geometry(is, &P.ntx, &P.coarse_px, &P.ncs);
    P.aa = 0;
    P.fntx = (is + B200R_BLOCK_W - 1) / B200R_BLOCK_W;
    P.fnty = (is + B200R_BLOCK_H - 1) / B200R_BLOCK_H;
    P.queue_len = P.fntx * P.fnty * B;  // one entry per forward block
    return P;
}

}  // namespace

extern "C" {

const char* b200r_version(void) { return "b200raster 0.1 (sm_90a)"; }

int b200r_set_option(const char* name, int value) {
    if (!name) return b200r_fail(B200R_EINVAL, "b200r_set_option: NULL name");
    if (!strcmp(name, "softras_exact_tail")) { g_exact_tail.store(value ? 1 : 0); return 0; }
    if (!strcmp(name, "softras_list_pool_chunks")) { g_pool_cap.store(value < 0 ? -1 : value); return 0; }
    return b200r_fail(B200R_EINVAL, "b200r_set_option: unknown option '%s'", name);
}

size_t b200r_softras_workspace_bytes(int batch_size, int num_faces, int image_size) {
    if (batch_size <= 0 || num_faces <= 0 || image_size <= 0) return 0;
    return b200r_carve(nullptr, nullptr, batch_size, num_faces, image_size).bytes;
}

size_t b200r_softras_state_bytes(int batch_size, int num_faces) {
    if (batch_size <= 0 || num_faces <= 0) return 0;
    return b200r_carve(nullptr, nullptr, batch_size, num_faces, 16).state_bytes;
}

static int softras_forward_impl(const float* face_vertices, const float* textures, float* soft_colors,
                                float* aggrs_info, int32_t* faces_id_buffer, float* faces_info, float* pooled, void* state,
                                size_t state_bytes, void* workspace, size_t workspace_bytes, int B, int nf, int T, int is, int K, float near_, float far_,
                                float eps, float sigma_val, float gamma_val, float dist_eps_logit, int dist_func,
                                int rgb_func, int alpha_func, int texture_type, int double_side, void* stream) {
    int rc = validate("b200r_softras_forward", B, nf, T, is, K, dist_func, rgb_func, alpha_func, texture_type, sigma_val, gamma_val);
    if (rc) return rc;
    if (!face_vertices || !textures || !soft_colors || !aggrs_info || !faces_id_buffer || !workspace || !state)
        return b200r_fail(B200R_EINVAL, "b200r_softras_forward: NULL pointer argument");
    SoftRasWorkspace W = b200r_carve(state, workspace, B, nf, is);
    {
        const int cap = g_pool_cap.load();
        if (cap >= 0 && cap < W.pool_chunks) W.pool_chunks = cap;
    }
    if (workspace_bytes < W.bytes)
        return b200r_fail(B200R_EWORKSPACE, "b200r_softras_forward: workspace %zu < required %zu bytes", workspace_bytes, W.bytes);
    if (state_bytes < W.state_bytes)
        return b200r_fail(B200R_EWORKSPACE, "b200r_softras_forward: state %zu < required %zu bytes", state_bytes, W.state_bytes);
    const SoftRasParams P = make_params(B, nf, T, is, K, near_, far_, eps, sigma_val, gamma_val, dist_eps_logit,
                                        dist_func, rgb_func, alpha_func, texture_type, double_side);
    cudaStream_t st = (cudaStream_t)stream;
    const float border = sqrtf(dist_eps_logit * sigma_val);  // sqrt(threshold), :289,:316 (IEEE sqrt on host == device)

    const int total = B * nf;
    if (int rc = b200r_launch("k_face_setup", B200R_K_FACE_SETUP, k_face_setup, (total + 255) / 256, 256, 0, st, face_vertices,
                              textures, W.recs, W.rects, faces_info, total, nf, T, texture_type, is, border))
        return rc;
    if (int rc = b200r_zero(W.counters, 256 * sizeof(int), st, "memset counters")) return rc;
    if (int rc = b200r_launch("k_chunk_rects", B200R_K_CHUNK_RECTS, k_chunk_rects, dim3((nf + 255) / 256, B), 256, 0, st, W.rects,
                              W.chunk_rects, nf))
        return rc;
    if (int rc = b200r_launch("k_coarse_bin", B200R_K_COARSE_BIN, k_coarse_bin, dim3(P.ncs * P.ncs, B), 256, 0, st, W.rects,
                              W.chunk_rects, W.coarse_cnt, W.chunk_table, W.coarse_pool, W.counters + 1, W.chunks_per_bin,
                              W.pool_chunks, W.tile_cost, W.counters + 64, nf, is, P.coarse_px, P.ncs, P.fntx, P.fnty))
        return rc;
    // k_tile_order writes a permutation of all queue_len slots: no holes to pre-fill
    if (int rc = b200r_launch("k_tile_order", B200R_K_TILE_ORDER, k_tile_order, (P.queue_len + 255) / 256, 256, 0, st,
                              W.tile_cost, W.counters + 64, W.counters + 128, W.tile_order, B, P.fntx, P.fnty))
        return rc;
    return b200r_launch_forward(P, W, textures, soft_colors, aggrs_info, faces_id_buffer, pooled, g_exact_tail.load(), st);
}

int b200r_softras_forward(const float* face_vertices, const float* textures, float* soft_colors,
                          float* aggrs_info, int32_t* faces_id_buffer, float* faces_info, void* state, size_t state_bytes,
                          void* workspace, size_t workspace_bytes, int B, int nf, int T, int is, int K, float near_, float far_,
                          float eps, float sigma_val, float gamma_val, float dist_eps_logit, int dist_func,
                          int rgb_func, int alpha_func, int texture_type, int double_side, void* stream) {
    return softras_forward_impl(face_vertices, textures, soft_colors, aggrs_info, faces_id_buffer, faces_info, nullptr, state,
                                state_bytes, workspace, workspace_bytes, B, nf, T, is, K, near_, far_, eps, sigma_val, gamma_val, dist_eps_logit, dist_func,
                                rgb_func, alpha_func, texture_type, double_side, stream);
}

int b200r_softras_forward_aa(const float* face_vertices, const float* textures, float* soft_colors, float* pooled_colors,
                             float* aggrs_info, int32_t* faces_id_buffer, float* faces_info, void* state, size_t state_bytes,
                             void* workspace, size_t workspace_bytes, int B, int nf, int T, int is, int K, float near_, float far_,
                             float eps, float sigma_val, float gamma_val, float dist_eps_logit, int dist_func,
                             int rgb_func, int alpha_func, int texture_type, int double_side, void* stream) {
    if (!pooled_colors) return b200r_fail(B200R_EINVAL, "b200r_softras_forward_aa: NULL pooled_colors");
    if (is & 1) return b200r_fail(B200R_EINVAL, "b200r_softras_forward_aa: supersampled image_size %d is odd", is);
    return softras_forward_impl(face_vertices, textures, soft_colors, aggrs_info, faces_id_buffer, faces_info, pooled_colors, state,
                                state_bytes, workspace, workspace_bytes, B, nf, T, is, K, near_, far_, eps, sigma_val, gamma_val, dist_eps_logit, dist_func,
                                rgb_func, alpha_func, texture_type, double_side, stream);
}

static int softras_backward_impl(const float* face_vertices, const float* textures, const float* soft_colors,
                                 const float* aggrs_info, const int32_t* faces_id_buffer, void* state,
                                 size_t state_bytes, const float* grad_soft_colors, int grad_is_pooled, float* grad_face_vertices,
                                 float* grad_textures, int B, int nf, int T, int is, int K, float near_, float far_,
                                 float eps, float sigma_val, float gamma_val, float dist_eps_logit, int dist_func,
                                 int rgb_func, int alpha_func, int texture_type, int double_side, void* stream) {
    int rc = validate("b200r_softras_backward", B, nf, T, is, K, dist_func, rgb_func, alpha_func, texture_type, sigma_val, gamma_val);
    if (rc) return rc;
    if (!face_vertices || !textures || !soft_colors || !aggrs_info || !faces_id_buffer || !state ||
        !grad_soft_colors || !grad_face_vertices || !grad_textures)
        return b200r_fail(B200R_EINVAL, "b200r_softras_backward: NULL pointer argument");
    const SoftRasWorkspace W = b200r_carve(state, nullptr, B, nf, is);   // the backward reads the records and owns the accumulator
    if (state_bytes < W.state_bytes)
        return b200r_fail(B200R_EWORKSPACE, "b200r_softras_backward: state %zu < required %zu bytes", state_bytes, W.state_bytes);
    SoftRasParams P = make_params(B, nf, T, is, K, near_, far_, eps, sigma_val, gamma_val, dist_eps_logit,
                                  dist_func, rgb_func, alpha_func, texture_type, double_side);
    P.aa = grad_is_pooled ? 1 : 0;
    return b200r_launch_backward(P, W, textures, soft_colors, aggrs_info, faces_id_buffer, grad_soft_colors, grad_face_vertices,
                                 grad_textures, g_exact_tail.load(), (cudaStream_t)stream);
}

int b200r_softras_backward(const float* face_vertices, const float* textures, const float* soft_colors,
                           const float* aggrs_info, const int32_t* faces_id_buffer, void* state,
                           size_t state_bytes, const float* grad_soft_colors, float* grad_face_vertices,
                           float* grad_textures, int B, int nf, int T, int is, int K, float near_, float far_,
                           float eps, float sigma_val, float gamma_val, float dist_eps_logit, int dist_func,
                           int rgb_func, int alpha_func, int texture_type, int double_side, void* stream) {
    return softras_backward_impl(face_vertices, textures, soft_colors, aggrs_info, faces_id_buffer, state, state_bytes,
                                 grad_soft_colors, 0, grad_face_vertices, grad_textures, B, nf, T, is, K, near_, far_, eps, sigma_val,
                                 gamma_val, dist_eps_logit, dist_func, rgb_func, alpha_func, texture_type, double_side, stream);
}

int b200r_softras_backward_aa(const float* face_vertices, const float* textures, const float* soft_colors,
                              const float* aggrs_info, const int32_t* faces_id_buffer, void* state,
                              size_t state_bytes, const float* grad_pooled_colors, float* grad_face_vertices,
                              float* grad_textures, int B, int nf, int T, int is, int K, float near_, float far_,
                              float eps, float sigma_val, float gamma_val, float dist_eps_logit, int dist_func,
                              int rgb_func, int alpha_func, int texture_type, int double_side, void* stream) {
    if (is & 1) return b200r_fail(B200R_EINVAL, "b200r_softras_backward_aa: supersampled image_size %d is odd", is);
    return softras_backward_impl(face_vertices, textures, soft_colors, aggrs_info, faces_id_buffer, state, state_bytes,
                                 grad_pooled_colors, 1, grad_face_vertices, grad_textures, B, nf, T, is, K, near_, far_, eps, sigma_val,
                                 gamma_val, dist_eps_logit, dist_func, rgb_func, alpha_func, texture_type, double_side, stream);
}

}  // extern "C"
