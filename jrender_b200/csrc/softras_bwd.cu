// softras_bwd.cu -- backward kernel instantiations.
#include "api_util.cuh"
#include "softras_backward.cuh"
#include "softras_launch.cuh"

using namespace b200r;

// memset(gacc) -> per-lane kernel -> finalize (writes every element of grad_faces, and of grad_textures when T == 1 surface)
int b200r_launch_backward(const SoftRasParams& P, const SoftRasWorkspace& W, const float* textures,
                          const float* soft_colors, const float* aggrs_info, const int32_t* ids,
                          const float* grad_soft_colors, float* grad_faces, float* grad_textures,
                          int exact, cudaStream_t st) {
    const size_t nfaces = (size_t)P.B * P.nf;
    const bool tex_in_acc = (P.tex_type == 0 && P.T == 1);
    if (int rc = b200r_zero(W.gacc, sizeof(float) * 12 * nfaces, st, "memset gradient accumulator")) return rc;
    if (!tex_in_acc) {
        if (int rc = b200r_zero(grad_textures, sizeof(float) * 3 * (size_t)P.T * nfaces, st, "memset grad_textures")) return rc;
    }
    decltype(&k_softras_backward_lane<2, 1, true>) lane = nullptr;
    // fp32 tails + optimistic divisions only for the default euclidean distance, as in the forward: EXACT = (D != 2)
    // names the exact instance for the other distances, whose fp32 instances are never built
    B200R_DISPATCH_DIST_RGB(lane = exact ? k_softras_backward_lane<D, R, true> : k_softras_backward_lane<D, R, D != 2>)
    if (int rc = b200r_launch("k_softras_backward_lane", B200R_K_SOFTRAS_BWD, lane, dim3(P.ntx * P.ntx, P.B), B200R_TILE_THREADS,
                              0, st, P, W.recs, textures, soft_colors, aggrs_info, ids, grad_soft_colors, W.gacc, grad_textures))
        return rc;
    return b200r_launch("k_softras_bwd_finalize", B200R_K_SOFTRAS_BWD_FINALIZE, k_softras_bwd_finalize,
                        (unsigned)((nfaces + 255) / 256), 256, 0, st, W.gacc, grad_faces, grad_textures, (int)nfaces,
                        tex_in_acc ? 1 : 0);
}
