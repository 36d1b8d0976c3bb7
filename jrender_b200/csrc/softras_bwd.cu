// softras_bwd.cu -- backward kernel instantiations.
#include <atomic>

#include "api_util.cuh"
#include "softras_backward.cuh"
#include "softras_launch.cuh"

using namespace b200r;

namespace {
template <int DIST, int RGB, bool EXACT>
cudaError_t launch_lane(const SoftRasParams& P, const SoftRasWorkspace& W, const float* textures, const float* soft_colors,
                        const float* aggrs_info, const int32_t* ids, const float* grad_soft_colors, float* grad_textures,
                        cudaStream_t st) {
    dim3 grid(P.ntx * P.ntx, P.B);
    {
        B200rProfScope prof(B200R_K_SOFTRAS_BWD, st);
        k_softras_backward_lane<DIST, RGB, EXACT><<<grid, B200R_TILE_THREADS, 0, st>>>(P, W.recs, textures, soft_colors, aggrs_info, ids,
                                                                                 grad_soft_colors, W.gacc, grad_textures);
    }
    return cudaGetLastError();
}
}  // namespace

// memset(gacc) -> per-lane kernel -> finalize (writes every element of grad_faces, and of grad_textures when T == 1 surface)
cudaError_t b200r_launch_backward(const SoftRasParams& P, const SoftRasWorkspace& W, const float* textures,
                                  const float* soft_colors, const float* aggrs_info, const int32_t* ids,
                                  const float* grad_soft_colors, float* grad_faces, float* grad_textures,
                                  int exact, cudaStream_t st) {
    cudaError_t e = cudaSuccess;
    const size_t nfaces = (size_t)P.B * P.nf;
    const bool tex_in_acc = (P.tex_type == 0 && P.T == 1);
    e = cudaMemsetAsync(W.gacc, 0, sizeof(float) * 12 * nfaces, st);
    if (e != cudaSuccess) return e;
    if (!tex_in_acc) {
        e = cudaMemsetAsync(grad_textures, 0, sizeof(float) * 3 * (size_t)P.T * nfaces, st);
        if (e != cudaSuccess) return e;
    }
    decltype(&launch_lane<2, 1, true>) launch = nullptr;
    // fp32 tails + optimistic divisions only for the default euclidean distance, as in the forward
    B200R_DISPATCH_DIST_RGB(if constexpr (D == 2) launch = exact ? launch_lane<D, R, true> : launch_lane<D, R, false>;
                            else launch = launch_lane<D, R, true>)
    e = launch(P, W, textures, soft_colors, aggrs_info, ids, grad_soft_colors, grad_textures, st);
    if (e != cudaSuccess) return e;
    {
        B200rProfScope prof(B200R_K_SOFTRAS_BWD_FINALIZE, st);
        k_softras_bwd_finalize<<<(unsigned)((nfaces + 255) / 256), 256, 0, st>>>(W.gacc, grad_faces, grad_textures, (int)nfaces, tex_in_acc ? 1 : 0);
    }
    return cudaGetLastError();
}
