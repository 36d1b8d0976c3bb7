// softras_fwd.cu -- forward kernel instantiations (one-warp CTAs on 8x4 pixel blocks) and their launcher.
#include <atomic>

#include "api_util.cuh"
#include "softras_forward.cuh"
#include "softras_launch.cuh"

using namespace b200r;

namespace {
constexpr int MAXDEV = 64;   // function attributes and occupancy are per DEVICE: cached per ordinal

template <int DIST, int RGB, bool EXACT>
cudaError_t launch_forward(const SoftRasParams& P, const SoftRasWorkspace& W, const float* textures, float* soft_colors,
                           float* aggrs_info, int32_t* ids, float* pooled, int persistent, cudaStream_t st) {
    const size_t smem = fwd_smem_bytes(P.K);
    static std::atomic<size_t> cfg_smem[MAXDEV];
    static std::atomic<int> cfg_occ[MAXDEV];
    static std::atomic<int> cfg_sms[MAXDEV];
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const int slot = dev < MAXDEV ? dev : MAXDEV - 1;
    if (cfg_smem[slot].load() != smem || dev >= MAXDEV) {
        e = cudaFuncSetAttribute(k_softras_forward<DIST, RGB, EXACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        // The persistent grid is sized for the occupancy the FULL shared-memory carve-out allows.  Left to the driver's
        // per-function heuristic the carve-out sometimes came out smaller: the same kernel then ran with fewer resident
        // CTAs than the grid assumed and was 25-35 % slower for the lifetime of the process (seen on C2 / C5).
        e = cudaFuncSetAttribute(k_softras_forward<DIST, RGB, EXACT>, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
        if (e != cudaSuccess) return e;
        int occ = 1, sms = 0;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_softras_forward<DIST, RGB, EXACT>, 32, smem);
        if (e != cudaSuccess) return e;
        e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (e != cudaSuccess) return e;
        cfg_occ[slot].store(occ < 1 ? 1 : occ);
        cfg_sms[slot].store(sms < 1 ? 1 : sms);
        cfg_smem[slot].store(smem);
    }
    const int tiles = P.fntx * P.fnty;
    int* counter = nullptr;
    dim3 grid(tiles, P.B);
    if (persistent) {
        counter = W.counters;
        const long long total = (long long)tiles * P.B;
        const long long slots = (long long)cfg_sms[slot].load() * cfg_occ[slot].load();
        grid = dim3((unsigned)(total < slots ? total : slots), 1);
    }
    {
        B200rProfScope prof(B200R_K_SOFTRAS_FWD, st);
        k_softras_forward<DIST, RGB, EXACT><<<grid, 32, smem, st>>>(
            P, W.recs, W.rects, W.coarse_cnt, W.chunk_table, W.coarse_pool, W.chunks_per_bin, textures, soft_colors, aggrs_info, ids, counter, W.tile_order, pooled);
    }
    return cudaGetLastError();
}

}  // namespace

cudaError_t b200r_launch_forward(const SoftRasParams& P, const SoftRasWorkspace& W, const float* textures, float* soft_colors,
                                 float* aggrs_info, int32_t* ids, float* pooled, int persistent, int exact, cudaStream_t st) {
    decltype(&launch_forward<2, 1, true>) launch = nullptr;
    // fp32 tails + optimistic divisions only for the default euclidean distance; the other modes keep the exact tails
    B200R_DISPATCH_DIST_RGB(if constexpr (D == 2) launch = exact ? launch_forward<D, R, true> : launch_forward<D, R, false>;
                            else launch = launch_forward<D, R, true>)
    return launch(P, W, textures, soft_colors, aggrs_info, ids, pooled, persistent, st);
}
