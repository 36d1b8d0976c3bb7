// softras_backward.cuh -- SoftRas top-K backward (replaces K6 of the reference:
// backward_soft_rasterize_cuda_kernel, cuda/soft_rasterize.py:1177-1360).
//
// The reference issues 9 + 3T scalar global atomicAdd per (pixel, face) pair.  Here every lane walks its own <=K saved
// ids, reads the face record straight from the L1-resident record array, and adds its 12 gradient values (9 vertex +
// 3 colour for T == 1) with THREE 16-byte REDG.E.ADD.F32x4 into a padded accumulator [B*nf][12];
// k_softras_bwd_finalize then unpacks it into grad_face_vertices [.,9] and grad_textures [.,1,3] (36-byte rows cannot
// take 16-byte atomics directly).  Atomic packets drop 4x against the reference and no zero-fill of the outputs is
// needed.  Before the atomics of a step, lanes ^1 and ^8 (horizontal / vertical neighbour pixels) that hold the same
// face add their values by shuffle into the lower lane (merge_same_face).
//
// Measured and dropped, all slower at C3: a walk in ascending face id (ids staged and sorted in shared memory so that
// neighbouring lanes sit on the same record at the same step -- the sort costs more than the L1 sectors it saves);
// merging lanes ^2 and ^16 as well; a complete per-face reduction (match.any groups + block-floating-point REDUX.SUM,
// several times the time of the two-level merge); a warp walking the union of its lanes' ids.
//
// The per-pair arithmetic (pair_gradient) is the reference's, in its order; only the floating-point summation order of
// the atomics differs (as it does run to run in the reference).
#pragma once
#include "softras_math.cuh"

namespace b200r {

// resident 256-thread CTAs per SM the backward's register allocation must allow.  Measured on the H100 at C3: 2 -> 0.675 ms,
// 3 -> 0.606 ms, 4 -> 0.638 ms -- past 24 warps/SM the divergent 160-byte record gathers and the float atomics bind, not
// latency.
constexpr int kBwdMinBlocks = 3;

// Per-pixel constants of the backward.
struct BwdPixel {
    float xp, yp;
    float g[4], oc[4];           // upstream gradient, forward output RGBA
    float softmax_sum, softmax_max;
    float r_ssum; bool s_ssum;   // reciprocal of softmax_sum
    double d_galpha, d_one_minus_alpha;
};

// Gradient contribution of one (pixel, face) pair: gv[k*3+l] = d/d vertex k coord l; gt = texture
// gradient (T == 1 surface: gt[0..2]; vertex: gt[j*3+k]).  For surface textures with T > 1 the hit
// texel index is returned in texel_out and gt[0..2] holds its gradient.  (:1240-1358)
// OPT (only with !EXACT): every division is the branch-free optimistic flavour (exact_math.cuh, DivGuard) and
// `guard.ok` says whether all of them were in range; the caller re-runs the pair with OPT = false otherwise.
template <int DIST, int RGB, bool EXACT, bool OPT = false>
__device__ __forceinline__ void pair_gradient(const FaceRec* rec, int fn, const BwdPixel& px, const SoftRasParams& P,
                                              const DivConst& dc, float nmf, float r_nmf, bool s_nmf,
                                              const float* __restrict__ tex, float gv[9], float gt[9], int& texel_out,
                                              DivGuard& guard) {
    static_assert(!(OPT && EXACT), "the optimistic divisions replace the relaxed ones only");
    auto by_sigma = [&](float a) -> float { if constexpr (OPT) return dc.by_sigma_o(a, guard); else return dc.template by_sigma_t<EXACT>(a); };
    auto by_gamma = [&](float a) -> float { if constexpr (OPT) return dc.by_gamma_o(a, guard); else return dc.template by_gamma_t<EXACT>(a); };
    auto by_span = [&](float a) -> float { if constexpr (OPT) return dc.by_span_o(a, guard); else return dc.template by_span_t<EXACT>(a); };
    auto dv = [&](float a, float b, float r, bool safe) -> float { if constexpr (OPT) return optimistic_div(a, b, r, safe, guard); else return div_t<EXACT>(a, b, r, safe); };
    auto dvar = [&](float a, float b) -> float { if constexpr (OPT) return optimistic_div_var(a, b, guard); else return div_var_t<EXACT>(a, b); };
    auto sigmoid = [&](float x) -> float { if constexpr (OPT) return sigmoid_from_negarg_opt(x, guard); else return sigmoid_from_negarg<EXACT>(x); };
    const float* f = rec->v;
    const float xp = px.xp, yp = px.yp;
    const int T = P.T;
    float w[3], t[3] = {0.f, 0.f, 0.f};
    float dis = 0.f, dis_x = 0.f, dis_y = 0.f, sign = 0.f, soft_fragment;
    texel_out = 0;
    barycentric_coordinate(w, xp, yp, rec->inv);
    if (DIST == 0) {
        soft_fragment = 1.f;  // :1259
    } else if (DIST == 1) {
        dis = barycentric_p2f_distance(w);
        t[0] = w[0]; t[1] = w[1]; t[2] = w[2];
        soft_fragment = sigmoid(by_sigma(-dis));
    } else {
        sign = euclidean_p2f_distance<EXACT>(dis_x, dis_y, t, w, rec, xp, yp, OPT ? &guard : nullptr);
        dis = dis_x * dis_x + dis_y * dis_y;
        soft_fragment = sigmoid(by_sigma(-sign * dis));
    }

    float C_grad_xy = 0.f;
    float C_grad_xy_alpha = px.g[3];
    if (P.alpha_func == 1) {
        C_grad_xy_alpha = C_grad_xy_alpha / (float)P.nf;
    } else if (P.alpha_func == 2) {
        // (float)((double)g_a * ((double)(1 - alpha_out) / max((double)(1 - D), 1e-6)))  (:1289)
        const float omd = 1.f - soft_fragment;
        if (EXACT) {
            const double den = fmax(midrange(omd) ? f2d_mid(omd) : (double)omd, 1e-6);
            const double prod = px.d_galpha * (px.d_one_minus_alpha / den);
            C_grad_xy_alpha = d_midrange(prod) ? d2f_mid(prod) : (float)prod;
        } else {
            C_grad_xy_alpha = C_grad_xy_alpha * dvar(1.f - px.oc[3], fmaxf(omd, 1e-6f));
        }
    }
    C_grad_xy += C_grad_xy_alpha;

    const float w0[3] = {w[0], w[1], w[2]};
    float zp;
    if constexpr (OPT) zp = clip_and_z_opt(w, rec, guard);
    else zp = clip_and_z<EXACT>(w, rec);

    if (RGB == 0) {
        if ((float)fn == px.softmax_max) {  // :1300 (int vs float compare, Q10)
            if (P.tex_type == 0) {
                texel_out = surface_texel(w, P.R);
                gt[0] = px.g[0]; gt[1] = px.g[1]; gt[2] = px.g[2];
            } else {
#pragma unroll
                for (int j = 0; j < 3; j++)
#pragma unroll
                    for (int k = 0; k < 3; k++) gt[j * 3 + k] = w[j] * px.g[k];
            }
        }
    } else if (RGB == 1) {
        float C_grad_xyz_rgb = 0.f;
        const float zp_norm = by_span(P.far_ - zp);
        const float zp_softmax = dv(soft_fragment * expf(by_gamma(zp_norm - px.softmax_max)), px.softmax_sum, px.r_ssum, px.s_ssum);
        float col[3];
        if (P.tex_type == 0) {
            const int j = surface_texel(w, P.R);
            texel_out = j;
            if (T == 1) { col[0] = rec->col[0]; col[1] = rec->col[1]; col[2] = rec->col[2]; }
            else {
#pragma unroll
                for (int k = 0; k < 3; k++) col[k] = __ldg(tex + j * 3 + k);
            }
#pragma unroll
            for (int k = 0; k < 3; k++) gt[k] = zp_softmax * px.g[k];
        } else {
#pragma unroll
            for (int k = 0; k < 3; k++)
                col[k] = w[0] * __ldg(tex + k) + w[1] * __ldg(tex + 3 + k) + w[2] * __ldg(tex + 6 + k);
#pragma unroll
            for (int j = 0; j < 3; j++)
#pragma unroll
                for (int k = 0; k < 3; k++) gt[j * 3 + k] = zp_softmax * (w[j] * px.g[k]);
        }
#pragma unroll
        for (int k = 0; k < 3; k++) C_grad_xyz_rgb += px.g[k] * (col[k] - px.oc[k]);
        C_grad_xyz_rgb *= zp_softmax;
        C_grad_xy += dvar(C_grad_xyz_rgb, soft_fragment);

        const float C_grad_z_rgb = dv(by_gamma(C_grad_xyz_rgb), nmf, r_nmf, s_nmf) * zp * zp;
        const uint32_t fl = rec->flags;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const bool sz = (fl & (16u << k)) != 0;
            const float z = f[3 * k + 2], rz = rec->rz[k];
            gv[k * 3 + 2] = dv(dv(C_grad_z_rgb * w[k], z, rz, sz), z, rz, sz);
        }
    }

    C_grad_xy *= by_sigma(soft_fragment * (1.f - soft_fragment));  // :1336
    if (DIST == 1) {  // backward_barycentric_p2f_distance (:1118-1132), w := t (unclipped)
        const int pm = t[0] > t[1] ? (t[1] > t[2] ? 2 : 1) : (t[0] > t[2] ? 2 : 0);
        const float* inv = rec->inv;
        const float scale2 = dis > 0.f ? sqrtf(dis) : sqrtf(-dis);
#pragma unroll
        for (int l = 0; l < 2; l++)
#pragma unroll
            for (int k = 0; k < 3; k++) {
                float grad_kl = 0.f;
                const float a = -inv[3 * pm + l];
                grad_kl += a * inv[3 * k + 0] * xp;
                grad_kl += a * inv[3 * k + 1] * yp;
                grad_kl += a * inv[3 * k + 2] * 1.f;
                float v = grad_kl * C_grad_xy;
                v = (float)((double)v * (2.0 * (double)scale2));
                gv[k * 3 + l] = v;
            }
    } else if (DIST == 2) {  // :1341-1347
#pragma unroll
        for (int k = 0; k < 3; k++) {
            gv[k * 3 + 0] = 2.f * sign * C_grad_xy * (t[k] + w0[k]) * dis_x;
            gv[k * 3 + 1] = 2.f * sign * C_grad_xy * (t[k] + w0[k]) * dis_y;
        }
    }
}

// aa: grad_soft_colors is the gradient of the 2x2 mean-pooled image [B,4,is/2,is/2]; avg_pool2d's backward hands every
// one of the four source pixels grad / 4 (rasterizer.py:54-55), formed here instead of by a pass over a 4x larger tensor.
__device__ __forceinline__ void load_pixel(BwdPixel& px, const float* __restrict__ soft_colors,
                                           const float* __restrict__ aggrs_info, const float* __restrict__ grad_soft_colors,
                                           int b, size_t pn, size_t npix, bool valid, int aa = 0, int row = 0, int col = 0, int is = 0) {
#pragma unroll
    for (int k = 0; k < 4; k++) { px.g[k] = 0.f; px.oc[k] = 0.f; }
    px.softmax_sum = 1.f;
    px.softmax_max = 0.f;
    if (valid) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (aa) {
                const int hp = is >> 1;
                px.g[k] = __ldg(grad_soft_colors + (((size_t)b * 4 + k) * hp + (row >> 1)) * hp + (col >> 1)) / 4.f;
            } else {
                px.g[k] = __ldg(grad_soft_colors + ((size_t)b * 4 + k) * npix + pn);
            }
            px.oc[k] = __ldg(soft_colors + ((size_t)b * 4 + k) * npix + pn);
        }
        px.softmax_sum = __ldg(aggrs_info + ((size_t)b * 2 + 0) * npix + pn);
        px.softmax_max = __ldg(aggrs_info + ((size_t)b * 2 + 1) * npix + pn);
    }
    px.r_ssum = rcp_refined(px.softmax_sum);
    px.s_ssum = midrange(px.softmax_sum);
    px.d_galpha = (double)px.g[3];
    px.d_one_minus_alpha = (double)(1.f - px.oc[3]);
}

// One butterfly level of warp-side aggregation: lanes L and L ^ D that hold the SAME face add their 12 (silhouette: 6)
// gradient values into the lower lane; the upper lane drops out (key = -1).  Keys differ -> nothing happens.
template <int D, int RGB>
__device__ __forceinline__ void merge_same_face(int& key, float gv[9], float gt[9], int lane) {
    const int pkey = __shfl_xor_sync(0xffffffffu, key, D);
    const bool same = (pkey == key) && (key >= 0);
    const bool lower = (lane & D) == 0;
#pragma unroll
    for (int c = 0; c < 9; c++) {
        if (RGB == 2 && (c % 3) == 2) continue;   // silhouettes: the z gradients are identically 0
        const float o = __shfl_xor_sync(0xffffffffu, gv[c], D);
        if (same && lower) gv[c] += o;
    }
    if (RGB != 2) {
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const float o = __shfl_xor_sync(0xffffffffu, gt[c], D);
            if (same && lower) gt[c] += o;
        }
    }
    if (same && !lower) key = -1;
}

// ---------------------------------------------------------------- per-lane walk + vector atomics
template <int DIST, int RGB, bool EXACT>
__global__ void __launch_bounds__(B200R_TILE_THREADS, kBwdMinBlocks)
k_softras_backward_lane(const SoftRasParams P, const FaceRec* __restrict__ recs, const float* __restrict__ textures,
                        const float* __restrict__ soft_colors, const float* __restrict__ aggrs_info,
                        const int* __restrict__ ids_in, const float* __restrict__ grad_soft_colors,
                        float* __restrict__ gacc /*[B*nf][12]*/, float* __restrict__ grad_textures) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int is = P.is, nf = P.nf, K = P.K, T = P.T;
    const int b = blockIdx.y;
    const int tx = blockIdx.x % P.ntx, ty = blockIdx.x / P.ntx;
    const int pxi = tx * B200R_TILE + (warp & 1) * 8 + (lane & 7);
    const int row = ty * B200R_TILE + (warp >> 1) * 4 + (lane >> 3);
    const bool valid = pxi < is && row < is;
    const size_t npix = (size_t)is * is;
    const size_t pn = (size_t)row * is + pxi;
    const int* src = ids_in + (size_t)b * K * npix + pn;
    int fn = valid ? __ldg(src) : -1;
    // the warp stays convergent (lanes whose list is empty or exhausted idle with key -1) so that lanes holding the same
    // face can combine their contributions by shuffle before the atomics; a list ends at the first -1 (:1236)
    if (__all_sync(0xffffffffu, fn < 0)) return;
    const bool has_list = fn >= 0;

    DivConst dc;
    dc.init(P);
    const bool consts_ok = dc.consts_ok();
    BwdPixel px;
    px.xp = b200r_pix_coord(pxi, is);
    px.yp = b200r_pix_coord(is - 1 - row, is);
    load_pixel(px, soft_colors, aggrs_info, grad_soft_colors, b, pn, npix, has_list, P.aa, row, pxi, is);
    const float nmf = P.near_ - P.far_;
    const float r_nmf = rcp_refined(nmf);
    const bool s_nmf = midrange(nmf);
    const FaceRec* brecs = recs + (size_t)b * nf;
    const float* btex = textures + (size_t)b * nf * T * 3;
    float* bacc = gacc + (size_t)b * nf * 12;
    float* bgt = grad_textures + (size_t)b * nf * T * 3;
    const bool tex_in_acc = (P.tex_type == 0 && T == 1);

    // ids are fetched two slots ahead, so the id of the NEXT face is already in a register when
    // its record is prefetched (waiting for a just-issued id load here stalled every iteration).
    // Prefetching two pairs ahead (ids three ahead) was measured too: no gain at C3.
    const bool merge_ok = tex_in_acc || RGB == 2;   // texel-indexed texture gradients are not merged
    int fn_next = (1 < K && has_list) ? __ldg(src + npix) : -1;
    for (int m = 0; m < K; m++) {
        if (__all_sync(0xffffffffu, fn < 0)) break;
        const int fn_next2 = (m + 2 < K && has_list) ? __ldg(src + (size_t)(m + 2) * npix) : -1;
        if (fn_next >= 0) {  // pull the next face's record (two 128-byte lines) towards L1 behind this pair's math
            const char* nr = reinterpret_cast<const char*>(brecs + fn_next);
            asm volatile("prefetch.global.L1 [%0];" ::"l"(nr));
            asm volatile("prefetch.global.L1 [%0];" ::"l"(nr + 128));
        }
        const FaceRec* rec = brecs + fn;
        float gv[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        float gt[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        int texel;
        DivGuard guard;
        guard.ok = consts_ok;   // launch-constant denominators (sigma, gamma, far - near) validated once per thread
        if (fn < 0) {
            texel = 0;   // idle lane: contributes nothing, only takes part in the shuffles below
        } else if constexpr (!EXACT) {
            // all divisions branch-free; one range flag for the whole pair, one (cold) re-run if it dropped
            pair_gradient<DIST, RGB, false, true>(rec, fn, px, P, dc, nmf, r_nmf, s_nmf, btex + (size_t)fn * T * 3, gv, gt, texel, guard);
            if (!guard.ok) {
#pragma unroll
                for (int c = 0; c < 9; c++) { gv[c] = 0.f; gt[c] = 0.f; }
                pair_gradient<DIST, RGB, false, false>(rec, fn, px, P, dc, nmf, r_nmf, s_nmf, btex + (size_t)fn * T * 3, gv, gt, texel, guard);
            }
        } else {
            pair_gradient<DIST, RGB, EXACT, false>(rec, fn, px, P, dc, nmf, r_nmf, s_nmf, btex + (size_t)fn * T * 3, gv, gt, texel, guard);
        }
        int key = fn;
        if (merge_ok) {
            // neighbouring pixels mostly hold the same face in the same slot (52 % of horizontal neighbours at C3, 79 %
            // at C2; ~4 / ~9 lanes per distinct face per step): the backward is bound by the L2's fp32 atomic rate
            // (~250 G adds/s measured at C2, C3 and C5 alike), so every merged pair of lanes is time saved
            merge_same_face<1, RGB>(key, gv, gt, lane);   // horizontal neighbour
            merge_same_face<8, RGB>(key, gv, gt, lane);   // vertical neighbour
        }
        if (key >= 0) {
            float4* a = reinterpret_cast<float4*>(bacc + (size_t)key * 12);
            atomicAdd(a + 0, make_float4(gv[0], gv[1], gv[2], gv[3]));
            atomicAdd(a + 1, make_float4(gv[4], gv[5], gv[6], gv[7]));
            if (RGB != 2)   // silhouettes: gv[8] (a z gradient) and the colour gradients are identically 0
                atomicAdd(a + 2, make_float4(gv[8], tex_in_acc ? gt[0] : 0.f, tex_in_acc ? gt[1] : 0.f, tex_in_acc ? gt[2] : 0.f));
        }
        if (RGB != 2 && !tex_in_acc && fn >= 0) {
            if (P.tex_type == 0) {
#pragma unroll
                for (int k = 0; k < 3; k++) atomicAdd(bgt + ((size_t)fn * T + texel) * 3 + k, gt[k]);
            } else {
#pragma unroll
                for (int c = 0; c < 9; c++) atomicAdd(bgt + (size_t)fn * 9 + c, gt[c]);
            }
        }
        fn = fn_next;
        fn_next = (fn < 0) ? -1 : fn_next2;   // the list ends at the first -1; the slots behind it were never written
    }
}

// Unpacks the padded accumulator: grad_face_vertices[i][0..8] and, for T == 1 surface textures,
// grad_textures[i][0..2].
__global__ void __launch_bounds__(256)
k_softras_bwd_finalize(const float* __restrict__ gacc, float* __restrict__ grad_faces, float* __restrict__ grad_textures,
                       int total_faces, int tex_in_acc) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total_faces) return;
    const float4* a = reinterpret_cast<const float4*>(gacc + (size_t)i * 12);
    const float4 v0 = a[0], v1 = a[1], v2 = a[2];
    float* g = grad_faces + (size_t)i * 9;
    g[0] = v0.x; g[1] = v0.y; g[2] = v0.z; g[3] = v0.w;
    g[4] = v1.x; g[5] = v1.y; g[6] = v1.z; g[7] = v1.w;
    g[8] = v2.x;
    if (tex_in_acc) {
        float* t = grad_textures + (size_t)i * 3;
        t[0] = v2.y; t[1] = v2.z; t[2] = v2.w;
    }
}

}  // namespace b200r
