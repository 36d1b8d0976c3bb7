// softras_forward.cuh -- tiled SoftRas forward (replaces K2 / K5 of the reference:
// forward_soft_rasterize_cuda_kernel, cuda/soft_rasterize.py:243-456 and
// cuda/soft_rasterize_coarse_to_fine.py:513-761).
//
// One warp = one CTA = an autonomous worker on 8x4 pixel blocks, one lane per pixel, no CTA-wide barrier anywhere: a
// warp sitting on a mesh pole (10x the work of its neighbours) stalls nobody.  (16x16 and 16x4 multi-warp CTAs were the
// first two versions; stall_barrier was their top stall reason.)  Per block the warp walks its coarse bin's face list
// (ascending face id), keeps the faces whose check_border rectangle touches the block (ordered ballot compaction), stages
// their 160-byte records in shared memory 24 at a time (one bulk copy per record), every lane marks the staged faces that
// cover ITS pixel in a private 24-bit mask, and the lanes then walk their masks in lock-step (lowest bit = lowest face
// id): each pixel visits its faces in ascending id exactly like the reference's `for (fn = 0; fn < nf; fn++)` (:311),
// minus the faces check_border would skip and, in euclidean mode, the pairs beyond the face's reach (reach_lane_mask),
// which the reference's body leaves at its distance threshold.
//
// Scheduling: a persistent grid pulls blocks from an atomic queue (head `tile_counter`) ordered by descending cost
// (number of (pixel, face) pairs per block, computed by k_coarse_bin and bucket-sorted by k_tile_order): blocks at
// poles / silhouettes of a mesh can cost 10x the mean and must start first.  Blocks no face rectangle touches (76 % at
// C3) only store constants; they ride along with the shaded blocks (kFwdEmptyShare) rather than queueing behind them.
#pragma once
#include "softras_math.cuh"
#include "softras_setup.cuh"

namespace b200r {


// shared-memory copy of a record, padded to 176 B: consecutive records then start 11
// 16-byte bank groups apart (11 is odd), so divergent per-lane record reads spread over
// the banks instead of hitting 4 of 8 groups as a 160-byte stride would.
struct __align__(16) FaceRecS {
    FaceRec r;
    uint4 pad;
};

constexpr int kFwdLanes = 32;   // one warp per B200R_BLOCK_W x B200R_BLOCK_H block
static_assert(B200R_BLOCK_W * B200R_BLOCK_H == kFwdLanes, "one lane per pixel of the block");

// resident one-warp CTAs per SM the register allocation must allow (96 registers).  H100, C3: forward 1.08 ms at 20, 1.10
// at 16, 1.29 at 24 (16-record rounds, LDG staging); with bulk copies 1.017 at 20, 1.016 at 22, 1.017 at 18.  Spills
// (ptxas, sm_90a): the C3 instantiation <2,1,false> 60 B stored / 72 B loaded at 96 registers; the others 0-32 B
constexpr int kFwdMinBlocks = 20;

// ---- mbarrier / bulk-copy (TMA) helpers.  Records are staged by cp.async.bulk + mbarrier rather than LDG -> registers
// -> STS: H100, C3 (24-record rounds), forward 0.995 ms with bulk copies, 1.063 ms with LDG staging
__device__ __forceinline__ uint32_t f2_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void f2_mbar_init(unsigned long long* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(f2_smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void f2_mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(f2_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void f2_bulk_g2s(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(f2_smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(f2_smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void f2_mbar_wait(unsigned long long* bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done)
                     : "r"(f2_smem_u32(bar)), "r"(parity)
                     : "memory");
    } while (!done);
}
// generic-proxy accesses to shared memory (the previous round's reads, the output staging writes) ordered before the
// async-proxy writes of the next bulk copies
__device__ __forceinline__ void f2_fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// records staged per round (a multiple of 4, <= 32).  H100, C3, bulk-copy staging: forward 1.017 ms at 16, 0.995 at 24,
// 1.011 at 32 (32 costs resident CTAs: 20 no longer fit the shared memory at K = 16)
constexpr int kFwdChunk = 24;
static_assert(kFwdChunk % 4 == 0 && kFwdChunk <= 32, "lane masks are 32-bit words read four at a time");
constexpr int kFwdUnr = 4;      // coarse entries filtered per lane per pass

struct FwdSmem {
    FaceRecS rec[kFwdChunk];                   // staged records; reused as the output staging area
    int ids[kFwdChunk + kFwdUnr * 32];         // pending block-face ids, ascending
    __align__(16) uint32_t lmask[kFwdChunk];   // per staged record, the lanes whose pixel it covers
    unsigned long long mbar;                   // completion barrier of the bulk copies
    unsigned long long pad_;
};
static_assert(sizeof(FwdSmem) % 16 == 0, "the top-K depth lists behind FwdSmem are read with 16-byte loads");

// Per-pixel depth list stride in floats: K rounded up to a multiple of 4, plus 4.  Pixel-major so that the
// "find the new maximum" rescan reads a lane's K depths with K/4 LDS.128; stride/4 is odd for K = 8, 16, 32, 64,
// which makes those 16-byte accesses bank-conflict free across the 8 lanes of a quarter warp.
__host__ __device__ static inline int fwd_qz_stride(int K) { return ((K + 3) / 4) * 4 + 4; }

// dynamic shared memory: FwdSmem | qz [32][stride] f32 | qid [K][32] i32
static inline size_t fwd_smem_bytes(int K) {
    const size_t b = sizeof(FwdSmem) + (size_t)32 * (fwd_qz_stride(K) + K) * 4;
    return (b + 15) & ~(size_t)15;
}

struct PixState {
    float sc0, sc1, sc2, alpha, softmax_sum, softmax_max, depth_min, q_max_z;
    int face_index_min, q_size, q_max_id;
};

// top-K by z with the reference's "replace the current max" policy (:367-385).  my_qz = this pixel's K depths
// (16-byte aligned, slot order), s_qid = ids [K][32].  The rescan after a replacement is the reference's loop
// (first strictly greater depth wins, so ties keep the lowest slot) reading four slots per LDS.128.
__device__ __forceinline__ void topk_insert(PixState& st, float zp, int fn, int K, float* my_qz, int* s_qid, int tid) {
    if (st.q_size < K) {
        my_qz[st.q_size] = zp;
        s_qid[st.q_size * kFwdLanes + tid] = fn;
        if (zp > st.q_max_z) { st.q_max_z = zp; st.q_max_id = st.q_size; }
        st.q_size++;
    } else if (zp < st.q_max_z) {
        my_qz[st.q_max_id] = zp;
        s_qid[st.q_max_id * kFwdLanes + tid] = fn;
        float m = -1.f;
        int id = st.q_max_id;
        int k = 0;
        for (; k + 4 <= st.q_size; k += 4) {
            const float4 v = *reinterpret_cast<const float4*>(my_qz + k);
            if (v.x > m) { m = v.x; id = k; }
            if (v.y > m) { m = v.y; id = k + 1; }
            if (v.z > m) { m = v.z; id = k + 2; }
            if (v.w > m) { m = v.w; id = k + 3; }
        }
        for (; k < st.q_size; k++) {
            const float z = my_qz[k];
            if (z > m) { m = z; id = k; }
        }
        st.q_max_z = m;
        st.q_max_id = id;
    }
}

// alpha aggregation, before any z test (:349-358, Q2)
template <class Div>
__device__ __forceinline__ void aggregate_alpha(PixState& st, int alpha_func, float soft_fragment, Div& dp) {
    if (alpha_func == 0) {
        if (soft_fragment > 0.5f) st.alpha = 1.f;
    } else if (alpha_func == 1) {
        st.alpha += soft_fragment;
    } else {
        st.alpha = dp.alpha_prod(st.alpha, soft_fragment);
    }
}

// The reference's per-face loop body (:318-420) for one (pixel, face) pair whose pixel is
// inside the face's check_border rectangle; DivPolicy<EXACT, OPT> gives every division its flavour.
// OPT: the pair's arithmetic up to the first state update runs without a single range branch, and a
// pair whose guard dropped (practically never) is re-run through <DIST, RGB, false, false> before
// anything was committed.  The OPT body also collapses the two exp() of the online softmax into one:
// exp((max - z)/gamma) and exp((z - max)/gamma) are never both different from 1 for a finite zp_norm.
// The guarded body keeps both, as it is the one that sees a non-finite zp_norm.
template <int DIST, int RGB, bool EXACT, bool OPT>
__device__ __forceinline__ void shade_face(const FaceRec* rec, PixState& st, const SoftRasParams& P, const DivConst& dc,
                                           float xp, float yp, float threshold, float* s_qz, int* s_qid, int tid,
                                           const float* __restrict__ btex, bool consts_ok) {
    DivPolicy<EXACT, OPT> dp(dc, consts_ok);   // consts_ok = dc.consts_ok(), evaluated once per thread by the kernel
    float w[3];
    barycentric_coordinate(w, xp, yp, rec->inv);

    float soft_fragment = 1.f;
    if (DIST == 0) {
        if (!check_pixel_inside(w)) return;  // :332-333
    } else if (DIST == 1) {
        const float dis = barycentric_p2f_distance(w);
        if (-dis >= threshold) return;  // :337
        soft_fragment = dp.sigmoid(dp.by_sigma(-dis));
    } else {
        float dis_x, dis_y, t[3];
        const float sign = euclidean_p2f_distance<true>(dis_x, dis_y, t, w, rec, xp, yp, dp);
        const float dis = dis_x * dis_x + dis_y * dis_y;
        if (sign < 0.f && dis >= threshold && dp.ok()) return;  // :343 (OPT: an out-of-range pair falls through to the re-run)
        soft_fragment = dp.sigmoid(dp.by_sigma(-sign * dis));
    }

    if constexpr (!OPT) aggregate_alpha(st, P.alpha_func, soft_fragment, dp);

    float wc[3] = {w[0], w[1], w[2]};
    const float zp = clip_and_z<true>(wc, rec, dp);  // barycentric_clip :363 + zp :364
    float zp_norm = 0.f, dz = 0.f, ex = 1.f;
    if constexpr (OPT) {
        if (RGB == 1) {
            zp_norm = dp.by_span(P.far_ - zp);
            dz = zp_norm - st.softmax_max;
            ex = expf(dp.by_gamma(-fabsf(dz)));   // = exp_delta_zp when dz > 0, exp_z otherwise (:402-407)
        }
        if (!dp.ok()) {  // cold: nothing has been committed yet
            shade_face<DIST, RGB, false, false>(rec, st, P, dc, xp, yp, threshold, s_qz, s_qid, tid, btex, consts_ok);
            return;
        }
        aggregate_alpha(st, P.alpha_func, soft_fragment, dp);
    }
    if (zp < P.near_ || zp > P.far_) return;       // :365

    const int fn = (int)rec->face_id;
    topk_insert(st, zp, fn, P.K, s_qz, s_qid, tid);   // s_qz = this pixel's depth list

    const bool front = (rec->flags & 8u) != 0;
    if (RGB == 0) {  // :390-397
        if (zp < st.depth_min && check_pixel_inside(w) && (P.double_side || front)) {
            st.depth_min = zp;
            st.face_index_min = fn;
            float col[3];
            sample_texture_fwd(col, btex, fn, P.T, wc, P.R, P.tex_type, rec, zp);
            st.sc0 = col[0]; st.sc1 = col[1]; st.sc2 = col[2];
        }
    } else if (RGB == 1) {  // :399-419
        if (front || P.double_side) {
            float exp_delta_zp = 1.f, exp_z;
            if constexpr (OPT) {
                const bool up = dz > 0.f;        // zp_norm > softmax_max
                exp_delta_zp = up ? ex : 1.f;
                exp_z = up ? 1.f : ex;           // exp(0 / gamma) == 1 exactly
                if (up) st.softmax_max = zp_norm;
            } else {
                zp_norm = dp.by_span(P.far_ - zp);
                if (zp_norm > st.softmax_max) {
                    exp_delta_zp = expf(dp.by_gamma(st.softmax_max - zp_norm));
                    st.softmax_max = zp_norm;
                }
                exp_z = expf(dp.by_gamma(zp_norm - st.softmax_max));
            }
            st.softmax_sum = exp_delta_zp * st.softmax_sum + exp_z * soft_fragment;
            float col[3];
            sample_texture_fwd(col, btex, fn, P.T, wc, P.R, P.tex_type, rec, zp);
            st.sc0 = exp_delta_zp * st.sc0 + exp_z * soft_fragment * col[0];
            st.sc1 = exp_delta_zp * st.sc1 + exp_z * soft_fragment * col[1];
            st.sc2 = exp_delta_zp * st.sc2 + exp_z * soft_fragment * col[2];
        }
    }
}

// Anti-aliasing epilogue (SoftRasterizer.execute renders at 2x and mean-pools 2x2, rasterizer.py:45,54-55): the 2x2 means
// of one 8x4 block's four colour planes, straight from the block's output staging area s_out[ch][32] (row-major 8x4) to
// pooled [B,4,is/2,is/2].  Lane -> (plane, pooled row, pooled column); a quarter warp writes 16 contiguous bytes.
// Summation order and the division are avg_pool2d's (window scanned row-major, sum / 4).
__device__ __forceinline__ void store_pooled_8x4(const float* s_out, float* __restrict__ pooled, int b, int tx0, int tr0, int is, int lane) {
    const int ch = lane >> 3, pr = (lane >> 2) & 1, pc = lane & 3;
    const float* s = s_out + ch * 32 + (2 * pr) * 8 + 2 * pc;
    const float v = (((s[0] + s[1]) + s[8]) + s[9]) / 4.f;
    const int hp = is >> 1, orow = (tr0 >> 1) + pr, ocol = (tx0 >> 1) + pc;
    if (orow < hp && ocol < hp) pooled[(((size_t)b * 4 + ch) * hp + orow) * hp + ocol] = v;
}

// lanes (row-major 8x4 block at pixel (tx0, tr0)) covered by a check_border rectangle rx = x0 | x1 << 16, rr = r0 | r1 << 16:
// a column mask replicated over the covered rows; 0 when the rectangle misses the block (or is the empty rectangle (1, 0))
__device__ __forceinline__ uint32_t rect_lane_mask(uint32_t rx, uint32_t rr, int tx0, int tr0) {
    const int cx0 = max((int)(rx & 0xffffu) - tx0, 0), cx1 = min((int)(rx >> 16) - tx0, 7);
    const int ry0 = max((int)(rr & 0xffffu) - tr0, 0), ry1 = min((int)(rr >> 16) - tr0, 3);
    if (cx0 > cx1 || ry0 > ry1) return 0u;
    const uint32_t cols = (2u << cx1) - (1u << cx0);
    const uint32_t rows = (0xffffffffu >> (24 - 8 * ry1)) & (0xffffffffu << (8 * ry0));
    return (cols * 0x01010101u) & rows;
}

// Euclidean mode: the lanes a staged record can still shade, i.e. the pixels inside its reach polygon, the rectangle cut
// by the three edge lines moved out by R: support lines of "triangle + disk(R)" (DESIGN.md §4.4).  Only for records
// whose k_face_setup margin (flags bits 10-15, 1/16 px) is set.  Local frame: pixels, column / row offsets from the
// block's first pixel (xb, yb), hs = is / 2; reach = the cull radius without the margin, slack included.  A line's
// direction need not be exact: its offset is the maximum over the three vertices along the computed direction, so it
// contains triangle + disk(R) whatever the direction's rounding.  Per block row a line bounds the column range from
// one side (c <= q or c >= q, q linear in the row); lines too close to horizontal (|a| < 2^-20), or NaN, bound nothing.
// (The three vertex bisectors as well cut 2 % more pairs than the edges alone and cost more than they save.)
__device__ __forceinline__ uint32_t reach_lane_mask(const FaceRec& rec, float xb, float yb, float hs, float reach) {
    const float R = reach + (float)((rec.flags >> 10) & 63u) * 0.0625f;
    float X[3], Y[3], ux[3], uy[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        X[k] = (rec.v[3 * k] - xb) * hs;
        Y[k] = (yb - rec.v[3 * k + 1]) * hs;
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {   // unit vector of edge k: v_k -> v_(k+1)
        const int k1 = (k + 1) % 3;
        const float ex = X[k1] - X[k], ey = Y[k1] - Y[k];
        const float rl = rsqrtf(__fmaf_rn(ex, ex, ey * ey));
        ux[k] = ex * rl;
        uy[k] = ey * rl;
    }
    const float o = __fmaf_rn(ux[0], uy[1], -uy[0] * ux[1]) > 0.f ? 1.f : -1.f;   // (o uy, -o ux) points outward
    float lo[4] = {0.f, 0.f, 0.f, 0.f}, hi[4] = {7.f, 7.f, 7.f, 7.f};
#pragma unroll
    for (int k = 0; k < 3; k++) {
        // edge k's outward normal, of length 1 within 2^-21 (the slack in reach covers R's share of that)
        const float a = o * uy[k], b = -o * ux[k];
        const float H = fmaxf(fmaxf(__fmaf_rn(a, X[0], b * Y[0]), __fmaf_rn(a, X[1], b * Y[1])), __fmaf_rn(a, X[2], b * Y[2])) + R;
        const float ra = __fdividef(1.f, a);
        const float q0 = H * ra, dq = -b * ra;   // row r: a c <= H - b r  <=>  c <= (a > 0) or >= (a < 0) q0 + r dq
        const bool use = fabsf(a) >= 0x1p-20f;
        const float h0 = (use && a > 0.f) ? q0 : 7.f, hd = (use && a > 0.f) ? dq : 0.f;
        const float l0 = (use && a < 0.f) ? q0 : 0.f, ld = (use && a < 0.f) ? dq : 0.f;
#pragma unroll
        for (int r = 0; r < 4; r++) {
            hi[r] = fminf(hi[r], __fmaf_rn((float)r, hd, h0));
            lo[r] = fmaxf(lo[r], __fmaf_rn((float)r, ld, l0));
        }
    }
    uint32_t m = 0u;
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int c0 = __float2int_ru(lo[r]), c1 = __float2int_rd(hi[r]);   // 0 <= c0, c1 <= 7
        if (c0 <= c1) m |= ((2u << c1) - (1u << c0)) << (8 * r);
    }
    return m;
}

// :425-455: a pixel's six output values from its final state.  The three colour quotients share one refined reciprocal
// (fast_div returns the correctly rounded quotient for every input, exact_math.cuh).
template <int RGB>
__device__ __forceinline__ void finalize_pixel(const PixState& st, const SoftRasParams& P, float& o0, float& o1, float& o2,
                                               float& out_a, float& g0, float& g1) {
    if (P.alpha_func == 0) out_a = st.alpha;
    else if (P.alpha_func == 1) out_a = st.alpha / (float)P.nf;
    else out_a = (float)(1.0 - (double)st.alpha);
    if (RGB == 0) {
        o0 = st.sc0; o1 = st.sc1; o2 = st.sc2;  // stays at the (zero) background when no face was hit
        g0 = st.depth_min; g1 = (float)st.face_index_min;
    } else if (RGB == 1) {
        const float r = rcp_refined(st.softmax_sum);
        const bool safe = midrange(st.softmax_sum);
        o0 = fast_div(st.sc0, st.softmax_sum, r, safe);
        o1 = fast_div(st.sc1, st.softmax_sum, r, safe);
        o2 = fast_div(st.sc2, st.softmax_sum, r, safe);
        g0 = st.softmax_sum; g1 = st.softmax_max;
    } else {
        o0 = o1 = o2 = 0.f; g0 = g1 = 0.f;
    }
}

// per-pixel state before the first face, as :291-309 (background buffer is all zero, Q1); softmax_sum0 = exp(eps / gamma)
template <int RGB>
__device__ __forceinline__ PixState initial_state(const SoftRasParams& P, float softmax_sum0) {
    PixState st;
    st.softmax_sum = softmax_sum0;
    st.softmax_max = P.eps;
    if (RGB == 0) { st.sc0 = st.sc1 = st.sc2 = 0.f; }
    else if (RGB == 1) { st.sc0 = st.sc1 = st.sc2 = 0.f * softmax_sum0; }
    else { st.sc0 = st.sc1 = st.sc2 = 1.f; }
    st.alpha = (P.alpha_func == 2) ? 1.f : 0.f;
    st.depth_min = 10000000.f;
    st.face_index_min = -1;
    st.q_size = 0;
    st.q_max_z = -1.f;
    st.q_max_id = -1;
    return st;
}

// Blocks no face rectangle touches: every pixel leaves with its initial state.  Lane j < ne holds queue entry j (ne <= 32,
// warp-uniform).  Six constant planes and the terminator of the id lists, straight from registers, as 16-byte row
// segments (is % 4 == 0 and K % 4 == 0): per block, lane l stores row (l >> 1) & 3, half l & 1 of colour plane l >> 3,
// then lanes 0-15 the same of aggregate plane (l >> 3) & 1 and lanes 16-23 the id terminator -- two stores per lane.
// The values and the lane's offsets are set up once per call, so a block costs its address and its stores.  Nothing
// reads these stores back, so the warp does not wait for them.
template <int RGB>
__device__ __forceinline__ void store_empty_blocks(uint2 ee, int ne, const SoftRasParams& P, float softmax_sum0,
                                                   float* __restrict__ soft_colors, float* __restrict__ aggrs_info,
                                                   int* __restrict__ ids_out, int lane) {
    const int is = P.is;
    const size_t npix = (size_t)is * is;
    float o[6];
    finalize_pixel<RGB>(initial_state<RGB>(P, softmax_sum0), P, o[0], o[1], o[2], o[3], o[4], o[5]);
    const int ch = lane >> 3, r = (lane >> 1) & 3, c = (lane & 1) * 4;
    const float v0 = ch == 0 ? o[0] : ch == 1 ? o[1] : ch == 2 ? o[2] : o[3];
    const float v1 = (ch & 1) ? o[5] : o[4];
    for (int j = 0; j < ne; j++) {
        const uint32_t ex = __shfl_sync(0xffffffffu, ee.x, j), ey = __shfl_sync(0xffffffffu, ee.y, j);
        const int row = (int)(ex >> 16) * B200R_BLOCK_H + r, col = (int)(ex & 0xffffu) * B200R_BLOCK_W + c;
        const size_t b = ey & 0x7fffffffu;
        if (row < is && col < is) {
            const size_t px = (size_t)row * is + col;
            *reinterpret_cast<float4*>(soft_colors + (b * 4 + ch) * npix + px) = make_float4(v0, v0, v0, v0);
            if (lane < 16)
                *reinterpret_cast<float4*>(aggrs_info + (b * 2 + (ch & 1)) * npix + px) = make_float4(v1, v1, v1, v1);
            else if (lane < 24)
                *reinterpret_cast<int4*>(ids_out + b * P.K * npix + px) = make_int4(-1, -1, -1, -1);
        }
    }
}

// Empty blocks stored per shaded block, at most (<= 32: one tile_order load per lane).  Holds the whole empty list of
// the dense workloads (C3: ~3.2 per shaded block); when the shaded blocks are few (a small object in a large image) the
// rest goes through the queue, so that every worker shares the empty blocks and not only those holding a shaded one.
constexpr int kFwdEmptyShare = 8;
static_assert(kFwdEmptyShare <= kFwdLanes, "one tile_order entry per lane");

template <int DIST, int RGB, bool EXACT>
__global__ void __launch_bounds__(32, kFwdMinBlocks)
k_softras_forward(const SoftRasParams P, const FaceRec* __restrict__ recs, const uint2* __restrict__ rects,
                  const int* __restrict__ coarse_cnt, const int* __restrict__ chunk_table,
                  const int* __restrict__ coarse_pool, const int chunks_per_bin, const float* __restrict__ textures, float* __restrict__ soft_colors,
                  float* __restrict__ aggrs_info, int* __restrict__ ids_out, int* tile_counter,
                  const int* __restrict__ n_empty_blocks, const uint2* __restrict__ tile_order, float* __restrict__ pooled) {
    constexpr int NT = kFwdLanes, CHUNK = kFwdChunk, UNR = kFwdUnr, TW = B200R_BLOCK_W, TH = B200R_BLOCK_H;
    constexpr unsigned FULL = 0xffffffffu;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    FwdSmem& S = *reinterpret_cast<FwdSmem*>(smem_raw);
    const int qzs = fwd_qz_stride(P.K);
    float* s_qz_all = reinterpret_cast<float*>(smem_raw + sizeof(FwdSmem));   // [32][qzs]
    int* s_qid = reinterpret_cast<int*>(s_qz_all + (size_t)NT * qzs);         // [K][32]
    const int lane = threadIdx.x;
    float* s_qz = s_qz_all + (size_t)lane * qzs;                              // this pixel's K depths, slot order
    const int is = P.is, nf = P.nf, K = P.K;
    const int lx = lane & 7, ly = lane >> 3;   // lane = row-major pixel index inside the block = index of the [K][4][8] id planes
    const float threshold = P.dist_eps * P.sigma;  // :289
    // reach polygon radius in pixels before a face's margin: border (1 + 2^-19) -- border = sqrt(threshold) as
    // k_face_setup's rectangle uses it -- plus the slack that covers reach_lane_mask's float evaluation (DESIGN.md §4.4).
    // Radii beyond the image size cull nothing the rectangle does not, and keep that evaluation's magnitudes bounded.
    float reach = sqrtf(threshold) * (0.5f * (float)is) * (1.f + 0x1p-19f) + (float)(is + 64) * 0x1p-16f;
    if (!(reach <= (float)is)) reach = -1.f;   // off
    const size_t npix = (size_t)is * is;
    DivConst dc;
    dc.init(P);
    const bool consts_ok = dc.consts_ok();
    const float softmax_sum0 = expf(P.eps / P.gamma);
    const uint32_t lt_mask = (1u << lane) - 1u;
    const bool vec_out = (is & 3) == 0;
    const bool vec_ids = vec_out && ((K & 3) == 0);
    // The queue: tile_order[0, n_shaded) holds the blocks some face rectangle touches, most expensive first, and
    // tile_order[n_shaded, queue_len) the empty ones (cost bucket 0, k_tile_order).  When empty blocks have their
    // constant-store path (vec_ids, no pooled epilogue), shaded entry q also stores its share of the first n_shared empty
    // entries, [q n_shared / n_shaded, (q + 1) n_shared / n_shaded): those stores drain while the warp shades, instead of
    // costing every worker a queue atomic and a tile_order round trip each at the end of the launch, when nothing is left
    // to hide them behind.  The queue head skips the shared entries and hands out what the shares leave.
    const int n_shaded = P.queue_len - *n_empty_blocks;
    const int n_shared = (vec_ids && pooled == nullptr)
                             ? (int)min((long long)P.queue_len - n_shaded, (long long)n_shaded * kFwdEmptyShare) : 0;
    if (lane == 0) f2_mbar_init(&S.mbar, 1);
    __syncwarp();
    uint32_t parity = 0;

    for (;;) {
        // ---- which block
        __syncwarp();  // previous block fully written
        int q = 0;
        if (lane == 0) q = atomicAdd(tile_counter, 1);
        q = __shfl_sync(FULL, q, 0);
        const int slot = q < n_shaded ? q : q + n_shared;
        if (slot >= P.queue_len) break;
        const uint2 te = __ldg(tile_order + slot);  // x | y << 16, image | empty << 31
        if (q < n_shaded && n_shared > 0) {
            const int e0 = (int)((long long)q * n_shared / n_shaded), ne = (int)((long long)(q + 1) * n_shared / n_shaded) - e0;
            const uint2 ee = lane < ne ? __ldg(tile_order + n_shaded + e0 + lane) : make_uint2(0u, 0u);
            store_empty_blocks<RGB>(ee, ne, P, softmax_sum0, soft_colors, aggrs_info, ids_out, lane);
        }
        const int tx = (int)(te.x & 0xffffu);
        const int ty = (int)(te.x >> 16);
        const int b = (int)(te.y & 0x7fffffffu);
        const bool empty = (te.y >> 31) != 0u;   // no face rectangle touches the block (k_coarse_bin's exact per-block count is 0)
        const int tx0 = tx * TW, tr0 = ty * TH;   // block origin
        const int px = tx0 + lx, row = tr0 + ly;

        // ---- empty blocks the shares left to the queue (all of them when no block of the batch is shaded)
        if (empty && vec_ids && pooled == nullptr) {
            store_empty_blocks<RGB>(te, 1, P, softmax_sum0, soft_colors, aggrs_info, ids_out, lane);
            continue;
        }
        PixState st = initial_state<RGB>(P, softmax_sum0);

        const float xp = b200r_pix_coord(px, is);
        const float yp = b200r_pix_coord(is - 1 - row, is);
        // id slots start as -1 (the reference memsets the whole buffer, :470): the block's ids are then written out plane
        // by plane as 16-byte row segments straight from shared memory.  The previous block's stores finished reading
        // s_qid at the __syncwarp at the top of this iteration.
        if (vec_ids) {
            for (int j = lane; j < K * NT / 4; j += NT) reinterpret_cast<int4*>(s_qid)[j] = make_int4(-1, -1, -1, -1);
        }

        const int cbin = (tr0 / P.coarse_px) * P.ncs + (tx0 / P.coarse_px);
        // the bin's face list: runs of B200R_LIST_CHUNK ids in pool chunks (k_coarse_bin); -1 = the pool ran out while this
        // bin was listed, so its blocks filter the complete face list (identity) -- same faces, same order
        const int cnt = empty ? 0 : coarse_cnt[b * P.ncs * P.ncs + cbin];
        const bool unlisted = cnt < 0;
        const int n_coarse = unlisted ? nf : cnt;
        const int* tbl = chunk_table + ((size_t)b * P.ncs * P.ncs + cbin) * chunks_per_bin;
        const uint2* brects = rects + (size_t)b * nf;
        const FaceRec* brecs = recs + (size_t)b * nf;
        const float* btex = textures + (size_t)b * nf * P.T * 3;

        int n_pending = 0, head = 0;  // pending ids live in S.ids[head, head + n_pending); warp-uniform
        for (int base = 0; base < n_coarse; base += NT * UNR) {
            // ---- leftover of the previous pass (< CHUNK entries) back to the front
            if (head > 0) {
                int keep = 0;
                if (lane < n_pending) keep = S.ids[head + lane];
                __syncwarp();
                if (lane < n_pending) S.ids[lane] = keep;
                head = 0;
            }
            // ---- fine filter: next UNR*32 coarse entries -> S.ids (ordered).  All id loads are issued before the
            // dependent rectangle gathers so one pass costs two memory latencies, not 2*UNR.
            {
                int id[UNR];
                uint2 rc[UNR];
                // one pass = 128 consecutive list entries starting at a multiple of 128: inside one chunk
                const int* chunk = unlisted ? nullptr
                                            : coarse_pool + ((size_t)__ldg(tbl + (base >> B200R_LIST_CHUNK_SHIFT)) << B200R_LIST_CHUNK_SHIFT) + (base & (B200R_LIST_CHUNK - 1));
#pragma unroll
                for (int u = 0; u < UNR; u++) {
                    const int i = base + u * NT + lane;
                    id[u] = (i < n_coarse) ? (unlisted ? i : __ldg(chunk + u * NT + lane)) : -1;
                }
#pragma unroll
                for (int u = 0; u < UNR; u++) rc[u] = (id[u] >= 0) ? __ldg(brects + id[u]) : make_uint2(1u, 1u);
#pragma unroll
                for (int u = 0; u < UNR; u++) {
                    const bool pass = id[u] >= 0 && rect_overlaps(rc[u], tx0, tx0 + TW - 1, tr0, tr0 + TH - 1);
                    const unsigned bal = __ballot_sync(FULL, pass);
                    if (pass) S.ids[n_pending + __popc(bal & lt_mask)] = id[u];
                    n_pending += __popc(bal);
                }
            }
            const bool last = base + NT * UNR >= n_coarse;

            while (n_pending >= CHUNK || (last && n_pending > 0)) {
                const int m = min(n_pending, CHUNK);
                __syncwarp();  // S.ids complete; previous round's readers of S.rec done
                // ---- stage m records: one 160-byte bulk copy each, completion counted in bytes on the mbarrier
                f2_fence_async_smem();
                if (lane == 0) f2_mbar_expect_tx(&S.mbar, (uint32_t)m * (uint32_t)sizeof(FaceRec));
                __syncwarp();
                if (lane < m) f2_bulk_g2s(&S.rec[lane].r, brecs + S.ids[head + lane], (uint32_t)sizeof(FaceRec), &S.mbar);
                f2_mbar_wait(&S.mbar, parity);
                parity ^= 1u;
                // ---- per-lane face masks by transposition: lane j turns record j's rectangle, clipped to the 8x4
                // block, into the 32-bit set of covered lanes; every lane then picks its own bit out of the kFwdChunk
                // words (kFwdChunk / 4 broadcast LDS.128).
                // Euclidean mode ANDs in the record's reach polygon when k_face_setup gave it a margin.
                uint32_t lm = 0u;
                const float xb = __shfl_sync(FULL, xp, 0), yb = __shfl_sync(FULL, yp, 0);   // the block's first pixel
                if (lane < m) {
                    const FaceRec& rec = S.rec[lane].r;
                    lm = rect_lane_mask(rec.rect_x, rec.rect_r, tx0, tr0);
                    if (DIST == 2 && reach >= 0.f && (rec.flags >> 10) != 0u) lm &= reach_lane_mask(rec, xb, yb, 0.5f * (float)is, reach);
                }
                if (lane < CHUNK) S.lmask[lane] = lm;
                __syncwarp();
                unsigned mask = 0u;   // bit j: staged record j covers this lane's pixel (ascending record = ascending face id)
#pragma unroll
                for (int q = 0; q < CHUNK / 4; q++) {
                    const uint4 m4 = reinterpret_cast<const uint4*>(S.lmask)[q];
                    mask |= ((m4.x >> lane) & 1u) << (4 * q + 0);
                    mask |= ((m4.y >> lane) & 1u) << (4 * q + 1);
                    mask |= ((m4.z >> lane) & 1u) << (4 * q + 2);
                    mask |= ((m4.w >> lane) & 1u) << (4 * q + 3);
                }
                // ---- the lanes walk their masks in lock-step
                const int maxcnt = __reduce_max_sync(FULL, __popc(mask));
                for (int i = 0; i < maxcnt; i++) {
                    if (mask != 0u) {
                        const FaceRec* rec = &S.rec[__ffs(mask) - 1].r;
                        mask &= mask - 1u;
                        // EXACT (softras_exact_tail = 1): the reference's double-precision tails, guarded divisions
                        shade_face<DIST, RGB, EXACT, !EXACT>(rec, st, P, dc, xp, yp, threshold, s_qz, s_qid, lane, btex, consts_ok);
                    }
                }
                head += m;
                n_pending -= m;
            }
        }

        // ---- finalise (:425-455)
        float o0, o1, o2, out_a, g0, g1;
        finalize_pixel<RGB>(st, P, o0, o1, o2, out_a, g0, g1);

        // Stage the 6 output planes of the block in shared memory and write each plane row with 16-byte stores
        // (32 contiguous bytes per block row).
        __syncwarp();
        float* s_out = reinterpret_cast<float*>(S.rec);  // 6 * 32 floats
        s_out[0 * NT + lane] = o0;
        s_out[1 * NT + lane] = o1;
        s_out[2 * NT + lane] = o2;
        s_out[3 * NT + lane] = out_a;
        s_out[4 * NT + lane] = g0;
        s_out[5 * NT + lane] = g1;
        __syncwarp();
        if (pooled != nullptr) store_pooled_8x4(s_out, pooled, b, tx0, tr0, is, lane);   // anti-aliasing epilogue
        if (vec_out) {
            constexpr int QPR = TW / 4;  // float4 per block row
            for (int j = lane; j < 6 * TH * QPR; j += NT) {
                const int ch = j / (TH * QPR), r = (j % (TH * QPR)) / QPR, q = j % QPR;
                const int orow = tr0 + r, ocol = tx0 + q * 4;
                if (orow < is && ocol < is) {
                    const float4 v = *reinterpret_cast<const float4*>(&s_out[ch * NT + r * TW + q * 4]);
                    float* dst = (ch < 4) ? soft_colors + ((size_t)b * 4 + ch) * npix
                                          : aggrs_info + ((size_t)b * 2 + (ch - 4)) * npix;
                    *reinterpret_cast<float4*>(dst + (size_t)orow * is + ocol) = v;
                }
            }
        } else {
            for (int j = lane; j < 6 * NT; j += NT) {
                const int ch = j / NT, r = (j % NT) / TW, c = j % TW;
                const int orow = tr0 + r, ocol = tx0 + c;
                if (orow < is && ocol < is) {
                    float* dst = (ch < 4) ? soft_colors + ((size_t)b * 4 + ch) * npix
                                          : aggrs_info + ((size_t)b * 2 + (ch - 4)) * npix;
                    dst[(size_t)orow * is + ocol] = s_out[j];
                }
            }
        }
        // top-K ids, slot order, -1 TERMINATED: a pixel's list is slots [0, q_size) followed by one -1 (unless q_size == K);
        // the slots behind the terminator are not written at all (the reference memsets the whole buffer,
        // cudaMemsetAsync(out3_p, -1, ...) :470 + :453-455 -- 268 MB per launch at C3, most of the forward's DRAM traffic).
        // Granularity: an 8-pixel row segment of one id plane is one 32-byte sector, written whole (shorter lists of the
        // segment padded with -1) up to the plane of the segment's longest list + 1, so no sector is partially written.
        if (vec_ids) {
            // s_qid is [K][4][8]: int4 number u covers plane u / 8, block row (u % 8) / 2 (every lane's own id writes were
            // ordered before these cross-lane reads by the __syncwarp above)
            constexpr int QPR = TW / 4, QPP = NT / 4;
            static_assert(TW == 8 && NT == 32 && QPP == 8, "the row-segment maximum below assumes 8x4 blocks");
            int seg = st.q_size;   // longest list of this lane's 8-pixel row segment
            seg = max(seg, __shfl_xor_sync(FULL, seg, 1));
            seg = max(seg, __shfl_xor_sync(FULL, seg, 2));
            seg = max(seg, __shfl_xor_sync(FULL, seg, 4));
            // this lane stores int4 (lane & 7) of planes lane / 8 + 4 i: block row (lane & 7) / 2, whose lanes are 8 * row ...
            const int last_plane = __shfl_sync(FULL, seg, ((lane & 7) >> 1) * 8);
            int* bids = ids_out + (size_t)b * K * npix;
            for (int u = lane; u < K * QPP; u += NT) {
                const int k = u / QPP, pq = u - k * QPP;
                const int orow = tr0 + pq / QPR, ocol = tx0 + (pq % QPR) * 4;
                if (orow < is && ocol < is && k <= last_plane)
                    *reinterpret_cast<int4*>(bids + (size_t)k * npix + (size_t)orow * is + ocol) = reinterpret_cast<const int4*>(s_qid)[u];
            }
        } else if (px < is && row < is) {
            int* dst = ids_out + (size_t)b * K * npix + (size_t)row * is + px;
            for (int k = 0; k < K && k <= st.q_size; k++)
                dst[(size_t)k * npix] = (k < st.q_size) ? s_qid[k * NT + lane] : -1;
        }
    }
}

}  // namespace b200r
