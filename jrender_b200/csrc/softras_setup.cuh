// softras_setup.cuh -- per-face setup (K1 replacement) and deterministic coarse binning.
#pragma once
#include "common.cuh"
#include "exact_math.cuh"

namespace b200r {

// First index i in [0, is] whose coordinate does NOT satisfy (coord < lim); i.e. the first
// pixel that survives the `x < min - threshold` half of check_border (:31,:33).
__device__ __forceinline__ int first_not_below(float lim, int is) {
    if (isnan(lim)) return 0;  // comparisons with NaN are false -> nothing is rejected
    const double e = ceil(((double)lim * (double)is + (double)is - 1.0) * 0.5);
    int i = e < 0.0 ? 0 : (e > (double)is ? is : (int)e);
    while (i > 0 && !(b200r_pix_coord(i - 1, is) < lim)) --i;
    while (i < is && (b200r_pix_coord(i, is) < lim)) ++i;
    return i;
}

// Last index i in [-1, is-1] whose coordinate does NOT satisfy (coord > lim) (:30,:32).
__device__ __forceinline__ int last_not_above(float lim, int is) {
    if (isnan(lim)) return is - 1;
    const double e = floor(((double)lim * (double)is + (double)is - 1.0) * 0.5);
    int i = e < -1.0 ? -1 : (e > (double)(is - 1) ? is - 1 : (int)e);
    while (i < is - 1 && !(b200r_pix_coord(i + 1, is) > lim)) ++i;
    while (i >= 0 && (b200r_pix_coord(i, is) > lim)) --i;
    return i;
}

// Reach-cull margin of one face (DESIGN.md §4.4), in 1/16 pixel, 1..63; 0 = the face keeps the rectangle mask.  For
// every pixel centre p of the face's rectangle [xlo, xhi] x [ylo, yhi] whose distance to the triangle is at least
// border (1 + 4u) + margin, the euclidean per-pair body computes sign < 0 and dis >= threshold, whichever edge it picks.
// inv = the record's float inverse, exactly as the body uses it: lam_k(p) = inv_k . (x, y, 1) is affine in p, so its
// excursion from the true barycentrics (E, S below) is bounded over the rectangle by its four corners, in double.
__device__ __forceinline__ uint32_t reach_margin_q(const float f[9], const float inv[9], double xlo, double xhi, double ylo,
                                                  double yhi, int is) {
    const double u = 0x1p-24, g3 = 3 * u / (1 - 3 * u), g4 = 4 * u / (1 - 4 * u);
    double M = 0.0, Lmax2 = 0.0;
    for (int k = 0; k < 3; k++) {
        if (!isfinite(f[3 * k]) || !isfinite(f[3 * k + 1])) return 0u;
        M = fmax(M, fmax(fabs((double)f[3 * k]), fabs((double)f[3 * k + 1])));
        const int k1 = (k + 1) % 3;
        const double dx = (double)f[3 * k1] - f[3 * k], dy = (double)f[3 * k1 + 1] - f[3 * k + 1];
        Lmax2 = fmax(Lmax2, dx * dx + dy * dy);
    }
    for (int k = 0; k < 9; k++)
        if (!isfinite(inv[k])) return 0u;
    const double D = ((double)f[3] - f[0]) * ((double)f[7] - f[1]) - ((double)f[4] - f[1]) * ((double)f[6] - f[0]);
    // bounded vertices; conditioning: twice the area against the longest edge squared (smallest altitude / longest
    // edge >= 2^-12) keeps the barycentrics over the rectangle, and with them the rounding terms below, bounded
    if (!(M <= 4.0) || !(fabs(D) >= 0x1p-12 * Lmax2) || !(Lmax2 > 0.0)) return 0u;
    const double X = fmax(fabs(xlo), fabs(xhi)), Y = fmax(fabs(ylo), fabs(yhi));
    double ex = 0.0, ey = 0.0, es = 0.0, lam_max[3] = {0.0, 0.0, 0.0}, mag = 0.0;
    for (int c = 0; c < 4; c++) {
        const double px = (c & 1) ? xhi : xlo, py = (c & 2) ? yhi : ylo;
        double sx = -px, sy = -py, ss = -1.0;
        for (int k = 0; k < 3; k++) {
            const double l = (double)inv[3 * k] * px + (double)inv[3 * k + 1] * py + inv[3 * k + 2];
            sx += l * f[3 * k];
            sy += l * f[3 * k + 1];
            ss += l;
            lam_max[k] = fmax(lam_max[k], fabs(l));
        }
        ex = fmax(ex, fabs(sx)); ey = fmax(ey, fabs(sy)); es = fmax(es, fabs(ss));
    }
    double sig = 0.0, sig_v = 0.0, W = 0.0;   // sig: the float evaluation of w_k = inv_k . (x, y, 1), summed over k
    for (int k = 0; k < 3; k++) {
        const double s = g3 * (fabs((double)inv[3 * k]) * X + fabs((double)inv[3 * k + 1]) * Y + fabs((double)inv[3 * k + 2]));
        sig += s;
        sig_v += s * sqrt((double)f[3 * k] * f[3 * k] + (double)f[3 * k + 1] * f[3 * k + 1]);
        W += lam_max[k] + s;
        mag += fabs((double)inv[3 * k]) * X + fabs((double)inv[3 * k + 1]) * Y + fabs((double)inv[3 * k + 2]);
    }
    const double slop = 0x1p-40 * (mag + 1.0) * (M + X + Y + 1.0);   // the double evaluation above
    const double E = sqrt(ex * ex + ey * ey) + slop, S = es + sig + slop;
    if (!(S < 0.5)) return 0u;
    // (a) all three w in (0, 1): the point sum w_k v_k / sum w_k lies in the triangle and within dA of p
    const double dA = (sqrt(X * X + Y * Y) * S + E + sig_v) / (1.0 - S);
    // (b) some w outside (0, 1): the computed (dis_x, dis_y) is p's offset to a point of the triangle, up to dB
    const double dB = sqrt(2.0) * u * M + E + sig_v + sqrt(2.0) * g4 * (1.0 + u + W) * M;
    const double q = ceil(fmax(dA, dB) * 0.5 * is * 16.0);
    return q <= 63.0 ? (uint32_t)fmax(q, 1.0) : 0u;
}

// One thread per (batch, face).  Computes the 160-byte record, the exact pixel rectangle
// equivalent to check_border, and (optionally) the reference's faces_info[27].
// Reference: forward_soft_rasterize_inv_cuda_kernel, cuda/soft_rasterize.py:176-236.
static __global__ void __launch_bounds__(256) k_face_setup(const float* __restrict__ faces, const float* __restrict__ textures,
                                                    FaceRec* __restrict__ recs, uint2* __restrict__ rects,
                                                    float* __restrict__ faces_info, int total_faces, int nf,
                                                    int T, int tex_type, int is, float border) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total_faces) return;
    const float* face = faces + (size_t)i * 9;
    float f[9];
#pragma unroll
    for (int k = 0; k < 9; k++) f[k] = __ldg(face + k);

    const float p00 = f[0], p01 = f[1], p10 = f[3], p11 = f[4], p20 = f[6], p21 = f[7];
    float star[9] = {p11 - p21, p20 - p10, p10 * p21 - p20 * p11,
                     p21 - p01, p00 - p20, p20 * p01 - p00 * p21,
                     p01 - p11, p10 - p00, p00 * p11 - p10 * p01};
    float det = p20 * (p01 - p11) + p00 * (p11 - p21) + p10 * (p21 - p01);
    det = det > 0.f ? fmaxf(det, 1e-10f) : fminf(det, -1e-10f);

    FaceRec r;
#pragma unroll
    for (int k = 0; k < 9; k++) r.inv[k] = star[k] / det;
#pragma unroll
    for (int k = 0; k < 9; k++) r.v[k] = f[k];
    float sym[9];
#pragma unroll
    for (int j = 0; j < 3; j++)
#pragma unroll
        for (int k = 0; k < 3; k++) sym[j * 3 + k] = f[j * 3 + 0] * f[k * 3 + 0] + f[j * 3 + 1] * f[k * 3 + 1] + 1.f;
#pragma unroll
    for (int k = 0; k < 3; k++)
#pragma unroll
        for (int j = 0; j < 3; j++) r.a0[3 * k + j] = sym[3 * k + j] - sym[3 * ((k + 1) % 3) + j];

    uint32_t flags = 0;
    {
        const float px[3] = {p00, p10, p20}, py[3] = {p01, p11, p21};
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const int k1 = (k + 1) % 3, k2 = (k + 2) % 3;
            if (flags == 0 && (px[k1] - px[k]) * (px[k2] - px[k]) + (py[k1] - py[k]) * (py[k2] - py[k]) < 0.f)
                flags = 1u << k;
        }
    }
    // check_face_frontside (:37-40)
    if ((f[7] - f[1]) * (f[3] - f[0]) < (f[4] - f[1]) * (f[6] - f[0])) flags |= 8u;
    // refined reciprocals of the per-face denominators (exact_math.cuh).  A face whose inverse is not finite (a NaN or
    // infinite vertex) gets no z bits, so that clip_and_z sends its pairs to the guarded body (NaN weights)
    bool inv_finite = true;
#pragma unroll
    for (int k = 0; k < 9; k++) inv_finite = inv_finite && isfinite(r.inv[k]);
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float z = f[3 * k + 2];
        const float den = r.a0[3 * k + k] - r.a0[3 * k + (k + 1) % 3];
        r.rz[k] = rcp_refined(z);
        r.rden[k] = rcp_refined(den);
        if (midrange(z) && inv_finite) flags |= 16u << k;
        if (midrange(den)) flags |= 128u << k;
    }
    r.face_id = (uint32_t)(i % nf);
#pragma unroll
    for (int k = 0; k < 3; k++) r.col[k] = (T == 1 && tex_type == 0) ? __ldg(textures + (size_t)i * 3 + k) : 0.f;

    // check_border (:28-34) as an exact pixel rectangle
    const float xhi = fmaxf(fmaxf(f[0], f[3]), f[6]) + border;
    const float xlo = fminf(fminf(f[0], f[3]), f[6]) - border;
    const float yhi = fmaxf(fmaxf(f[1], f[4]), f[7]) + border;
    const float ylo = fminf(fminf(f[1], f[4]), f[7]) - border;
    int x0 = first_not_below(xlo, is), x1 = last_not_above(xhi, is);
    const int y0 = first_not_below(ylo, is), y1 = last_not_above(yhi, is);
    int r0 = is - 1 - y1, r1 = is - 1 - y0;  // row = is-1-yi (:280)
    if (x0 > x1 || r0 > r1) { x0 = 1; x1 = 0; r0 = 1; r1 = 0; }
    else if ((flags & 0x3f0u) == 0x3f0u)   // reach-cull margin, bits 10-15 (the forward's euclidean lane masks)
        flags |= reach_margin_q(f, r.inv, b200r_pix_coord(x0, is), b200r_pix_coord(x1, is), b200r_pix_coord(is - 1 - r1, is),
                                b200r_pix_coord(is - 1 - r0, is), is) << 10;
    r.flags = flags;
    r.rect_x = (uint32_t)x0 | ((uint32_t)x1 << 16);
    r.rect_r = (uint32_t)r0 | ((uint32_t)r1 << 16);

    // 160-byte record as 10 x 16-byte stores
    const uint4* src = reinterpret_cast<const uint4*>(&r);
    uint4* dst = reinterpret_cast<uint4*>(recs + i);
#pragma unroll
    for (int k = 0; k < B200R_REC_UINT4; k++) dst[k] = src[k];
    rects[i] = make_uint2(r.rect_x, r.rect_r);

    if (faces_info != nullptr) {
        float* fi = faces_info + (size_t)i * 27;
#pragma unroll
        for (int k = 0; k < 9; k++) fi[k] = r.inv[k];
#pragma unroll
        for (int k = 0; k < 9; k++) fi[9 + k] = sym[k];
#pragma unroll
        for (int k = 0; k < 3; k++) fi[18 + k] = ((flags >> k) & 1u) ? 1.f : 0.f;
#pragma unroll
        for (int k = 21; k < 27; k++) fi[k] = 0.f;
    }
}

__device__ __forceinline__ bool rect_overlaps(uint2 rc, int x0, int x1, int r0, int r1) {
    const int fx0 = (int)(rc.x & 0xffffu), fx1 = (int)(rc.x >> 16);
    const int fr0 = (int)(rc.y & 0xffffu), fr1 = (int)(rc.y >> 16);
    return fx0 <= x1 && fx1 >= x0 && fr0 <= r1 && fr1 >= r0 && fx0 <= fx1;
}

// Block-wide ORDERED compaction step of a 256-thread (8-warp) block: thread `tid` contributes `cnt` items; returns the
// exclusive prefix over the block (in thread order) and the block total.
__device__ __forceinline__ int block_excl_scan(int cnt, int* s_warp /*[8]*/, int& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += n;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int base = 0, tot = 0;
#pragma unroll
    for (int wi = 0; wi < 8; wi++) {
        const int v = s_warp[wi];
        if (wi < warp) base += v;
        tot += v;
    }
    __syncthreads();
    total = tot;
    return base + incl - cnt;
}
// Same for a 0/1 contribution: one ballot instead of a 5-step shuffle scan.
__device__ __forceinline__ int block_excl_scan_flag(bool flag, int* s_warp /*[8]*/, int& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    const int excl = __popc(bal & ((1u << lane) - 1u));
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int base = 0, tot = 0;
#pragma unroll
    for (int wi = 0; wi < 8; wi++) {
        const int v = s_warp[wi];
        if (wi < warp) base += v;
        tot += v;
    }
    __syncthreads();
    total = tot;
    return base + excl;
}

// Coarse binning, tile-centric and deterministic: CTA (bin, b) scans the face rectangles of
// batch element b in ascending face id and appends the overlapping ids, in order, to its
// list.  Replaces TriangleBoundingBoxKernel + RasterizeCoarseCudaKernel
// (cuda/soft_rasterize_coarse_to_fine.py:96-280) whose per-bin order is race-dependent and
// whose fixed-capacity bins silently overflow; here the lists grow chunk by chunk out of a shared
// pool (a bin that finds the pool exhausted is flagged and its blocks filter the whole face list
// instead -- nothing is dropped) and the test is the exact check_border rectangle.
#define B200R_COARSE_PER_THREAD 4
#define B200R_COST_BUCKETS 64

// log-scale cost bucket, 4 per octave, larger cost -> larger bucket; cost 0 -> bucket 0
__device__ __forceinline__ int cost_bucket(int cost) {
    if (cost <= 0) return 0;
    const int lg = 31 - __clz(cost);                       // floor(log2)
    const int frac = lg >= 2 ? ((cost >> (lg - 2)) & 3) : 0;  // next two bits
    const int bkt = 1 + lg * 4 + frac;
    return bkt < B200R_COST_BUCKETS ? bkt : B200R_COST_BUCKETS - 1;
}

// Union rectangle of every run of 256 consecutive faces (CTA (chunk, b)).  Mesh faces that are
// close in index are close on screen, so k_coarse_bin can discard most runs against its bin
// with one test instead of scanning them.  An empty union is stored as (1, 0) like an empty rect.
static __global__ void __launch_bounds__(256) k_chunk_rects(const uint2* __restrict__ rects, uint2* __restrict__ chunk_rects, int nf) {
    __shared__ int s_red[4][8];
    const int f = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
    int x0 = 0xffff, x1 = -1, r0 = 0xffff, r1 = -1;
    if (f < nf) {
        const uint2 rc = __ldg(rects + (size_t)b * nf + f);
        const int fx0 = (int)(rc.x & 0xffffu), fx1 = (int)(rc.x >> 16), fr0 = (int)(rc.y & 0xffffu), fr1 = (int)(rc.y >> 16);
        if (fx0 <= fx1 && fr0 <= fr1) { x0 = fx0; x1 = fx1; r0 = fr0; r1 = fr1; }
    }
    x0 = __reduce_min_sync(0xffffffffu, x0); x1 = __reduce_max_sync(0xffffffffu, x1);
    r0 = __reduce_min_sync(0xffffffffu, r0); r1 = __reduce_max_sync(0xffffffffu, r1);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s_red[0][warp] = x0; s_red[1][warp] = x1; s_red[2][warp] = r0; s_red[3][warp] = r1; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; w++) {
            x0 = min(x0, s_red[0][w]); x1 = max(x1, s_red[1][w]);
            r0 = min(r0, s_red[2][w]); r1 = max(r1, s_red[3][w]);
        }
        uint2 out = make_uint2(1u, 1u);  // empty: x0 = 1 > x1 = 0
        if (x0 <= x1 && r0 <= r1) out = make_uint2((uint32_t)x0 | ((uint32_t)x1 << 16), (uint32_t)r0 | ((uint32_t)r1 << 16));
        chunk_rects[(size_t)b * gridDim.x + blockIdx.x] = out;
    }
}

static __global__ void __launch_bounds__(256) k_coarse_bin(const uint2* __restrict__ rects, const uint2* __restrict__ chunk_rects,
                                                    int* __restrict__ coarse_cnt, int* __restrict__ chunk_table,
                                                    int* __restrict__ coarse_pool, int* __restrict__ pool_cursor,
                                                    int chunks_per_bin, int pool_chunks, int* __restrict__ tile_cost,
                                                    int* __restrict__ cost_hist, int nf, int is,
                                                    int coarse_px, int ncs, int ntx, int nty) {
    constexpr int tw = B200R_BLOCK_W, th = B200R_BLOCK_H;   // cost per forward block
    __shared__ int s_warp[8];
    __shared__ int s_hist[B200R_COST_BUCKETS];
    __shared__ int s_cost[2048];  // blocks of this bin: (coarse_px/tw) * (coarse_px/th) <= 32 * 64 (256 px bins)
    __shared__ int s_overflow;
    __shared__ int s_chunk[4];    // [0]: the chunk the list currently ends in; [1..3]: chunks allocated for the current pass
    __shared__ int s_hits[256];   // passes of the current group of 256 that touch the bin, ascending
    const int bin = blockIdx.x, b = blockIdx.y;
    const int bx = bin % ncs, by = bin / ncs;
    const int x0 = bx * coarse_px, x1 = min(is, x0 + coarse_px) - 1;
    const int r0 = by * coarse_px, r1 = min(is, r0 + coarse_px) - 1;
    const int tpbx = coarse_px / tw, tpby = coarse_px / th;  // tiles per bin along x / y
    for (int i = threadIdx.x; i < tpbx * tpby; i += 256) s_cost[i] = 0;
    if (threadIdx.x == 0) s_overflow = 0;
    __syncthreads();
    const uint2* rc = rects + (size_t)b * nf;
    int* tbl = chunk_table + ((size_t)b * ncs * ncs + bin) * chunks_per_bin;   // pool chunk of list positions [512 k, 512 k + 512)
    int n_out = 0;
    bool overflow = false;   // the pool ran out: the list is abandoned (coarse_cnt = -1), the cost model keeps counting
    const bool vec_ok = (reinterpret_cast<uintptr_t>(rc) & 15) == 0;  // (b*nf) even
    const int n_chunks = (nf + 255) / 256;
    const uint2* crc = chunk_rects + (size_t)b * n_chunks;
    constexpr int PT = B200R_COARSE_PER_THREAD;
    const int n_pass = (nf + 256 * PT - 1) / (256 * PT);   // one pass = 256 threads x 4 consecutive faces = 4 runs of 256

    // the 4 rectangles a thread owns in pass `pass` (empty rectangles behind the last face)
    auto load_pass = [&](int pass, uint2 (&rr)[PT]) {
        const int first = pass * 256 * PT + threadIdx.x * PT;
        if (vec_ok && first + PT <= nf) {
            const uint4 a = __ldg(reinterpret_cast<const uint4*>(rc + first));
            const uint4 c = __ldg(reinterpret_cast<const uint4*>(rc + first + 2));
            rr[0] = make_uint2(a.x, a.y); rr[1] = make_uint2(a.z, a.w);
            rr[2] = make_uint2(c.x, c.y); rr[3] = make_uint2(c.z, c.w);
        } else {
#pragma unroll
            for (int u = 0; u < PT; u++) rr[u] = (first + u < nf) ? __ldg(rc + first + u) : make_uint2(1u, 1u);
        }
    };

    for (int g = 0; g < n_pass; g += 256) {
        // ---- which of the passes g .. g + 255 touch the bin: one thread per pass tests the union rectangles of its four
        // runs (k_chunk_rects), all at once -- consecutive faces are close on screen, so most passes miss (31 of 39 at C3)
        // and testing them one after the other cost a dependent L2 round trip each
        const int my_pass = g + threadIdx.x;
        bool hit = false;
        if (my_pass < n_pass) {
#pragma unroll
            for (int u = 0; u < PT; u++) {
                const int c = my_pass * PT + u;
                if (c < n_chunks && rect_overlaps(__ldg(crc + c), x0, x1, r0, r1)) hit = true;
            }
        }
        int n_hit;
        const int hpos = block_excl_scan_flag(hit, s_warp, n_hit);
        if (hit) s_hits[hpos] = my_pass;
        __syncthreads();

        // ---- the hitting passes in ascending order; the next pass's rectangles are in flight while this one is scanned
        uint2 nxt[PT];
        if (n_hit > 0) load_pass(s_hits[0], nxt);
        for (int i = 0; i < n_hit; i++) {
            const int first = s_hits[i] * 256 * PT + threadIdx.x * PT;
            uint2 rr[PT];
#pragma unroll
            for (int u = 0; u < PT; u++) rr[u] = nxt[u];
            if (i + 1 < n_hit) load_pass(s_hits[i + 1], nxt);
            uint32_t mask = 0;
#pragma unroll
            for (int u = 0; u < PT; u++)
                if (rect_overlaps(rr[u], x0, x1, r0, r1)) mask |= 1u << u;
            int total;
            int off = n_out + block_excl_scan(__popc(mask), s_warp, total);
            if (!overflow) {
                // chunks for list positions [n_out, n_out + total): the list so far ends inside chunk number have - 1
                const int have = (n_out + B200R_LIST_CHUNK - 1) >> B200R_LIST_CHUNK_SHIFT;
                const int need = ((n_out + total + B200R_LIST_CHUNK - 1) >> B200R_LIST_CHUNK_SHIFT) - have;
                if (need > 0) {   // uniform for the CTA; a pass lists <= 1024 faces, i.e. need <= 3
                    if (threadIdx.x == 0) {
                        const int c0 = atomicAdd(pool_cursor, need);
                        if (c0 + need > pool_chunks) s_overflow = 1;
                        else for (int k = 0; k < need; k++) { tbl[have + k] = c0 + k; s_chunk[1 + k] = c0 + k; }
                    }
                    __syncthreads();
                    overflow = s_overflow != 0;
                }
                if (!overflow) {
#pragma unroll
                    for (int u = 0; u < PT; u++)
                        if (mask & (1u << u)) {
                            const int c = s_chunk[(off >> B200R_LIST_CHUNK_SHIFT) - have + 1];   // have - 1 = the partly filled chunk
                            coarse_pool[((size_t)c << B200R_LIST_CHUNK_SHIFT) | (size_t)(off & (B200R_LIST_CHUNK - 1))] = first + u;
                            off++;
                        }
                    if (need > 0) {
                        __syncthreads();   // every writer has read s_chunk
                        if (threadIdx.x == 0) s_chunk[0] = s_chunk[need];
                    }
                }
            }
            n_out += total;
            // ---- cost model: faces per fine tile of the bin as a 2-D difference array -- 4 shared-memory atomics per
            // listed face at the corners of its tile range, row / column prefix sums at the end.  (Adding the clipped
            // area to every overlapped tile costs ~12 atomics per face with 32-way conflicts.)  The rectangle is still
            // in registers here; a separate pass over the finished list re-fetched id and rectangle of every entry.
#pragma unroll
            for (int u = 0; u < PT; u++)
                if (mask & (1u << u)) {
                    const int fx0 = max((int)(rr[u].x & 0xffffu), x0), fx1 = min((int)(rr[u].x >> 16), x1);
                    const int fr0 = max((int)(rr[u].y & 0xffffu), r0), fr1 = min((int)(rr[u].y >> 16), r1);
                    const int ty_first = (fr0 - r0) / th, ty_end = (fr1 - r0) / th + 1;
                    const int tx_first = (fx0 - x0) / tw, tx_end = (fx1 - x0) / tw + 1;
                    atomicAdd(&s_cost[ty_first * tpbx + tx_first], 1);
                    if (tx_end < tpbx) atomicAdd(&s_cost[ty_first * tpbx + tx_end], -1);
                    if (ty_end < tpby) {
                        atomicAdd(&s_cost[ty_end * tpbx + tx_first], -1);
                        if (tx_end < tpbx) atomicAdd(&s_cost[ty_end * tpbx + tx_end], 1);
                    }
                }
        }
        __syncthreads();   // s_hits is rewritten by the next group
    }
    __syncthreads();
    for (int ty = threadIdx.x; ty < tpby; ty += 256) {  // along x
        int acc = 0;
        for (int tx = 0; tx < tpbx; tx++) { acc += s_cost[ty * tpbx + tx]; s_cost[ty * tpbx + tx] = acc; }
    }
    __syncthreads();
    for (int tx = threadIdx.x; tx < tpbx; tx += 256) {  // along y
        int acc = 0;
        for (int ty = 0; ty < tpby; ty++) { acc += s_cost[ty * tpbx + tx]; s_cost[ty * tpbx + tx] = acc; }
    }
    if (threadIdx.x == 0) coarse_cnt[b * ncs * ncs + bin] = overflow ? -1 : n_out;
    if (threadIdx.x < B200R_COST_BUCKETS) s_hist[threadIdx.x] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < tpbx * tpby; i += 256) {
        const int gtx = bx * tpbx + i % tpbx, gty = by * tpby + i / tpbx;
        if (gtx < ntx && gty < nty) {
            const int c = s_cost[i] * tw * th;  // ~ (pixel, face) pairs
            tile_cost[(size_t)b * ntx * nty + gty * ntx + gtx] = c;
            atomicAdd(&s_hist[cost_bucket(c)], 1);
        }
    }
    __syncthreads();  // one global atomic per (CTA, non-empty bucket), not one per tile
    if (threadIdx.x < B200R_COST_BUCKETS && s_hist[threadIdx.x] > 0) atomicAdd(&cost_hist[threadIdx.x], s_hist[threadIdx.x]);
}

// Orders all forward blocks by descending cost bucket (longest-processing-time-first for the
// persistent raster grid): each queue entry takes the bucket of its own block's cost (k_coarse_bin),
// so a silhouette block that is long-running starts early even when its neighbours are cheap.
// hist[] counts blocks per bucket (complete after k_coarse_bin).  Block-aggregated reservation:
// one global atomic per (CTA, bucket) instead of one per block.  Bucket 0 (no rectangle touches the block) comes last:
// tile_order[0, total - hist[0]) are the blocks with faces to shade, tile_order[total - hist[0], total) the empty
// ones, which k_softras_forward stores on the side of the shaded blocks.
static __global__ void __launch_bounds__(256) k_tile_order(const int* __restrict__ tile_cost, const int* __restrict__ hist,
                                                           int* __restrict__ cursor, uint2* __restrict__ tile_order,
                                                           int B, int fntx, int fnty) {
    __shared__ int s_start[B200R_COST_BUCKETS];
    __shared__ int s_cnt[B200R_COST_BUCKETS];
    __shared__ int s_base[B200R_COST_BUCKETS];
    if (threadIdx.x < B200R_COST_BUCKETS) s_cnt[threadIdx.x] = 0;
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int k = B200R_COST_BUCKETS - 1; k >= 0; k--) { s_start[k] = acc; acc += hist[k]; }
    }
    __syncthreads();
    const int total = B * fntx * fnty;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    int bkt = 0, lrank = 0;
    uint2 entry = make_uint2(0u, 0u);
    if (t < total) {
        const int b = t / (fntx * fnty), tt = t % (fntx * fnty);
        entry.x = (uint32_t)(tt % fntx) | ((uint32_t)(tt / fntx) << 16);
        bkt = cost_bucket(tile_cost[t]);   // [B][fnty][fntx], the order of t
        lrank = atomicAdd(&s_cnt[bkt], 1);
        entry.y = (uint32_t)b | (bkt == 0 ? 0x80000000u : 0u);   // bucket 0 <=> no rectangle touches the block (exact count)
    }
    __syncthreads();
    if (threadIdx.x < B200R_COST_BUCKETS && s_cnt[threadIdx.x] > 0)
        s_base[threadIdx.x] = atomicAdd(&cursor[threadIdx.x], s_cnt[threadIdx.x]);
    __syncthreads();
    if (t < total) tile_order[s_start[bkt] + s_base[bkt] + lrank] = entry;
}

}  // namespace b200r
