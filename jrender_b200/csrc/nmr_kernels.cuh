// nmr_kernels.cuh -- Neural Mesh Renderer (dr_type='n3mr') hard rasterizer, forward + backward.
//
// Replaces the reference kernels of jrender/renderer/dr/n3mr/cuda/rasterize.py:
//   K7  forward_face_index_map_cuda_kernel   :30-164   thread per FACE scanning its bounding box,
//                                                       per-pixel atomicCAS spin lock for the z test
//   K8  forward_texture_sampling_cuda_kernel :227-298
//   K9  backward_pixel_map_cuda_kernel       :351-610  thread per face, serial scans
//   K10 backward_textures_cuda_kernel        :659-694
//   K11 backward_depth_map_cuda_kernel       :738-788
//
// Design: the forward is a face-parallel z-buffer pass (a warp per face over its bounding box, one 64-bit atomicMin
// of (depth, face id) per covered pixel: lock-free and deterministic -- lowest face id wins equal depth; the reference's
// winner is race-dependent) followed by a per-pixel resolve pass that fuses K7's map writes with K8: the pixel recomputes
// its winning face's weights, samples the texture and writes every map once.  K9 keeps the reference's per-face edge walk but gives a WARP to each
// face so that the long "out" scans (up to image_size pixels each) run 32 pixels at a time on
// coalesced rows.  Maps keep the kernels' orientation [B, yi, xi] with yi up.
#pragma once
#include "common.cuh"
#include "exact_math.cuh"
#include "softras_setup.cuh"

namespace b200r {

struct NmrParams {
    int B, nf, ts, is;
    float near_, far_, eps;
    float bg[3];
    int return_rgb, return_alpha, return_depth;
};

// Per-face quantities of K7 (:59-105), computed identically wherever a face is touched (z-buffer pass, resolve pass):
// back-face flag, pixel-space inverse with the UNCLAMPED determinant, integer bounding box, reciprocals of the depths.
struct NmrFace {
    float v[9];        // NDC x, y and z per vertex
    float inv[9];      // pixel-space face_inv (:75-87)
    float rz[3];       // rcp_refined(z_k)
    uint32_t zsafe;    // bit k: midrange(z_k)
    int ix_min, ix_max, iy_min, iy_max;   // :102-105, yi up; empty when culled
};

__device__ __forceinline__ void nmr_face_setup(const float* __restrict__ face, int is, NmrFace& r) {
    float f[9];
#pragma unroll
    for (int k = 0; k < 9; k++) f[k] = __ldg(face + k);
#pragma unroll
    for (int k = 0; k < 9; k++) r.v[k] = f[k];
    r.zsafe = 0;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        r.rz[k] = rcp_refined(f[3 * k + 2]);
        if (midrange(f[3 * k + 2])) r.zsafe |= 1u << k;
    }
    float p[3][2];
#pragma unroll
    for (int num = 0; num < 3; num++)
#pragma unroll
        for (int dim = 0; dim < 2; dim++) p[num][dim] = 0.5f * (f[3 * num + dim] * is + is - 1);  // :70 (0.5*x exact)
    const float fi[9] = {p[1][1] - p[2][1], p[2][0] - p[1][0], p[1][0] * p[2][1] - p[2][0] * p[1][1],
                         p[2][1] - p[0][1], p[0][0] - p[2][0], p[2][0] * p[0][1] - p[0][0] * p[2][1],
                         p[0][1] - p[1][1], p[1][0] - p[0][0], p[0][0] * p[1][1] - p[1][0] * p[0][1]};
    const float den = (p[2][0] * (p[0][1] - p[1][1]) + p[0][0] * (p[1][1] - p[2][1]) + p[1][0] * (p[2][1] - p[0][1]));
#pragma unroll
    for (int k = 0; k < 9; k++) r.inv[k] = fi[k] / den;
    float x_min = (float)is, y_min = (float)is, x_max = 0.f, y_max = 0.f;
#pragma unroll
    for (int num = 0; num < 3; num++) {
        if (p[num][0] < x_min) x_min = p[num][0];
        if (p[num][0] > x_max) x_max = p[num][0];
        if (p[num][1] < y_min) y_min = p[num][1];
        if (p[num][1] > y_max) y_max = p[num][1];
    }
    r.ix_min = max(0, (int)x_min); r.ix_max = min(is - 1, (int)x_max);
    r.iy_min = max(0, (int)y_min); r.iy_max = min(is - 1, (int)y_max);
    const bool back = (f[7] - f[1]) * (f[3] - f[0]) < (f[4] - f[1]) * (f[6] - f[0]);  // :63
    if (back || r.ix_min > r.ix_max || r.iy_min > r.iy_max) { r.ix_min = 1; r.ix_max = 0; r.iy_min = 1; r.iy_max = 0; }
}

// K7's per-(face, pixel) body (:108-136): NDC inside test, clamped / normalised barycentric weights, depth.  Returns
// false when the pixel is outside the face or the depth fails the near / far test; a NaN depth is rejected too (the
// reference lets it past :136 but `zp < depth` at :146 is then false: it never wins a pixel).
__device__ __forceinline__ bool nmr_face_pixel(const NmrFace& r, int xi, int yi, int is, float near_, float far_,
                                               float& w0, float& w1, float& w2, float& zp) {
    const float xp = b200r_pix_coord(xi, is), yp = b200r_pix_coord(yi, is);   // :110-111
    const float* f = r.v;
    if (((yp - f[1]) * (f[3] - f[0]) < (xp - f[0]) * (f[4] - f[1])) ||
        ((yp - f[4]) * (f[6] - f[3]) < (xp - f[3]) * (f[7] - f[4])) ||
        ((yp - f[7]) * (f[0] - f[6]) < (xp - f[6]) * (f[1] - f[7])))
        return false;                                                          // :113-116
    const float fxi = (float)xi, fyi = (float)yi;
    const float* inv = r.inv;
    w0 = inv[0] * fxi + inv[1] * fyi + inv[2];   // :121-123
    w1 = inv[3] * fxi + inv[4] * fyi + inv[5];
    w2 = inv[6] * fxi + inv[7] * fyi + inv[8];
    w0 = fminf(fmaxf(w0, 0.f), 1.f);              // :128
    w1 = fminf(fmaxf(w1, 0.f), 1.f);
    w2 = fminf(fmaxf(w2, 0.f), 1.f);
    const float w_sum = ((0.f + w0) + w1) + w2;  // :126-129
    if (w_sum != 1.f) {
        const float rr = rcp_refined(w_sum);
        const bool safe = midrange(w_sum);
        w0 = fast_div(w0, w_sum, rr, safe);       // :132
        w1 = fast_div(w1, w_sum, rr, safe);
        w2 = fast_div(w2, w_sum, rr, safe);
    }
    zp = 1.f / (fast_div(w0, f[2], r.rz[0], (r.zsafe & 1u) != 0) + fast_div(w1, f[5], r.rz[1], (r.zsafe & 2u) != 0) +
                fast_div(w2, f[8], r.rz[2], (r.zsafe & 4u) != 0));   // :135
    if (zp <= near_ || far_ <= zp) return false;                     // :136
    return zp < far_;                                                 // NaN
}

// float -> unsigned with the same order (negative depths are possible when `near` is negative).  -0 is mapped to +0
// first: the oracle's `zp < depth` treats them as equal, so a tie between a -0 and a +0 face goes to the lower id.
__device__ __forceinline__ uint32_t nmr_order_bits(float z) {
    const uint32_t u = __float_as_uint(z == 0.f ? 0.f : z);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// K7, pass 1 -- face-parallel z-buffer.  The reference gives a THREAD to every face and serialises pixels behind an
// atomicCAS spin lock (:138-160, the winner of equal depths is whoever gets the lock first); the first version here was
// tile-centric (every pixel of a 16x16 tile tested every face binned to the tile: ~100 bounding-box tests per pixel for
// the 2-pixel triangles of the 39 200-face mesh, plus a binning pass).  Now every covered pixel of
// every face does ONE 64-bit atomicMin of (depth order bits << 32 | face id) into the z-buffer: lock-free, and
// deterministic -- lowest depth, then lowest face id, exactly the oracle's tie rule.  A thread sets its face up and walks a
// small bounding box itself (the per-face set-up with its nine divisions is most of the work for small faces: 32 faces
// per warp, not one); faces with a bounding box above kNmrSerialBox pixels are then taken one at a time by the whole warp,
// lanes striding over the box (any size).
constexpr int kNmrSerialBox = 32;

__device__ __forceinline__ void nmr_zbuffer_pixel(const NmrFace& r, int xi, int yi, int is, float near_, float far_, int fn,
                                                  unsigned long long* __restrict__ zb) {
    float w0, w1, w2, zp;
    if (!nmr_face_pixel(r, xi, yi, is, near_, far_, w0, w1, w2, zp)) return;
    atomicMin(zb + (size_t)yi * is + xi, ((unsigned long long)nmr_order_bits(zp) << 32) | (unsigned)fn);
}

__global__ void __launch_bounds__(256)
k_nmr_zbuffer(const float* __restrict__ faces, unsigned long long* __restrict__ zbuf, int B, int nf, int is, float near_, float far_) {
    const int lane = threadIdx.x & 31;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long total = (long)B * nf;
    NmrFace r;
    int npx = 0, bw = 1;
    if (i < total) {
        nmr_face_setup(faces + i * 9, is, r);
        if (r.ix_min <= r.ix_max) {
            bw = r.ix_max - r.ix_min + 1;
            npx = bw * (r.iy_max - r.iy_min + 1);
        }
    }
    const int b = (int)((i < total ? i : 0) / nf), fn = (int)((i < total ? i : 0) % nf);
    if (npx > 0 && npx <= kNmrSerialBox) {
        unsigned long long* zb = zbuf + (size_t)b * is * is;
        for (int j = 0; j < npx; j++) nmr_zbuffer_pixel(r, r.ix_min + j % bw, r.iy_min + j / bw, is, near_, far_, fn, zb);
    }
    // large faces: the warp takes them one at a time (set-up recomputed by every lane: cheaper than 22 shuffles)
    for (unsigned m = __ballot_sync(0xffffffffu, npx > kNmrSerialBox); m != 0u; m &= m - 1u) {
        const int src = __ffs(m) - 1;
        const long fi = i - lane + src;
        NmrFace q;
        nmr_face_setup(faces + fi * 9, is, q);
        const int qb = (int)(fi / nf), qfn = (int)(fi % nf);
        const int qw = q.ix_max - q.ix_min + 1, qn = qw * (q.iy_max - q.iy_min + 1);
        unsigned long long* zb = zbuf + (size_t)qb * is * is;
        for (int j = lane; j < qn; j += 32) nmr_zbuffer_pixel(q, q.ix_min + j % qw, q.iy_min + j / qw, is, near_, far_, qfn, zb);
    }
}

// K7 pass 2 + K8 + background / alpha (n3mr.py:135-148) -- thread per pixel: reads the winning face id, recomputes its
// weights and depth with the very same code the z-buffer pass ran (same bits), samples the texture and writes every map
// once (replaces the fills / memsets of :176-184, :311-313).  ~100 bytes written per pixel: this pass runs at HBM speed.
__global__ void __launch_bounds__(256)
k_nmr_resolve(const NmrParams P, const unsigned long long* __restrict__ zbuf, const float* __restrict__ faces,
              const float* __restrict__ textures, int* __restrict__ face_index_map, float* __restrict__ weight_map,
              float* __restrict__ depth_map, float* __restrict__ rgb_map, float* __restrict__ alpha_map,
              int* __restrict__ sampling_index_map, float* __restrict__ sampling_weight_map, float* __restrict__ face_inv_map) {
    const int is = P.is, nf = P.nf;
    const size_t i1 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i1 >= (size_t)P.B * is * is) return;
    const int b = (int)(i1 / ((size_t)is * is));
    const int rem = (int)(i1 - (size_t)b * is * is);
    const int yi = rem / is, xi = rem - yi * is;
    const unsigned long long key = zbuf[i1];
    float depth = P.far_;   // thrust::fill(depth_map, far) :181-182
    int best = -1;          // thrust::fill(face_index_map, -1) :176-177
    float bw0 = 0.f, bw1 = 0.f, bw2 = 0.f;
    NmrFace r;
    if (key != ~0ull) {
        best = (int)(unsigned)(key & 0xffffffffull);
        nmr_face_setup(faces + ((size_t)b * nf + best) * 9, is, r);
        nmr_face_pixel(r, xi, yi, is, P.near_, P.far_, bw0, bw1, bw2, depth);
    }
    face_index_map[i1] = best;
    weight_map[i1 * 3 + 0] = bw0;
    weight_map[i1 * 3 + 1] = bw1;
    weight_map[i1 * 3 + 2] = bw2;
    depth_map[i1] = depth;
    if (P.return_alpha) alpha_map[i1] = best >= 0 ? 1.f : 0.f;   // n3mr.py:145-148
    if (P.return_depth) {
#pragma unroll
        for (int k = 0; k < 9; k++) face_inv_map[i1 * 9 + k] = best >= 0 ? r.inv[k] : 0.f;   // :152-156
    }
    if (P.return_rgb) {
        float px0 = P.bg[0], px1 = P.bg[1], px2 = P.bg[2];   // forward_background, n3mr.py:135-143
        int sidx[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        float sw[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (best >= 0) {  // K8 :248-297
            const int ts = P.ts;
            const float* texture = textures + ((size_t)b * nf + best) * ts * ts * ts * 3;
            const float wk[3] = {bw0, bw1, bw2};
            float tif[3];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                float v = wk[k] * (ts - 1) * (depth / r.v[3 * k + 2]);
                v = fmaxf(v, 0.f);
                v = fminf(v, ts - 1 - P.eps);
                tif[k] = v;
            }
            float np0 = 0.f, np1 = 0.f, np2 = 0.f;
#pragma unroll
            for (int pn = 0; pn < 8; pn++) {
                float w = 1.f;
                int tii[3];
#pragma unroll
                for (int k = 0; k < 3; k++) {
                    const int base_i = (int)tif[k];
                    if (((pn >> k) & 1) == 0) { w *= 1 - (tif[k] - base_i); tii[k] = base_i; }
                    else { w *= tif[k] - base_i; tii[k] = base_i + 1; }
                }
                const int isc = tii[0] * ts * ts + tii[1] * ts + tii[2];
                // texture_size 1: ts - 1 - eps < 0 and the "+1" taps leave the face's block; the reference reads whatever
                // follows (next faces' texels; past the tensor for the last faces).  Taps inside the tensor are read
                // likewise, taps past it give 0.
                const size_t tap = ((size_t)b * nf + best) * ts * ts * ts + (size_t)isc;
                if (isc >= 0 && tap < (size_t)P.B * nf * ts * ts * ts) {
                    np0 += w * __ldg(texture + isc * 3 + 0);
                    np1 += w * __ldg(texture + isc * 3 + 1);
                    np2 += w * __ldg(texture + isc * 3 + 2);
                }
                sidx[pn] = isc;
                sw[pn] = w;
            }
            // rgb * mask + (1 - mask) * background with mask == 1
            px0 = np0 * 1.f + 0.f * P.bg[0];
            px1 = np1 * 1.f + 0.f * P.bg[1];
            px2 = np2 * 1.f + 0.f * P.bg[2];
        } else {
            px0 = 0.f * 0.f + 1.f * P.bg[0];
            px1 = 0.f * 0.f + 1.f * P.bg[1];
            px2 = 0.f * 0.f + 1.f * P.bg[2];
        }
        rgb_map[i1 * 3 + 0] = px0;
        rgb_map[i1 * 3 + 1] = px1;
        rgb_map[i1 * 3 + 2] = px2;
        int4* si = reinterpret_cast<int4*>(sampling_index_map + i1 * 8);
        si[0] = make_int4(sidx[0], sidx[1], sidx[2], sidx[3]);
        si[1] = make_int4(sidx[4], sidx[5], sidx[6], sidx[7]);
        float4* sv = reinterpret_cast<float4*>(sampling_weight_map + i1 * 8);
        sv[0] = make_float4(sw[0], sw[1], sw[2], sw[3]);
        sv[1] = make_float4(sw[4], sw[5], sw[6], sw[7]);
    }
}

// ---------------------------------------------------------------- K9 prologue: packed pixel records
// K9's scans evaluate, for long pixel runs (along x for axis 1, along y for axis 0),
//     diff_grad = sum_k (map_k - ref_k) * grad_k            (k over r, g, b and/or alpha; ref = the sample's in / out pixel)
// which is  A - sum_k ref_k * grad_k  with the per-pixel moment  A = sum_k map_k * grad_k.  This kernel stores (A, grad)
// per pixel -- 16 bytes for rgb (A, gr, gg, gb), 8 for alpha (A, ga), 32 for both -- twice: row-major (ph[b][y][x]) and
// column-major (pv[b][x][y]), so both scan directions read consecutive records.  (Reading the four maps separately, and
// columns with a stride of a whole image row, made the first version of the backward 20x slower than its instruction
// count warrants; 32-byte (rgb, grad, alpha, grad) records were the second version: the scans then ran at the L1's
// bandwidth, which this halves.)  32x32 tile transpose through shared memory.
// MODE 1: rgb, 2: alpha, 3: both.  FL = floats per record (4, 2, 8).
template <int MODE>
struct K9Rec {
    static constexpr int FL = (MODE == 1) ? 4 : ((MODE == 2) ? 2 : 8);
};

template <int MODE>
__global__ void __launch_bounds__(256)
k_nmr_pack(const float* __restrict__ rgb_map, const float* __restrict__ alpha_map, const float* __restrict__ grad_rgb_map,
           const float* __restrict__ grad_alpha_map, float* __restrict__ ph, float* __restrict__ pv, int is) {
    constexpr int FL = K9Rec<MODE>::FL;
    __shared__ float s[32][33][FL];
    const int b = blockIdx.z, x0 = blockIdx.x * 32, y0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const size_t img = (size_t)b * is * is;
    for (int r = ty; r < 32; r += 8) {
        const int x = x0 + tx, y = y0 + r;
        float v[FL];
#pragma unroll
        for (int k = 0; k < FL; k++) v[k] = 0.f;
        if (x < is && y < is) {
            const size_t i = img + (size_t)y * is + x;
            float A = 0.f;
            if (MODE & 1) {
                const float g0 = __ldg(grad_rgb_map + i * 3 + 0), g1 = __ldg(grad_rgb_map + i * 3 + 1), g2 = __ldg(grad_rgb_map + i * 3 + 2);
                A = __fmaf_rn(__ldg(rgb_map + i * 3 + 0), g0, A);
                A = __fmaf_rn(__ldg(rgb_map + i * 3 + 1), g1, A);
                A = __fmaf_rn(__ldg(rgb_map + i * 3 + 2), g2, A);
                v[1] = g0; v[2] = g1; v[3] = g2;
            }
            if (MODE & 2) {
                const float ga = __ldg(grad_alpha_map + i);
                A = __fmaf_rn(__ldg(alpha_map + i), ga, A);
                v[(MODE == 2) ? 1 : 4] = ga;
            }
            v[0] = A;
#pragma unroll
            for (int k = 0; k < FL; k++) ph[i * FL + k] = v[k];
        }
#pragma unroll
        for (int k = 0; k < FL; k++) s[r][tx][k] = v[k];
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int x = x0 + r, y = y0 + tx;   // pv[b][x][y] <- pixel (y, x) = s[y - y0][x - x0]
        if (x < is && y < is) {
            const size_t j = img + (size_t)x * is + y;
#pragma unroll
            for (int k = 0; k < FL; k++) pv[j * FL + k] = s[tx][r][k];
        }
    }
}

// ---------------------------------------------------------------- K9: warp per (batch, face)
__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    return v;
}

// 1 / x to 1 ulp (MUFU.RCP).  The edge-scan sums below run in a different order from the
// reference's serial per-face loop anyway (lanes, then a warp reduction), so the terms
// diff_grad / dist are formed with this reciprocal and one FMA instead of an IEEE division:
// <= 1.5 ulp per term, against the 2e-5 relative tolerance of the gradient parity tests.
__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));  // |x| >= eps: never denormal
    return r;
}

__device__ __forceinline__ float k9_sel3(int i, float a, float b, float c) { return i == 0 ? a : (i == 1 ? b : c); }
__device__ __forceinline__ int k9_sel6(int i, const int v[7]) {
    return i == 0 ? v[0] : (i == 1 ? v[1] : (i == 2 ? v[2] : (i == 3 ? v[3] : (i == 4 ? v[4] : v[5]))));
}

// One packed record of k_nmr_pack as every scan holds it: q = (A, gr, gg, gb) for rgb, (A, ga, -, -) for alpha,
// (A, gr, gg, gb) and ga for both.  Lanes without a pixel (`on` false) get a zero record.
template <int MODE>
struct K9Px { float4 q; float ga; };

template <int MODE>
__device__ __forceinline__ K9Px<MODE> k9_load_px(const float* __restrict__ p, bool on) {
    K9Px<MODE> r;
    r.q = make_float4(0.f, 0.f, 0.f, 0.f);
    r.ga = 0.f;
    if (on) {
        if (MODE == 2) { const float2 t = __ldg(reinterpret_cast<const float2*>(p)); r.q.x = t.x; r.q.y = t.y; }
        else r.q = __ldg(reinterpret_cast<const float4*>(p));
        if (MODE == 3) r.ga = __ldg(p + 4);
    }
    return r;
}

// diff_grad = A - sum_k ref_k * grad_k as one fma chain off A (the negations are operand modifiers): one instruction
// fewer per record than forming the sum first.  ref = (r, g, b, alpha) of the sample's in-pixel (outward scan) /
// out-pixel (inward scan).
template <int MODE>
__device__ __forceinline__ float k9_diff(const K9Px<MODE>& c, float r0, float r1, float r2, float ra) {
    if (MODE == 1) return __fmaf_rn(-r2, c.q.w, __fmaf_rn(-r1, c.q.z, __fmaf_rn(-r0, c.q.y, c.q.x)));
    if (MODE == 2) return __fmaf_rn(-ra, c.q.y, c.q.x);
    return __fmaf_rn(-ra, c.ga, __fmaf_rn(-r2, c.q.w, __fmaf_rn(-r1, c.q.z, __fmaf_rn(-r0, c.q.y, c.q.x))));
}

// acc += -d / dist with the reference's per-pixel distance  dist = delta * k + (dist > 0 ? eps : -eps)  (:510/:515)
__device__ __forceinline__ void k9_guarded_term(float d, float delta, float k, float eps, float& acc) {
    float dist = delta * k;
    dist = (0.f < dist) ? dist + eps : dist - eps;
    acc = __fmaf_rn(-d, rcp_approx(dist), acc);
}

// Adds a pass's two running sums to the face's six gradient slots gacc[vertex * 2 + (0: x, 1: y)]: acc0 / acc1 belong
// to vertex pi0 / pi1 of the pass's edge, coordinate (1 - axis).  Compare-and-add keeps gacc in registers.
__device__ __forceinline__ void k9_add_slots(int pass, float acc0, float acc1, float gacc[6]) {
    const int edge = pass >> 1, axis = pass & 1;
    const int g0 = edge * 2 + (1 - axis), g1 = ((edge == 2) ? 0 : edge + 1) * 2 + (1 - axis);
#pragma unroll
    for (int k = 0; k < 6; k++) {
        if (k == g0) gacc[k] += acc0;
        if (k == g1) gacc[k] += acc1;
    }
}

// One line scan of K9 (:486-520 outwards / :556-601 inwards): lanes take consecutive pixels d1_from + lane, + 32, ...
// of the packed row `prow` (k_nmr_pack) and add their  -diff_grad / dist  terms to acc0 / acc1 (only the terms whose
// vertex is off the sample's line: has0 = p[1][0] != d0, has1 = p[0][0] != d0, :508/:513).
//   OWNER  inward scan: only pixels whose face_index_map entry is this face count (:573)
// The loop is kept to one record load and ~20 arithmetic instructions per 32 pixels: pointers and the pixel
// coordinate advance by constants, the `diff_grad <= 0` skip is a select (a NaN still propagates like the reference's
// `continue` would let it), products are fused (sums of ~10^2..10^3 terms, compared at 2e-5 relative).
template <int MODE, bool OWNER>
__device__ __forceinline__ void k9_scan(const float* __restrict__ prow, const int* __restrict__ fim, int fim_stride,
                                        int d1_from, int d1_to, int lane, int fn, float r0, float r1, float r2, float ra,
                                        float d1_cross, float k0, float k1, bool has0, bool has1, float eps,
                                        float& acc0, float& acc1) {
    constexpr int FL = K9Rec<MODE>::FL;
    // offsets inside one image fit 32 bits (is <= 4096: is^2 * FL <= 2^27)
    const float* __restrict__ p = prow + (d1_from + lane) * FL;
    const int* __restrict__ o = OWNER ? fim + (d1_from + lane) * fim_stride : nullptr;
    float d1f = (float)(d1_from + lane);   // exact below 2^24
    int left = d1_to - d1_from - lane;
    // software pipeline: the record (and owner) of trip t + 1 is requested before trip t is evaluated -- one trip's
    // arithmetic is far shorter than an L1 / L2 round trip, and the scan is a chain of dependent trips otherwise
    K9Px<MODE> q = k9_load_px<MODE>(p, left >= 0);
    int own = fn;
    if (OWNER && left >= 0) own = __ldg(o);
    while (left >= 0) {
        const K9Px<MODE> c = q;
        const int cown = own;
        left -= 32;
        p += 32 * FL;
        if (OWNER) o += 32 * fim_stride;   // (pointer arithmetic in 64 bits, the product in 32)
        if (left >= 0) {
            q = k9_load_px<MODE>(p, true);
            if (OWNER) own = __ldg(o);
        }
        const float diff = k9_diff<MODE>(c, r0, r1, r2, ra);
        const bool mine = !OWNER || cown == fn;
        const float d = (mine && !(diff <= 0.f)) ? diff : 0.f;   // :503 / :587 `if (diff_grad <= 0) continue`
        const float delta = d1f - d1_cross;   // (d1 - d1_cross), one rounding like the reference's
        d1f += 32.f;
        if (has0) k9_guarded_term(d, delta, k0, eps, acc0);
        if (has1) k9_guarded_term(d, delta, k1, eps, acc1);
    }
}

// The outward scan (:486-520), specialised: it is 2/3 of K9's instructions and all of its load latency.
//  * Every pixel of an outward scan lies strictly beyond the crossing point (d1_out = floor(d1_cross) + 1 or
//    ceil(d1_cross) - 1, then away from it), so delta = d1 - d1_cross has ONE sign for the whole scan and the reference's
//    per-pixel `dist = (0 < dist) ? dist + eps : dist - eps` (:510/:515) adds a per-scan constant: dist = fma(delta, k, +-eps)
//    (|k| >= 2 / is, so delta * k never underflows; no cancellation, so |dist| >= eps).
//  * Lanes past the end of the scan (only in the last trip pair) evaluate a zero record with delta replaced by `side`
//    (d1_from - d1_cross), so their dist is nonzero and they add exactly 0.  Their own delta would not do: in a scan toward pixel 0 they sit at d1_in
//    and beyond, across the crossing, where fma(delta, k, e) can cancel to exactly 0 -- and 0 * inf is NaN.
//  * `diff_grad <= 0 -> continue` (:503) is max.NaN(diff, 0): a NaN still propagates like the reference's test lets it.
//  * delta advances by 64 per trip instead of being re-formed from the pixel number (<= 1 ulp of delta).
//  * Two records per lane in flight, ping-pong: the load of trip t + 2 is issued as soon as trip t's record has been
//    consumed and is only needed after trip t + 1's arithmetic -- k9_scan's one-deep pipeline re-uses the record's
//    registers and, on these scans, waited for every load (long-scoreboard stalls dominated).
// Trip count is warp-uniform; only the loads are predicated.
__device__ __forceinline__ float max_nan(float a, float b) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

template <int MODE>
__device__ __forceinline__ void k9_term(const K9Px<MODE>& c, float r0, float r1, float r2, float ra, float delta,
                                        float k0, float k1, float e0, float e1, float& acc0, float& acc1) {
    const float d = max_nan(k9_diff<MODE>(c, r0, r1, r2, ra), 0.f);
    acc0 = __fmaf_rn(-d, rcp_approx(__fmaf_rn(delta, k0, e0)), acc0);
    acc1 = __fmaf_rn(-d, rcp_approx(__fmaf_rn(delta, k1, e1)), acc1);
}

template <int MODE>
__device__ __forceinline__ void k9_scan_out(const float* __restrict__ prow, int d1_from, int d1_to, int lane,
                                            float r0, float r1, float r2, float ra, float d1_cross, float k0, float k1,
                                            float eps, float& acc0, float& acc1) {
    constexpr int FL = K9Rec<MODE>::FL;
    const int n = d1_to - d1_from + 1;   // pixels of the scan, warp-uniform
    const int mine = n - lane;           // this lane has a pixel in trip t (32 pixels each) iff 32 t < mine
    const float* __restrict__ p = prow + (d1_from + lane) * FL;
    float delta = (float)(d1_from + lane) - d1_cross;
    const float side = (float)d1_from - d1_cross;   // the sign every delta of this scan has
    const float e0 = (0.f < side * k0) ? eps : -eps;
    const float e1 = (0.f < side * k1) ? eps : -eps;
    K9Px<MODE> a = k9_load_px<MODE>(p, mine > 0);
    K9Px<MODE> b = k9_load_px<MODE>(p + 32 * FL, mine > 32);
    int t = 64;   // first pixel of the trip pair AFTER the one being evaluated
    for (; t < n; t += 64) {   // every lane of these pairs has a pixel
        p += 64 * FL;
        k9_term<MODE>(a, r0, r1, r2, ra, delta, k0, k1, e0, e1, acc0, acc1);
        a = k9_load_px<MODE>(p, mine > t);
        k9_term<MODE>(b, r0, r1, r2, ra, delta + 32.f, k0, k1, e0, e1, acc0, acc1);
        b = k9_load_px<MODE>(p + 32 * FL, mine > t + 32);
        delta += 64.f;
    }
    // the last pair (t - 64 < n <= t), peeled so that only it pays for the past-the-end select
    k9_term<MODE>(a, r0, r1, r2, ra, (mine > t - 64) ? delta : side, k0, k1, e0, e1, acc0, acc1);
    k9_term<MODE>(b, r0, r1, r2, ra, (mine > t - 32) ? delta + 32.f : side, k0, k1, e0, e1, acc0, acc1);
}

// One (edge, axis) pass of the reference's per-face loop (:386-410): the edge's vertices in (major, minor) pixel
// coordinates, the scan direction and the range of integer major coordinates d0 the edge crosses.
struct K9Pass {
    float p00, p01, p10, p11, p20, p21;
    int direction, d0_from, d0_to;
};

__device__ __forceinline__ K9Pass k9_pass(int pass, const float px[3], const float py[3], int is) {
    const int edge_num = pass >> 1, axis = pass & 1;
    const int pi0 = edge_num, pi1 = (edge_num == 2) ? 0 : edge_num + 1, pi2 = (edge_num == 0) ? 2 : edge_num - 1;
    // p[num][dim] = pp[num][(dim + axis) % 2]   (:396-401)
    const float ax0 = k9_sel3(pi0, px[0], px[1], px[2]), ay0 = k9_sel3(pi0, py[0], py[1], py[2]);
    const float ax1 = k9_sel3(pi1, px[0], px[1], px[2]), ay1 = k9_sel3(pi1, py[0], py[1], py[2]);
    const float ax2 = k9_sel3(pi2, px[0], px[1], px[2]), ay2 = k9_sel3(pi2, py[0], py[1], py[2]);
    K9Pass r;
    r.p00 = axis ? ay0 : ax0; r.p01 = axis ? ax0 : ay0;
    r.p10 = axis ? ay1 : ax1; r.p11 = axis ? ax1 : ay1;
    r.p20 = axis ? ay2 : ax2; r.p21 = axis ? ax2 : ay2;
    if (axis == 0) r.direction = (r.p00 < r.p10) ? -1 : 1;   // :404-414
    else r.direction = (r.p00 < r.p10) ? 1 : -1;
    r.d0_from = (int)fmax((double)ceilf(fminf(r.p00, r.p10)), 0.);   // :418-419
    r.d0_to = (int)fmin((double)fmaxf(r.p00, r.p10), is - 1.);
    return r;
}

// K9 (backward_pixel_map_cuda_kernel, n3mr/cuda/rasterize.py:351-610): warp per (batch, face).
//
// A face has six (edge, axis) passes and, per pass, one SAMPLE for every integer major coordinate the edge crosses
// (:420).  A sample's set-up -- crossing point, in / out pixel, their colours and owner, the in-scan limit, the two
// distance scales (:421-460, :523-540; ~190 instructions and five dependent loads) -- is independent of every other
// sample's, and for the small faces of a dense mesh it outweighed the scans themselves when the whole warp ran it once
// per sample.  So the lanes take one sample each: the set-up of up to 32 samples runs once, in parallel, and the warp then
// visits the samples one by one (parameters broadcast by shuffle) only for the two line scans of k9_scan, where all 32
// lanes have pixels to work on.  d1_cross / d0_cross2 -- which pick pixels through floor / ceil -- keep the reference's
// exact, unfused arithmetic; the per-sample quotients that only scale `dist` use the approximate reciprocal.
// resident 256-thread CTAs per SM (80 registers, no spills).  H100, C4: 4.51 ms at 3, 4.70 at 2 (128 registers), 4.55 at
// 4 (64, spills), 5.14 at 5, 5.55 at 6, 6.23 at 8 -- the scans are latency-bound
constexpr int kK9MinBlocks = 3;
template <int MODE>
__global__ void __launch_bounds__(256, kK9MinBlocks)
k_nmr_backward_pixel_map(const float* __restrict__ faces, const int* __restrict__ face_index_map,
                         const float* __restrict__ rgb_map, const float* __restrict__ alpha_map,
                         const float* __restrict__ ph, const float* __restrict__ pv,
                         float* __restrict__ grad_faces, int batch_size, int num_faces, int is, float eps) {
    constexpr int FL = K9Rec<MODE>::FL;
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const long i = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= (long)batch_size * num_faces) return;
    const int bn = (int)(i / num_faces);
    const int fn = (int)(i % num_faces);
    const float* __restrict__ face = faces + i * 9;
    float fx[3], fy[3];
#pragma unroll
    for (int k = 0; k < 3; k++) { fx[k] = __ldg(face + 3 * k); fy[k] = __ldg(face + 3 * k + 1); }
    if ((fy[2] - fy[0]) * (fx[1] - fx[0]) < (fy[1] - fy[0]) * (fx[2] - fx[0])) return;  // :377 (zeros stay)
    // pixel-space vertices, pp[num][dim] = 0.5 * (face * is + is - 1)  (:389-393)
    float px[3], py[3];
#pragma unroll
    for (int k = 0; k < 3; k++) { px[k] = 0.5f * (fx[k] * is + is - 1); py[k] = 0.5f * (fy[k] * is + is - 1); }

    const float ndc_scale = 2.f / (float)is;
    const size_t img = (size_t)bn * is * is;
    // per-image bases: everything below indexes them with 32-bit offsets (is <= 4096: is^2 * FL <= 2^27)
    const int* __restrict__ fim_img = face_index_map + img;
    const float* __restrict__ rgb_img = (MODE & 1) ? rgb_map + img * 3 : nullptr;
    const float* __restrict__ alpha_img = (MODE & 2) ? alpha_map + img : nullptr;
    const float* __restrict__ ph_img = ph + img * FL;
    const float* __restrict__ pv_img = pv + img * FL;

    // samples of the six passes, enumerated pass-major: start[p] = first sample number of pass p
    int start[7];
    start[0] = 0;
#pragma unroll
    for (int p = 0; p < 6; p++) {
        const K9Pass q = k9_pass(p, px, py, is);
        start[p + 1] = start[p] + max(q.d0_to - q.d0_from + 1, 0);
    }
    const int total = start[6];

    float gacc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // [vertex*2 + (0:x, 1:y)]
    for (int s0 = 0; s0 < total; s0 += 32) {
        // ---- this lane's sample: everything of :421-460 and :523-540, no scan yet
        const int sidx = s0 + lane;
        int pass = 0;
#pragma unroll
        for (int p = 1; p < 6; p++) pass += (sidx >= start[p]) ? 1 : 0;
        bool live = sidx < total;
        const K9Pass q = k9_pass(pass, px, py, is);
        const int axis = pass & 1;
        const int d0 = q.d0_from + (sidx - k9_sel6(pass, start));
        const float d0f = (float)d0;
        const float d1_cross = (q.p11 - q.p01) / (q.p10 - q.p00) * (d0f - q.p00) + q.p01;   // :423
        const int d1_in = (0 < q.direction) ? (int)floorf(d1_cross) : (int)ceilf(d1_cross);
        const int d1_out = d1_in + q.direction;
        live = live && !(d1_in < 0 || is <= d1_in) && !(d1_out < 0 || is <= d1_out);         // :431-434
        const bool has0 = q.p10 != d0f, has1 = q.p00 != d0f;
        const float span = q.p10 - q.p00;
        // pixel -> NDC: the reference's (float)((double)(q * delta) * 2. / is) is formed as delta * (q * (2 / is)); q by
        // approximate reciprocal -- a few ulp on a quantity that is then offset by eps and inverted approximately
        const float k0 = span * rcp_approx(q.p10 - d0f) * ndc_scale, k1 = span * rcp_approx(d0f - q.p00) * ndc_scale;
        const int fim_stride = (axis == 0) ? is : 1;
        const int fim_base = (axis == 0) ? d0 : d0 * is;
        const int idx_in = fim_base + d1_in * fim_stride, idx_out = fim_base + d1_out * fim_stride;
        int owner_in = -2;
        float i0 = 0.f, i1 = 0.f, i2 = 0.f, ia = 0.f, o0 = 0.f, o1 = 0.f, o2 = 0.f, oa = 0.f;
        if (live) {
            owner_in = __ldg(fim_img + idx_in);
            if (MODE & 1) {
                i0 = __ldg(rgb_img + idx_in * 3); i1 = __ldg(rgb_img + idx_in * 3 + 1); i2 = __ldg(rgb_img + idx_in * 3 + 2);
                o0 = __ldg(rgb_img + idx_out * 3); o1 = __ldg(rgb_img + idx_out * 3 + 1); o2 = __ldg(rgb_img + idx_out * 3 + 2);
            }
            if (MODE & 2) { ia = __ldg(alpha_img + idx_in); oa = __ldg(alpha_img + idx_out); }
        }
        // outward scan range (:461-473), only if the face owns the in-pixel
        const int olim = (0 < q.direction) ? is - 1 : 0;
        int out_from = max(min(d1_out, olim), 0), out_to = min(max(d1_out, olim), is - 1);
        if (!(live && owner_in == fn)) { out_from = 1; out_to = 0; }
        // inward scan range (:525-540)
        float d0_cross2;
        if ((d0f - q.p00) * (d0f - q.p20) < 0.f) d0_cross2 = (q.p21 - q.p01) / (q.p20 - q.p00) * (d0f - q.p00) + q.p01;
        else d0_cross2 = (q.p11 - q.p21) / (q.p10 - q.p20) * (d0f - q.p20) + q.p21;
        const int ilim = (0 < q.direction) ? (int)ceilf(d0_cross2) : (int)floorf(d0_cross2);
        int in_from = max(min(d1_in, ilim), 0), in_to = min(max(d1_in, ilim), is - 1);
        if (!live) { in_from = 1; in_to = 0; }
        // ---- inward scans of small faces: a few pixels each, so every lane walks ITS OWN sample's pixels (:556-601) instead
        // of the warp visiting the samples one after the other for a single partly filled trip each.  (Requesting a pixel's
        // record together with its owner, instead of after the owner test, was slower at C4.)
        constexpr int kSerialIn = 64;
        if (in_from <= in_to && in_to - in_from < kSerialIn) {
            const float* __restrict__ prow_l = ((axis == 0) ? pv_img : ph_img) + d0 * is * FL;
            float a0 = 0.f, a1 = 0.f;
            for (int d1 = in_from; d1 <= in_to; d1++) {
                if (__ldg(fim_img + fim_base + d1 * fim_stride) != fn) continue;   // :573
                const float diff = k9_diff<MODE>(k9_load_px<MODE>(prow_l + d1 * FL, true), o0, o1, o2, oa);
                if (diff <= 0.f) continue;                                          // :587
                const float delta = (float)d1 - d1_cross;
                if (has0) k9_guarded_term(diff, delta, k0, eps, a0);
                if (has1) k9_guarded_term(diff, delta, k1, eps, a1);
            }
            k9_add_slots(pass, a0, a1, gacc);
            in_from = 1; in_to = 0;   // done
        }
        const unsigned todo = __ballot_sync(FULL, out_from <= out_to || in_from <= in_to);

        // ---- the warp visits the samples that still have pixels to scan (outward scans; inward scans of large faces).
        // Samples are numbered pass-major, so the pass of the visited samples never decreases: the two running sums are
        // flushed into the face's six gradient slots only when the pass changes.
        int cur_pass = -1;
        float acc0 = 0.f, acc1 = 0.f;   // contributions to vertex pi0 / pi1 of the current pass's edge, coordinate (1 - axis)
        auto flush = [&]() {
            if (cur_pass < 0) return;
            k9_add_slots(cur_pass, acc0, acc1, gacc);
            acc0 = 0.f; acc1 = 0.f;
        };
        for (unsigned m = todo; m != 0u; m &= m - 1u) {
            const int src = __ffs(m) - 1;
            const int s_pass = __shfl_sync(FULL, pass, src);
            if (s_pass != cur_pass) { flush(); cur_pass = s_pass; }
            const int s_d0 = __shfl_sync(FULL, d0, src);
            const float s_cross = __shfl_sync(FULL, d1_cross, src);
            const float s_k0 = __shfl_sync(FULL, k0, src), s_k1 = __shfl_sync(FULL, k1, src);
            const int s_flags = __shfl_sync(FULL, (has0 ? 1 : 0) | (has1 ? 2 : 0), src);
            const int s_of = __shfl_sync(FULL, out_from, src), s_ot = __shfl_sync(FULL, out_to, src);
            const int s_if = __shfl_sync(FULL, in_from, src), s_it = __shfl_sync(FULL, in_to, src);
            const int s_axis = s_pass & 1;
            const float* __restrict__ prow = ((s_axis == 0) ? pv_img : ph_img) + s_d0 * is * FL;
            const bool both = s_flags == 3;
            if (s_of <= s_ot) {   // outwards from the edge to the image border; reference colour = the in-pixel's
                const float r0 = __shfl_sync(FULL, i0, src), r1 = __shfl_sync(FULL, i1, src), r2 = __shfl_sync(FULL, i2, src);
                const float ra = (MODE & 2) ? __shfl_sync(FULL, ia, src) : 0.f;
                if (both) k9_scan_out<MODE>(prow, s_of, s_ot, lane, r0, r1, r2, ra, s_cross, s_k0, s_k1, eps, acc0, acc1);
                else k9_scan<MODE, false>(prow, nullptr, 0, s_of, s_ot, lane, fn, r0, r1, r2, ra, s_cross, s_k0, s_k1, (s_flags & 1) != 0, (s_flags & 2) != 0, eps, acc0, acc1);
            }
            if (s_if <= s_it) {   // inwards up to the opposite edge, pixels owned by the face; reference colour = the out-pixel's
                const float r0 = __shfl_sync(FULL, o0, src), r1 = __shfl_sync(FULL, o1, src), r2 = __shfl_sync(FULL, o2, src);
                const float ra = (MODE & 2) ? __shfl_sync(FULL, oa, src) : 0.f;
                const int s_stride = (s_axis == 0) ? is : 1;
                const int* __restrict__ frow = fim_img + ((s_axis == 0) ? s_d0 : s_d0 * is);
                k9_scan<MODE, true>(prow, frow, s_stride, s_if, s_it, lane, fn, r0, r1, r2, ra, s_cross, s_k0, s_k1, (s_flags & 1) != 0, (s_flags & 2) != 0, eps, acc0, acc1);
            }
        }
        flush();
    }
#pragma unroll
    for (int k = 0; k < 6; k++) gacc[k] = warp_sum_f(gacc[k]);
    if (lane == 0) {
        float* g = grad_faces + i * 9;
        g[0] = gacc[0]; g[1] = gacc[1]; g[2] = 0.f;
        g[3] = gacc[2]; g[4] = gacc[3]; g[5] = 0.f;
        g[6] = gacc[4]; g[7] = gacc[5]; g[8] = 0.f;
    }
}

// ---------------------------------------------------------------- K10 + K11 fused: thread per pixel
__global__ void __launch_bounds__(256)
k_nmr_backward_maps(const float* __restrict__ faces, const int* __restrict__ face_index_map,
                    const float* __restrict__ weight_map, const float* __restrict__ depth_map,
                    const float* __restrict__ face_inv_map, const int* __restrict__ sampling_index_map,
                    const float* __restrict__ sampling_weight_map, const float* __restrict__ grad_rgb_map,
                    const float* __restrict__ grad_depth_map, float* __restrict__ grad_faces,
                    float* __restrict__ grad_textures, int batch_size, int nf, int is, int ts,
                    int return_rgb, int return_depth) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)batch_size * is * is) return;
    const int fn = __ldg(face_index_map + i);
    if (fn < 0) return;
    const int bn = (int)(i / ((size_t)is * is));
    if (return_rgb) {  // K10 :675-692
        float* gt = grad_textures + ((size_t)bn * nf + fn) * ts * ts * ts * 3;
        const float g0 = __ldg(grad_rgb_map + i * 3 + 0), g1 = __ldg(grad_rgb_map + i * 3 + 1), g2 = __ldg(grad_rgb_map + i * 3 + 2);
        const int4 si0 = __ldg(reinterpret_cast<const int4*>(sampling_index_map + i * 8)), si1 = __ldg(reinterpret_cast<const int4*>(sampling_index_map + i * 8) + 1);
        const float4 sw0 = __ldg(reinterpret_cast<const float4*>(sampling_weight_map + i * 8)), sw1 = __ldg(reinterpret_cast<const float4*>(sampling_weight_map + i * 8) + 1);
        const int sidx[8] = {si0.x, si0.y, si0.z, si0.w, si1.x, si1.y, si1.z, si1.w};
        const float swt[8] = {sw0.x, sw0.y, sw0.z, sw0.w, sw1.x, sw1.y, sw1.z, sw1.w};
        // texture_size 2: the eight taps are the face's eight texels, tap pn at texel (pn&1)*4 + (pn&2) + (pn>>2) (:266-279):
        // 24 contiguous floats, added with six 16-byte atomics instead of 24 scalar ones (the kernel sits on the atomic rate)
        bool block8 = (ts == 2) && ((reinterpret_cast<uintptr_t>(gt) & 15) == 0);
#pragma unroll
        for (int pn = 0; pn < 8; pn++) block8 = block8 && sidx[pn] == ((pn & 1) * 4 + (pn & 2) + (pn >> 2));
        if (block8) {
            float v[24];
#pragma unroll
            for (int pn = 0; pn < 8; pn++) {
                const int t = (pn & 1) * 4 + (pn & 2) + (pn >> 2);
                v[t * 3 + 0] = swt[pn] * g0; v[t * 3 + 1] = swt[pn] * g1; v[t * 3 + 2] = swt[pn] * g2;
            }
            float4* gt4 = reinterpret_cast<float4*>(gt);
#pragma unroll
            for (int k = 0; k < 6; k++) atomicAdd(gt4 + k, make_float4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]));
        } else
#pragma unroll
        for (int pn = 0; pn < 8; pn++) {
            const float w = swt[pn];
            const int isc = sidx[pn];
            const size_t tap = ((size_t)bn * nf + fn) * ts * ts * ts + (size_t)isc;
            if (isc < 0 || tap >= (size_t)batch_size * nf * ts * ts * ts) continue;  // tap past the tensor (ts == 1, see K8)
            atomicAdd(gt + isc * 3 + 0, w * g0);
            atomicAdd(gt + isc * 3 + 1, w * g1);
            atomicAdd(gt + isc * 3 + 2, w * g2);
        }
    }
    if (return_depth) {  // K11 :755-786
        const float* face = faces + ((size_t)bn * nf + fn) * 9;
        const float depth = __ldg(depth_map + i);
        const float depth2 = depth * depth;
        const float grad_depth = __ldg(grad_depth_map + i);
        float* g = grad_faces + ((size_t)bn * nf + fn) * 9;
        float w[3], z[3], fi[9];
#pragma unroll
        for (int k = 0; k < 3; k++) { w[k] = __ldg(weight_map + i * 3 + k); z[k] = __ldg(face + 3 * k + 2); }
#pragma unroll
        for (int k = 0; k < 9; k++) fi[k] = __ldg(face_inv_map + i * 9 + k);
#pragma unroll
        for (int k = 0; k < 3; k++) atomicAdd(g + 3 * k + 2, grad_depth * w[k] * depth2 / (z[k] * z[k]));
        float tmp[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int k = 0; k < 3; k++)
#pragma unroll
            for (int l = 0; l < 3; l++) tmp[k] += -fi[3 * l + k] / z[l];
#pragma unroll
        for (int k = 0; k < 3; k++)
#pragma unroll
            for (int l = 0; l < 2; l++) atomicAdd(g + 3 * k + l, -grad_depth * tmp[l] * w[k] * depth2 * is / 2);
    }
}

}  // namespace b200r
