/*
 * softras_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement (plain C, IEEE fp32/fp64, no FMA contraction) of the
 * reference's SoftRas rasterizer kernels.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load this library.
 *
 * Follows, function by function (all paths relative to /root/reference):
 *   jrender/renderer/dr/softras/cuda/soft_rasterize.py
 *     :20-25    barycentric_coordinate
 *     :28-34    check_border
 *     :37-40    check_face_frontside
 *     :43-46    check_pixel_inside
 *     :49-54    barycentric_clip
 *     :57-147   euclidean_p2f_distance
 *     :150-154  forward_barycentric_p2f_distance
 *     :156-173  forward_sample_texture (forward flavour, perspective-correct)
 *     :176-236  forward_soft_rasterize_inv_cuda_kernel        (K1)
 *     :243-456  forward_soft_rasterize_cuda_kernel            (K2)
 *     :1118-1132 backward_barycentric_p2f_distance
 *     :1135-1151 forward_sample_texture (backward flavour, NOT perspective)
 *     :1154-1174 backward_sample_texture
 *     :1177-1360 backward_soft_rasterize_cuda_kernel (top-K)   (K6)
 *   host semantics: jrender/renderer/dr/softras/soft_rasterize.py:25,39-42,59-71,108
 *
 * Arithmetic contract.  scalar_t == float in the reference.  Every expression is
 * evaluated with the C/CUDA usual arithmetic conversions of the reference source:
 * a double literal (`1.`, `0.`, `1e-5`, `2.`) promotes that sub-expression to
 * double, and the result is rounded to float on assignment.  Build with
 * -ffp-contract=off so the compiler never fuses a*b+c (the product CUDA kernels
 * are built with -fmad=false for the same reason): +,-,*,/ and sqrt are then
 * bit-identical between this oracle and the GPU, and only expf() (libm vs CUDA
 * libdevice, both <= 2 ulp) differs.
 *
 * Documented deviations from the reference (both are UB in the reference):
 *   - backward_sample_texture returns an UNINITIALISED value for non-hit texels
 *     (:1155-1173); this oracle defines it as 0 (SURVEY.md Q9).
 *   - euclidean_p2f_distance with v0 == -1 (all w > 0 but some w >= 1, :107-121)
 *     indexes arrays at -1; this oracle skips the face's distance update by
 *     treating it as v0 = 0 (never hit by any test mesh; flagged in DESIGN.md).
 *
 * Parity status: pinned against outputs of the reference's own kernel strings
 * compiled by oracle/build_ref.py and run on a GPU (tests/golden/ref_gpu_*.npz, generated
 * by oracle/make_ref_golden.py; each file's provenance names the GPU and nvcc flags).  See DESIGN.md "Oracle".
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define K_MAX_POINTS_PER_PIXEL 64 /* :16 */

/* ------------------------------------------------------------------ rounding sites of the K6 backward
 * The CUDA backward computes every (pixel, face) term with this file's arithmetic except at the sites below, where it
 * may round differently.  softras_oracle_backward_stats re-evaluates each pair with its live sites moved by their
 * budgets in units in the last place (jointly, see there) to bound how far the kernel's term can be from this one:
 *   SITE_EXP_SIG   expf in the sigmoid: libm and CUDA's expf are each within 2 ulp of exp, so <= 3 ulp apart
 *                  (2 + 1 for a libm that is only faithful).
 *   SITE_EXP_SOFT  expf in the softmax weight, likewise.
 *   SITE_TAIL_D    softras_exact_tail = 0: D = 1 / (1 + e) in two fp32 roundings (each <= 2^-24 relative, < 1 ulp
 *                  together) against one rounding of the double quotient (<= 1/2 ulp): <= 2 ulp.
 *   SITE_PROD      softras_exact_tail = 0: the alpha-prod factor g * ((1 - alpha) / max(1 - D, 1e-6f)) in two fp32
 *                  roundings (< 2 ulp), a numerator below 2^-60 (one more ulp, as the divisions below), the double
 *                  1e-6 against 1e-6f (2.5e-9 relative) and the reference's one rounding (1/2 ulp): <= 4 ulp.
 *   SITE_DIV + i   softras_exact_tail = 0: the kernel's relaxed divisions are bit-exact for numerators >= 2^-60
 *                  (exact_math.cuh) and within 1 ulp below; a site is live only for a non-zero numerator < 2^-60.
 * With softras_exact_tail = 1 the tails and divisions are the reference's bit for bit and only the two expf sites
 * remain. */
enum {
    SITE_EXP_SIG, SITE_EXP_SOFT, SITE_TAIL_D, SITE_PROD,
    SITE_DIV_SIGARG, SITE_DIV_ZSOFT, SITE_DIV_COLD, SITE_DIV_GAMMA, SITE_DIV_NMF, SITE_DIV_SIGMA,
    SITE_DIV_Z1,          /* + k, k < 3: (C * w_k) / z_k */
    SITE_DIV_Z2 = SITE_DIV_Z1 + 3,      /* + k: (.. / z_k) / z_k */
    SITE_DIV_CLIPW = SITE_DIV_Z2 + 3,   /* + k: w_k / w_sum */
    SITE_DIV_CLIPZ = SITE_DIV_CLIPW + 3, /* + k: w_k / z_k inside zp */
    SITE_DIV_EUC = SITE_DIV_CLIPZ + 3,  /* + k: the euclidean edge parameter of edge k */
    N_SITES = SITE_DIV_EUC + 3,
    /* forward only (see "rounding sites of the K2 forward" below) */
    SITE_EXP_BG = N_SITES, SITE_DIV_SPAN,
    N_FWD_SITES
};
typedef struct {
    int exact_tail;       /* the kernel's softras_exact_tail */
    uint32_t up, down;    /* sites moved up / down by their budget */
    int hashed;           /* every live site moved, by a hashed sign per (pair, site) */
    uint32_t pair;        /* hash input */
    uint32_t live;        /* out: sites with a non-zero budget in this pair */
} Nudge;

static inline float move_ulps(float x, int n, int dir) {
    for (int i = 0; i < n; i++) x = nextafterf(x, dir > 0 ? INFINITY : -INFINITY);
    return x;
}

/* x at site s with a budget of n ulp */
static inline float site(Nudge *nd, int s, float x, int n) {
    if (!nd || n <= 0 || !isfinite(x)) return x;
    nd->live |= 1u << s;
    if (nd->up >> s & 1u) return move_ulps(x, n, 1);
    if (nd->down >> s & 1u) return move_ulps(x, n, -1);
    if (nd->hashed) {
        uint32_t h = nd->pair * 0x9E3779B1u ^ (uint32_t)(s + 1) * 0x85EBCA77u;
        h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12;
        return move_ulps(x, n, (h & 1u) ? 1 : -1);
    }
    return x;
}

/* a / b as one of the kernel's relaxed divisions */
static inline float rdiv(Nudge *nd, int s, float a, float b) {
    const float q = a / b;
    if (nd && !nd->exact_tail && a != 0.f && fabsf(a) < 0x1p-60f) return site(nd, s, q, 1);
    return q;
}

/* :20-25 */
static inline void barycentric_coordinate(float *w, float x, float y, const float *fi) {
    w[0] = fi[0] * x + fi[1] * y + fi[2];
    w[1] = fi[3] * x + fi[4] * y + fi[5];
    w[2] = fi[6] * x + fi[7] * y + fi[8];
}

/* :28-34 */
static inline int check_border(float x, float y, const float *face, float threshold) {
    return (x > fmaxf(fmaxf(face[0], face[3]), face[6]) + threshold ||
            x < fminf(fminf(face[0], face[3]), face[6]) - threshold ||
            y > fmaxf(fmaxf(face[1], face[4]), face[7]) + threshold ||
            y < fminf(fminf(face[1], face[4]), face[7]) - threshold);
}

/* :37-40 */
static inline int check_face_frontside(const float *face) {
    return (face[7] - face[1]) * (face[3] - face[0]) < (face[4] - face[1]) * (face[6] - face[0]);
}

/* :43-46 */
static inline int check_pixel_inside(const float *w) {
    return w[0] <= 1 && w[0] >= 0 && w[1] <= 1 && w[1] >= 0 && w[2] <= 1 && w[2] >= 0;
}

/* :49-54 -- min/max against double literals, sum clamp against 1e-5 (double) */
static inline void barycentric_clip(float *w) {
    for (int k = 0; k < 3; k++) w[k] = (float)fmax(fmin((double)w[k], 1.), 0.);
    const float w_sum = (float)fmax((double)(w[0] + w[1] + w[2]), 1e-5);
    for (int k = 0; k < 3; k++) w[k] /= w_sum;
}

/* :57-147.  nd: the backward's rounding sites (NULL in the forward, whose divisions are exact) */
static inline void euclidean_p2f_distance(float *sign, float *dis_x, float *dis_y,
                                          const float *w, float *t,
                                          const float *face, const float *face_info,
                                          float xp, float yp, Nudge *nd) {
    const float *face_sym = face_info + 9;
    const float *face_obt = face_info + 18;

    if (w[0] > 0 && w[1] > 0 && w[2] > 0 && w[0] < 1 && w[1] < 1 && w[2] < 1) {
        float dis_min = 100000000;
        float dis_x_min = 0;
        float dis_y_min = 0;
        float a0[3];
        float t0[3];
        for (int k = 0; k < 3; k++) {
            int v0 = k;
            int v1 = (k + 1) % 3;
            int v2 = (k + 2) % 3;
            a0[0] = face_sym[3 * v0 + 0] - face_sym[3 * v1 + 0];
            a0[1] = face_sym[3 * v0 + 1] - face_sym[3 * v1 + 1];
            a0[2] = face_sym[3 * v0 + 2] - face_sym[3 * v1 + 2];

            t0[v0] = rdiv(nd, SITE_DIV_EUC + k, w[0] * a0[0] + w[1] * a0[1] + w[2] * a0[2] - a0[v1], a0[v0] - a0[v1]);
            t0[v1] = 1 - t0[v0];
            t0[v2] = 0;

            t0[0] -= w[0];
            t0[1] -= w[1];
            t0[2] -= w[2];

            float dx = t0[0] * face[0] + t0[1] * face[3] + t0[2] * face[6];
            float dy = t0[0] * face[1] + t0[1] * face[4] + t0[2] * face[7];
            float dis = dx * dx + dy * dy;

            if (dis < dis_min) {
                dis_min = dis;
                dis_x_min = dx;
                dis_y_min = dy;
                t[0] = t0[0];
                t[1] = t0[1];
                t[2] = t0[2];
            }
        }
        *dis_x = dis_x_min;
        *dis_y = dis_y_min;
        *sign = 1;
    } else {
        int v0 = -1;

        if (w[1] <= 0 && w[2] <= 0) {
            v0 = 0;
            if (face_obt[0] == 1 && (xp - face[0]) * (face[6] - face[0]) + (yp - face[1]) * (face[7] - face[1]) > 0) v0 = 2;
        } else if (w[2] <= 0 && w[0] <= 0) {
            v0 = 1;
            if (face_obt[1] == 1 && (xp - face[3]) * (face[0] - face[3]) + (yp - face[4]) * (face[1] - face[4]) > 0) v0 = 0;
        } else if (w[0] <= 0 && w[1] <= 0) {
            v0 = 2;
            if (face_obt[2] == 1 && (xp - face[6]) * (face[3] - face[6]) + (yp - face[7]) * (face[4] - face[7]) > 0) v0 = 1;
        } else if (w[0] <= 0) v0 = 1;
        else if (w[1] <= 0) v0 = 2;
        else if (w[2] <= 0) v0 = 0;

        if (v0 < 0) v0 = 0; /* reference UB (index -1); see header */

        const int v1 = (v0 + 1) % 3;
        const int v2 = (v0 + 2) % 3;

        float a0[3];
        a0[0] = face_sym[3 * v0 + 0] - face_sym[3 * v1 + 0];
        a0[1] = face_sym[3 * v0 + 1] - face_sym[3 * v1 + 1];
        a0[2] = face_sym[3 * v0 + 2] - face_sym[3 * v1 + 2];

        t[v0] = rdiv(nd, SITE_DIV_EUC + v0, w[0] * a0[0] + w[1] * a0[1] + w[2] * a0[2] - a0[v1], a0[v0] - a0[v1]);
        t[v1] = 1 - t[v0];
        t[v2] = 0;

        for (int k = 0; k < 3; k++) {
            t[k] = (float)fmin(fmax((double)t[k], 0.), 1.);
            t[k] -= w[k];
        }

        *dis_x = t[0] * face[0] + t[1] * face[3] + t[2] * face[6];
        *dis_y = t[0] * face[1] + t[1] * face[4] + t[2] * face[7];
        *sign = -1;
    }
}

/* :150-154 */
static inline float forward_barycentric_p2f_distance(const float *w) {
    float dis = w[0] > w[1] ? (w[1] > w[2] ? w[2] : w[1]) : (w[0] > w[2] ? w[2] : w[0]);
    dis = dis > 0 ? dis * dis : -dis * dis;
    return dis;
}

/* :156-173 (forward flavour) */
static inline float forward_sample_texture_fwd(const float *texture, const float *w, int R, int k,
                                               int texture_sample_type, const float *face, float z) {
    float texture_k = 0;
    if (texture_sample_type == 0) {
        const int w_x = (int)fminf(w[0] * R, (float)(R - 1));
        const int w_y = (int)fminf(w[1] * R, (float)(R - 1));
        if ((w[0] + w[1]) * R - w_x - w_y <= 1) {
            texture_k = texture[(w_y * R + w_x) * 3 + k];
        } else {
            texture_k = texture[((R - 1 - w_y) * R + (R - 1 - w_x)) * 3 + k];
        }
    } else if (texture_sample_type == 1) {
        texture_k = w[0] * texture[k] / face[2] + w[1] * texture[3 + k] / face[5] + w[2] * texture[6 + k] / face[8];
        texture_k *= z;
    }
    return texture_k;
}

/* :1135-1151 (backward flavour: vertex mode is NOT perspective-correct, Q8) */
static inline float forward_sample_texture_bwd(const float *texture, const float *w, int R, int k,
                                               int texture_sample_type) {
    float texture_k = 0;
    if (texture_sample_type == 0) {
        const int w_x = (int)fminf(w[0] * R, (float)(R - 1));
        const int w_y = (int)fminf(w[1] * R, (float)(R - 1));
        if ((w[0] + w[1]) * R - w_x - w_y <= 1) {
            texture_k = texture[(w_y * R + w_x) * 3 + k];
        } else {
            texture_k = texture[((R - 1 - w_y) * R + (R - 1 - w_x)) * 3 + k];
        }
    } else if (texture_sample_type == 1) {
        texture_k = w[0] * texture[k] + w[1] * texture[3 + k] + w[2] * texture[6 + k];
    }
    return texture_k;
}

/* :1154-1174; non-hit texels are UB in the reference, defined as 0 here (Q9) */
static inline float backward_sample_texture(float grad_color, const float *w, int R, int k,
                                            int texture_sample_type) {
    float grad_texture_k = 0;
    if (texture_sample_type == 0) {
        const int w_x = (int)fminf(w[0] * R, (float)(R - 1));
        const int w_y = (int)fminf(w[1] * R, (float)(R - 1));
        if ((w[0] + w[1]) * R - w_x - w_y <= 1) {
            if (k == w_y * R + w_x) grad_texture_k = grad_color;
        } else {
            if (k == (R - 1 - w_y) * R + (R - 1 - w_x)) grad_texture_k = grad_color;
        }
    } else if (texture_sample_type == 1) {
        grad_texture_k = w[k] * grad_color;
    }
    return grad_texture_k;
}

/* :1118-1132 */
static inline void backward_barycentric_p2f_distance(float grad_v[3][3], const float *w,
                                                     const float *face_info, float xp, float yp,
                                                     float dis, float C) {
    const int p = w[0] > w[1] ? (w[1] > w[2] ? 2 : 1) : (w[0] > w[2] ? 2 : 0);
    const float *face_inv = face_info;
    for (int l = 0; l < 2; l++) {
        for (int k = 0; k < 3; k++) {
            float grad_kl = 0;
            for (int q = 0; q < 3; q++) {
                grad_kl += -face_inv[3 * p + l] * face_inv[3 * k + q] * (q == 0 ? xp : (q == 1 ? yp : 1));
            }
            grad_v[k][l] = grad_kl * C;
            grad_v[k][l] = (float)((double)grad_v[k][l] *
                                   (dis > 0 ? (2. * (double)sqrtf(dis)) : (2. * (double)sqrtf(-dis))));
        }
    }
}

/* ------------------------------------------------------------------ K1 :176-236 */
void softras_oracle_face_info(const float *faces, float *faces_info, int batch_size, int num_faces) {
    const long n = (long)batch_size * num_faces;
    memset(faces_info, 0, sizeof(float) * 27 * (size_t)n); /* cudaMemsetAsync(out0_p, 0, ...) :467 */
    for (long i = 0; i < n; i++) {
        const float *face = &faces[i * 9];
        float *face_inv = &faces_info[i * 27];
        float *face_sym = &faces_info[i * 27 + 9];
        float *face_obt = &faces_info[i * 27 + 18];
        float p[3][2];
        for (int num = 0; num < 3; num++)
            for (int dim = 0; dim < 2; dim++) p[num][dim] = face[3 * num + dim];
        float face_inv_star[9] = {
            p[1][1] - p[2][1], p[2][0] - p[1][0], p[1][0] * p[2][1] - p[2][0] * p[1][1],
            p[2][1] - p[0][1], p[0][0] - p[2][0], p[2][0] * p[0][1] - p[0][0] * p[2][1],
            p[0][1] - p[1][1], p[1][0] - p[0][0], p[0][0] * p[1][1] - p[1][0] * p[0][1]};
        float det = (p[2][0] * (p[0][1] - p[1][1]) + p[0][0] * (p[1][1] - p[2][1]) + p[1][0] * (p[2][1] - p[0][1]));
        det = det > 0 ? (float)fmax((double)det, 1e-10) : (float)fmin((double)det, -1e-10);
        for (int k = 0; k < 9; k++) face_inv[k] = face_inv_star[k] / det;
        for (int j = 0; j < 3; j++)
            for (int k = 0; k < 3; k++)
                face_sym[j * 3 + k] = face[j * 3 + 0] * face[k * 3 + 0] + face[j * 3 + 1] * face[k * 3 + 1] + 1;
        for (int k = 0; k < 3; k++) {
            const int k0 = k, k1 = (k + 1) % 3, k2 = (k + 2) % 3;
            if ((p[k1][0] - p[k0][0]) * (p[k2][0] - p[k0][0]) + (p[k1][1] - p[k0][1]) * (p[k2][1] - p[k0][1]) < 0) {
                face_obt[k0] = 1;
                break;
            }
        }
    }
}

typedef struct {
    int id;
    float z;
} Pixel; /* :238-241 */

/* ------------------------------------------------------------------ rounding sites of the K2 forward
 * The CUDA forward (softras_forward.cuh shade_face / aggregate_alpha / initial_state / finalize_pixel, with DivPolicy
 * of softras_math.cuh) evaluates every discrete decision of a pixel -- border, inside, distance threshold, zp, near /
 * far, top-K, the nearest face -- with this file's arithmetic bit for bit: its euclidean edge parameter, clip and zp
 * divisions and the vertex-texture divisions are strict (correctly rounded for every input), and finalize_pixel's
 * colour quotients are fast_div (correctly rounded too).  It may differ only at these sites:
 *   SITE_EXP_BG     expf(eps / gamma), the initial softmax_sum: <= 3 ulp, as SITE_EXP_SIG of the backward.
 *   SITE_EXP_SIG    expf in the sigmoid: <= 3 ulp.
 *   SITE_EXP_SOFT   expf of exp_delta_zp and of exp_z: <= 3 ulp.  expf(+-0) is 1 exactly in both libraries, so a site
 *                   whose argument is zero (exp_z of the face that raised softmax_max; the OPT body sets that weight to
 *                   1 without an expf) is not live.
 *   SITE_TAIL_D     softras_exact_tail = 0: D = rcp(1.f + e), two fp32 roundings (rcp is IEEE 1 / y), where this file
 *                   rounds the double quotient once.
 *   SITE_PROD       softras_exact_tail = 0: alpha * (1.f - D) in fp32, where this file rounds the double product once
 *                   (the same bits when D is exactly 0 or 1, as under hard distances).
 *   SITE_DIV_SIGARG softras_exact_tail = 0: by_sigma(-sign * dis), a relaxed division: exact for numerators >= 2^-60
 *                   and within 1 ulp below (exact_math.cuh relaxed_div; the slow path when sigma is not midrange).
 *   SITE_DIV_SPAN   softras_exact_tail = 0: by_span(far - zp), likewise; it feeds zp_norm, softmax_max and the
 *                   `zp_norm > softmax_max` decision.
 *   SITE_DIV_GAMMA  softras_exact_tail = 0: by_gamma of the two exp arguments, likewise.
 * With softras_exact_tail = 1 the tails and divisions are the reference's bit for bit: only the expf sites remain.
 *
 * The bound.  Beside each state variable of a pixel (softmax_sum, sc0..2, alpha, softmax_max) the forward carries an
 * interval [lo, hi] in float that holds every value the kernel can have there.  An expf site widens its value by its
 * budget: the libm expf of each end moved 3 ulp outwards.  That needs no monotone libm: CUDA's expf is within 2 ulp of
 * exp and libm's within 1, and exp itself is monotone, so for any x' in [lo, hi] the kernel's expf(x') is at least
 * exp(lo) - 2 ulp >= expf_libm(lo) - 3 ulp, and at most expf_libm(hi) + 3 ulp likewise; a division
 * site widens the quotient by 1 ulp whenever the numerator's interval reaches a non-zero value below 2^-60; the tail
 * sites are the kernel's own fp32 expressions, evaluated on the interval's ends.  Every update the pixel makes
 * (s' = a s + b c, the exp_delta_zp rescale, 1 - alpha, / nf, sc / softmax_sum) is monotone in each operand once the
 * operands' signs are fixed, and rounding to nearest is monotone, so evaluating the kernel's float operations on the
 * corners of the operand intervals (min and max of the four products, ends of sums) encloses the kernel's result --
 * this is at least as tight as adding |x - y| + ulp(x) / 2 + ulp(y) / 2 per operation.  The bound of an output is its
 * interval's largest distance from this file's value.  Zero stays zero: an interval that never met a live site is the
 * single value this file computes, so its bound is exactly 0 and the kernel must match it bit for bit.
 *
 * Decisions that read a widened value: hard alpha's `D > 0.5` and `zp_norm > softmax_max`.  Where the decision's
 * interval straddles the threshold the pixel is marginal: FWD_MARG_ALPHA (its alpha's bound is infinite) or
 * FWD_MARG_MAX (its colours' and softmax_sum's bounds are infinite; softmax_max is bit-exact only where no
 * SITE_DIV_SPAN is live).  Near / far and the top-K read zp, which is exact, so they never are.
 *
 * Nudging (FwdBound.nudge = +1 / -1 / >= 2): every live expf and division site moved by its budget up / down / by a
 * hashed sign per (pixel, face, site; the hash seeded by nudge - 2), and, with exact_tail = 0, the tails taken in the kernel's fp32 form: a forward
 * the kernel could have computed, which must stay within the bound of the plain one. */
enum { FWD_MARG_ALPHA = 1, FWD_MARG_MAX = 2 };
typedef struct {
    int exact_tail;                    /* the kernel's softras_exact_tail */
    int nudge;                         /* 0, +1, -1, >= 2 (above) */
    double *bound_colors, *bound_sum;  /* [B,4,H,W], [B,H,W] */
    int32_t *marginal;                 /* [B,H,W] FWD_MARG_* */
    uint32_t *live;                    /* [B,H,W] bit s: site s was live in one of the pixel's pairs */
} FwdBound;

typedef struct {
    float lo, hi;
} Iv;
static inline Iv iv(float x) { Iv r = {x, x}; return r; }
static inline Iv iv2(float a, float b) {   /* NaN anywhere: the NaN interval */
    if (isnan(a) || isnan(b)) return iv(NAN);
    Iv r = {fminf(a, b), fmaxf(a, b)};
    return r;
}
static inline Iv iv4(float a, float b, float c, float d) {
    const Iv x = iv2(a, b), y = iv2(c, d);
    return iv2(fminf(x.lo, y.lo), fmaxf(x.hi, y.hi));
}
static inline int iv_point(Iv a) { return a.lo == a.hi; }
static inline Iv iv_add(Iv a, Iv b) { return iv2(a.lo + b.lo, a.hi + b.hi); }
static inline Iv iv_mul(Iv a, Iv b) { return iv4(a.lo * b.lo, a.lo * b.hi, a.hi * b.lo, a.hi * b.hi); }
static inline Iv iv_div(Iv a, Iv b) {
    if (iv_point(a) && iv_point(b)) return iv(a.lo / b.lo);
    if (!(b.lo > 0.f || b.hi < 0.f)) return iv2(-INFINITY, INFINITY);
    return iv4(a.lo / b.lo, a.lo / b.hi, a.hi / b.lo, a.hi / b.hi);
}
static inline float move_fin(float x, int n, int dir) { return isfinite(x) ? move_ulps(x, n, dir) : x; }
static inline float clamp0(float x) { return x < 0.f ? 0.f : x; }   /* NaN stays NaN */

/* |kernel - this file's value o| over the interval; 0 exactly for the point interval {o} */
static inline double iv_bound(float o, Iv r) {
    if (iv_point(r) && (r.lo == o || (isnan(r.lo) && isnan(o)))) return 0.0;
    const double b = fmax((double)r.hi - (double)o, (double)o - (double)r.lo);
    return isnan(b) ? INFINITY : b;
}

/* the sigmoid tail, D = 1 / (1 + e): the reference's double quotient, or the kernel's fp32 one */
static inline float tail_d(float e, int fp32) { return fp32 ? 1.f / (1.f + e) : (float)(1. / (1. + (double)e)); }
/* alpha "prod": alpha * (1 - D), likewise */
static inline float tail_prod(float a, float D, int fp32) {
    return fp32 ? a * (1.f - D) : (float)((double)a * (1. - (double)D));
}

/* a / b as a relaxed division of the kernel (by_sigma, by_span, by_gamma): returns this file's (possibly nudged) a / b
 * and sets *qi to the interval of the kernel's quotient for a numerator anywhere in ai */
static float fwd_rdiv(Nudge *nd, int s, float a, Iv ai, float b, Iv *qi) {
    float q = a / b;
    if (!nd) return q;
    *qi = iv2(ai.lo / b, ai.hi / b);
    if (!nd->exact_tail && fabsf(b) >= 0x1p-60f && fabsf(b) < 0x1p61f && ai.lo < 0x1p-60f && ai.hi > -0x1p-60f &&
        !(ai.lo == 0.f && ai.hi == 0.f)) {
        nd->live |= 1u << s;
        qi->lo = move_fin(qi->lo, 1, -1);
        qi->hi = move_fin(qi->hi, 1, 1);
        if (a != 0.f && fabsf(a) < 0x1p-60f) q = site(nd, s, q, 1);
    }
    return q;
}

/* expf(x) at site s for x in xi: returns this file's (possibly nudged) value, *ei the kernel's interval */
static float fwd_exp(Nudge *nd, int s, float x, Iv xi, Iv *ei) {
    float e = expf(x);
    if (!nd) return e;
    if (xi.lo == 0.f && xi.hi == 0.f) {
        *ei = iv(1.f);
        return e;
    }
    *ei = iv2(clamp0(move_fin(expf(xi.lo), 3, -1)), move_fin(expf(xi.hi), 3, 1));
    return clamp0(site(nd, s, e, 3));
}

/* soft_fragment = 1. / (1. + exp(num / sigma)) (:338, :344); *Di the kernel's interval */
static float fwd_sigmoid(Nudge *nd, const FwdBound *fb, float num, float sigma_val, Iv *Di) {
    if (!nd) return (float)(1. / (1. + (double)expf(num / sigma_val)));
    Iv xi, ei;
    const float x = fwd_rdiv(nd, SITE_DIV_SIGARG, num, iv(num), sigma_val, &xi);
    const float e = fwd_exp(nd, SITE_EXP_SIG, x, xi, &ei);
    const int fp32 = !fb->exact_tail;
    if (fp32) nd->live |= 1u << SITE_TAIL_D;
    *Di = iv2(tail_d(ei.hi, fp32), tail_d(ei.lo, fp32));
    return tail_d(e, fp32 && fb->nudge);
}

/* ------------------------------------------------------------------ K2 :243-456
 * Processes output rows row_begin, row_begin+row_stride, ... < row_end of every batch
 * element (row 0 = top); the full op is row_begin=0, row_end=image_size, row_stride=1.  Buffers must be pre-initialised
 * by softras_oracle_forward below (memsets of :467-470). */
static void forward_rows(const float *faces, const float *textures, const float *faces_info,
                         float *aggrs_info, float *soft_colors, int32_t *faces_id_buffers,
                         int batch_size, int num_faces, int image_size, int max_faces_id,
                         int texture_size, int texture_res, float near, float far, float eps,
                         float sigma_val, int func_id_dist, float dist_eps, float gamma_val,
                         int func_id_rgb, int func_id_alpha, int texture_sample_type,
                         int double_side, int row_begin, int row_end, int row_stride, int nthreads,
                         const FwdBound *fb) {
    const int is = image_size;
    const int nf = num_faces;
    const long npix = (long)is * is;
    const float threshold = dist_eps * sigma_val; /* :289 */
    const float border = sqrtf(threshold);        /* :316 */

    /* Hoisted check_border operands (same float adds as :30-33, computed once per face). */
    float *bb = (float *)malloc(sizeof(float) * 4 * (size_t)batch_size * nf);
    for (long f = 0; f < (long)batch_size * nf; f++) {
        const float *face = &faces[f * 9];
        bb[4 * f + 0] = fmaxf(fmaxf(face[0], face[3]), face[6]) + border;
        bb[4 * f + 1] = fminf(fminf(face[0], face[3]), face[6]) - border;
        bb[4 * f + 2] = fmaxf(fmaxf(face[1], face[4]), face[7]) + border;
        bb[4 * f + 3] = fminf(fminf(face[1], face[4]), face[7]) - border;
    }

    if (row_stride < 1) row_stride = 1;
    const long rows_per_image = (row_end - row_begin + row_stride - 1) / row_stride;
    const long rows = (long)batch_size * rows_per_image;
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#pragma omp parallel for schedule(dynamic, 1)
#endif
    for (long r = 0; r < rows; r++) {
        const int bn = (int)(r / rows_per_image);
        const int row = row_begin + (int)(r % rows_per_image) * row_stride;
        for (int col = 0; col < is; col++) {
            const long pn = (long)row * is + col;
            const int yi = is - 1 - row; /* :280 */
            const int xi = col;
            const float yp = (float)((2. * yi + 1. - is) / is);
            const float xp = (float)((2. * xi + 1. - is) / is);

            const float *face = &faces[(long)bn * nf * 9] - 9;
            const float *texture = &textures[(long)bn * nf * texture_size * 3] - texture_size * 3;
            const float *face_info = &faces_info[(long)bn * nf * 27] - 27;
            const float *fbb = &bb[(long)bn * nf * 4] - 4;

            /* fb: the kernel's intervals beside the state (see "rounding sites of the K2 forward") */
            Nudge nd = {fb ? fb->exact_tail : 1, 0, 0, fb && fb->nudge >= 2, 0, 0};
            if (fb && fb->nudge == 1) nd.up = ~0u;
            if (fb && fb->nudge == -1) nd.down = ~0u;
            Nudge *ndp = fb ? &nd : NULL;
            int marg = 0;

            float soft_color[4] = {1.f, 1.f, 1.f, 0.f};
            if (func_id_alpha == 2) soft_color[3] = 1.f;
            Iv sumi = iv(0.f), smi = iv(eps), sci[4];
            const float softmax_sum0 = eps / gamma_val;
            float softmax_sum = func_id_rgb == 1 ? fwd_exp(ndp, SITE_EXP_BG, softmax_sum0, iv(softmax_sum0), &sumi)
                                                 : expf(softmax_sum0);
            float softmax_max = eps;
            for (int k = 0; k < 3; k++) {
                if (func_id_rgb == 0) soft_color[k] = soft_colors[((long)bn * 4 + k) * npix + pn];
                else if (func_id_rgb == 1) soft_color[k] = soft_colors[((long)bn * 4 + k) * npix + pn] * softmax_sum;
                if (fb) sci[k] = iv_mul(iv(soft_colors[((long)bn * 4 + k) * npix + pn]), sumi);
            }
            sci[3] = iv(soft_color[3]);   /* (the intervals are only read when fb is set) */
            float depth_min = 10000000;
            int face_index_min = -1;
            Pixel q[K_MAX_POINTS_PER_PIXEL];
            int q_size = 0;
            float q_max_z = -1;
            int q_max_id = -1;

            for (int fn = 0; fn < nf; fn++) {
                face += 9;
                texture += texture_size * 3;
                face_info += 27;
                fbb += 4;

                if (xp > fbb[0] || xp < fbb[1] || yp > fbb[2] || yp < fbb[3]) continue; /* :316 */

                float dis, dis_x, dis_y, t[3], w[3], w_clip[3], sign, soft_fragment;
                Iv Di = iv(1.f);
                nd.pair = (uint32_t)(((long)bn * npix + pn) * 0x9E3779B1u) ^ (uint32_t)fn * 0x85EBCA77u ^
                          (uint32_t)(fb && fb->nudge > 2 ? fb->nudge : 0) * 0x27D4EB2Fu;

                barycentric_coordinate(w, xp, yp, face_info);

                if (func_id_dist == 0) {
                    soft_fragment = check_pixel_inside(w) ? 1.f : 0.f;
                    if (soft_fragment == 0.f) continue;
                } else if (func_id_dist == 1) {
                    dis = forward_barycentric_p2f_distance(w);
                    if (-dis >= threshold) continue;
                    soft_fragment = fwd_sigmoid(ndp, fb, -dis, sigma_val, &Di);
                } else {
                    euclidean_p2f_distance(&sign, &dis_x, &dis_y, w, t, face, face_info, xp, yp, NULL);
                    dis = dis_x * dis_x + dis_y * dis_y;
                    if (sign < 0 && dis >= threshold) continue;
                    soft_fragment = fwd_sigmoid(ndp, fb, -sign * dis, sigma_val, &Di);
                }

                if (func_id_alpha == 0) {
                    if (soft_fragment > 0.5) soft_color[3] = 1.f;
                    if (fb) {
                        if (Di.hi > 0.5f) sci[3].hi = 1.f;
                        if (Di.lo > 0.5f) sci[3].lo = 1.f;
                        if (!iv_point(Di) && Di.lo <= 0.5f && Di.hi > 0.5f) marg |= FWD_MARG_ALPHA;
                    }
                } else if (func_id_alpha == 1) {
                    soft_color[3] += soft_fragment;
                    if (fb) sci[3] = iv_add(sci[3], Di);
                } else if (func_id_alpha == 2) {
                    const int fp32 = fb && !fb->exact_tail;
                    soft_color[3] = tail_prod(soft_color[3], soft_fragment, fp32 && fb->nudge);
                    if (fp32 && !(iv_point(Di) && (Di.lo == 0.f || Di.lo == 1.f))) nd.live |= 1u << SITE_PROD;   /* else exact */
                    if (fb)
                        sci[3] = iv4(tail_prod(sci[3].lo, Di.lo, fp32), tail_prod(sci[3].lo, Di.hi, fp32),
                                     tail_prod(sci[3].hi, Di.lo, fp32), tail_prod(sci[3].hi, Di.hi, fp32));
                }

                for (int k = 0; k < 3; k++) w_clip[k] = w[k];
                barycentric_clip(w_clip);
                const float zp = (float)(1. / (double)(w_clip[0] / face[2] + w_clip[1] / face[5] + w_clip[2] / face[8]));
                if (zp < near || zp > far) continue;

                /* top-K by z, "replace the current max" policy :367-385 */
                if (q_size < max_faces_id) {
                    q[q_size].id = fn;
                    q[q_size].z = zp;
                    if (zp > q_max_z) {
                        q_max_z = zp;
                        q_max_id = q_size;
                    }
                    q_size++;
                } else if (zp < q_max_z) {
                    q[q_max_id].id = fn;
                    q[q_max_id].z = zp;
                    q_max_z = -1;
                    for (int k = 0; k < q_size; k++) {
                        if (q[k].z > q_max_z) {
                            q_max_z = q[k].z;
                            q_max_id = k;
                        }
                    }
                }

                if (func_id_rgb == 0) {
                    if (zp < depth_min && check_pixel_inside(w) && (double_side || check_face_frontside(face))) {
                        depth_min = zp;
                        face_index_min = fn;
                        for (int k = 0; k < 3; k++) {
                            soft_color[k] = forward_sample_texture_fwd(texture, w_clip, texture_res, k, texture_sample_type, face, zp);
                            if (fb) sci[k] = iv(soft_color[k]);
                        }
                    }
                } else if (func_id_rgb == 1) {
                    if (check_face_frontside(face) || double_side) {
                        Iv zni = iv(0.f), qi = iv(0.f), edi = iv(1.f), ezi = iv(1.f);
                        const float zp_norm = fwd_rdiv(ndp, SITE_DIV_SPAN, far - zp, iv(far - zp), far - near, &zni);
                        float exp_delta_zp = 1.f;
                        const int up = zp_norm > softmax_max;
                        if (fb && !(iv_point(zni) && iv_point(smi)) && (up ? !(zni.lo > smi.hi) : !(zni.hi <= smi.lo)))
                            marg |= FWD_MARG_MAX;
                        if (up) {
                            const float q = fwd_rdiv(ndp, SITE_DIV_GAMMA, softmax_max - zp_norm,
                                                     fb ? iv2(smi.lo - zni.hi, smi.hi - zni.lo) : qi, gamma_val, &qi);
                            exp_delta_zp = fwd_exp(ndp, SITE_EXP_SOFT, q, qi, &edi);
                            softmax_max = zp_norm;
                            smi = zni;
                        }
                        const float q = fwd_rdiv(ndp, SITE_DIV_GAMMA, zp_norm - softmax_max,
                                                 !fb ? qi : up ? iv(zp_norm - softmax_max) : iv2(zni.lo - smi.hi, zni.hi - smi.lo),
                                                 gamma_val, &qi);
                        const float exp_z = fwd_exp(ndp, SITE_EXP_SOFT, q, qi, &ezi);
                        softmax_sum = exp_delta_zp * softmax_sum + exp_z * soft_fragment;
                        const Iv wi = fb ? iv_mul(ezi, Di) : ezi;
                        if (fb) sumi = iv_add(iv_mul(edi, sumi), wi);
                        for (int k = 0; k < 3; k++) {
                            const float color_k = forward_sample_texture_fwd(texture, w_clip, texture_res, k, texture_sample_type, face, zp);
                            soft_color[k] = exp_delta_zp * soft_color[k] + exp_z * soft_fragment * color_k;
                            if (fb) sci[k] = iv_add(iv_mul(edi, sci[k]), iv_mul(wi, iv(color_k)));
                        }
                    }
                }
            }

            /* finalise :425-455 */
            if (func_id_alpha == 0) soft_colors[((long)bn * 4 + 3) * npix + pn] = soft_color[3];
            else if (func_id_alpha == 1) soft_colors[((long)bn * 4 + 3) * npix + pn] = soft_color[3] / nf;
            else if (func_id_alpha == 2) soft_colors[((long)bn * 4 + 3) * npix + pn] = (float)(1. - (double)soft_color[3]);
            if (fb) {
                Iv ai = sci[3];
                if (func_id_alpha == 1) ai = iv2(ai.lo / nf, ai.hi / nf);
                else if (func_id_alpha == 2) ai = iv2((float)(1. - (double)ai.hi), (float)(1. - (double)ai.lo));
                const long o = (long)bn * npix + pn;
                for (int k = 0; k < 3; k++) {
                    double b = 0.0;
                    if (func_id_rgb == 1) b = (marg & FWD_MARG_MAX) ? INFINITY : iv_bound(soft_color[k] / softmax_sum, iv_div(sci[k], sumi));
                    fb->bound_colors[((long)bn * 4 + k) * npix + pn] = b;
                }
                fb->bound_colors[((long)bn * 4 + 3) * npix + pn] =
                    (marg & FWD_MARG_ALPHA) ? INFINITY : iv_bound(soft_colors[((long)bn * 4 + 3) * npix + pn], ai);
                fb->bound_sum[o] = func_id_rgb != 1 ? 0.0 : (marg & FWD_MARG_MAX) ? INFINITY : iv_bound(softmax_sum, sumi);
                fb->marginal[o] = marg;
                fb->live[o] = nd.live;
            }

            if (func_id_rgb == 0) {
                if (face_index_min != -1)
                    for (int k = 0; k < 3; k++) soft_colors[((long)bn * 4 + k) * npix + pn] = soft_color[k];
                aggrs_info[((long)bn * 2 + 0) * npix + pn] = depth_min;
                aggrs_info[((long)bn * 2 + 1) * npix + pn] = (float)face_index_min;
            } else if (func_id_rgb == 1) {
                for (int k = 0; k < 3; k++) soft_colors[((long)bn * 4 + k) * npix + pn] = soft_color[k] / softmax_sum;
                aggrs_info[((long)bn * 2 + 0) * npix + pn] = softmax_sum;
                aggrs_info[((long)bn * 2 + 1) * npix + pn] = softmax_max;
            }
            for (int k = 0; k < q_size; k++)
                faces_id_buffers[((long)bn * max_faces_id + k) * npix + pn] = q[k].id;
        }
    }
    free(bb);
}

/* Full forward op = the reference's cuda_src :467-516: memsets, K1, K2.
 * faces_id_buffer layout [B, K, H, W] (as the forward writes it, :454). */
void softras_oracle_forward(const float *faces, const float *textures, float *faces_info,
                            float *aggrs_info, float *soft_colors, int32_t *faces_id_buffer,
                            int batch_size, int num_faces, int texture_size, int image_size,
                            int max_faces_id, float near, float far, float eps, float sigma_val,
                            int func_id_dist, float dist_eps, float gamma_val, int func_id_rgb,
                            int func_id_alpha, int texture_sample_type, int double_side,
                            int row_begin, int row_end, int row_stride, int nthreads) {
    const size_t npix = (size_t)image_size * image_size;
    memset(aggrs_info, 0, sizeof(float) * 2 * npix * batch_size);
    memset(soft_colors, 0, sizeof(float) * 4 * npix * batch_size); /* background is always 0 (Q1) */
    memset(faces_id_buffer, 0xFF, sizeof(int32_t) * (size_t)max_faces_id * npix * batch_size);
    softras_oracle_face_info(faces, faces_info, batch_size, num_faces);
    const int texture_res = (int)sqrt((double)texture_size); /* :475 */
    forward_rows(faces, textures, faces_info, aggrs_info, soft_colors, faces_id_buffer, batch_size,
                 num_faces, image_size, max_faces_id, texture_size, texture_res, near, far, eps,
                 sigma_val, func_id_dist, dist_eps, gamma_val, func_id_rgb, func_id_alpha,
                 texture_sample_type, double_side, row_begin, row_end, row_stride, nthreads, NULL);
}

/* softras_oracle_forward with the kernel's error bound per output entry ("rounding sites of the K2 forward"):
 * bound_colors [B,4,H,W] on |CUDA soft_colors - this file's|, bound_sum [B,H,W] on softmax_sum (aggrs_info channel 0;
 * 0 where it is not the softmax sum), marginal [B,H,W] FWD_MARG_* bits, live [B,H,W] the sites live in the pixel.
 * exact_tail: the kernel's softras_exact_tail.  nudge != 0: the outputs are the nudged forward (the bounds then mean
 * nothing).  Rows outside row_begin + i row_stride keep the memsets' values and bound 0. */
void softras_oracle_forward_bound(const float *faces, const float *textures, float *faces_info,
                                  float *aggrs_info, float *soft_colors, int32_t *faces_id_buffer,
                                  int batch_size, int num_faces, int texture_size, int image_size,
                                  int max_faces_id, float near, float far, float eps, float sigma_val,
                                  int func_id_dist, float dist_eps, float gamma_val, int func_id_rgb,
                                  int func_id_alpha, int texture_sample_type, int double_side, int exact_tail,
                                  int nudge, double *bound_colors, double *bound_sum, int32_t *marginal,
                                  uint32_t *live, int row_begin, int row_end, int row_stride, int nthreads) {
    const size_t npix = (size_t)image_size * image_size;
    memset(aggrs_info, 0, sizeof(float) * 2 * npix * batch_size);
    memset(soft_colors, 0, sizeof(float) * 4 * npix * batch_size);
    memset(faces_id_buffer, 0xFF, sizeof(int32_t) * (size_t)max_faces_id * npix * batch_size);
    memset(bound_colors, 0, sizeof(double) * 4 * npix * batch_size);
    memset(bound_sum, 0, sizeof(double) * npix * batch_size);
    memset(marginal, 0, sizeof(int32_t) * npix * batch_size);
    memset(live, 0, sizeof(uint32_t) * npix * batch_size);
    softras_oracle_face_info(faces, faces_info, batch_size, num_faces);
    const int texture_res = (int)sqrt((double)texture_size);
    const FwdBound fb = {exact_tail, nudge, bound_colors, bound_sum, marginal, live};
    forward_rows(faces, textures, faces_info, aggrs_info, soft_colors, faces_id_buffer, batch_size,
                 num_faces, image_size, max_faces_id, texture_size, texture_res, near, far, eps,
                 sigma_val, func_id_dist, dist_eps, gamma_val, func_id_rgb, func_id_alpha,
                 texture_sample_type, double_side, row_begin, row_end, row_stride, nthreads, &fb);
}

/* ------------------------------------------------------------------ K6 :1177-1360
 * The terms of one (pixel, face) pair: gv[k*3+l] for grad_faces[fn][k][l]; when it returns 1, gtex[3*j+k] for
 * grad_textures[fn][j][k] (j < texture_size; 0 for texels the pair does not hit).  nd: rounding sites (NULL: none). */
typedef struct {
    int nf, texture_size, texture_res, func_id_dist, func_id_rgb, func_id_alpha, texture_sample_type;
    float near, far, sigma_val, gamma_val;
} BwdParams;

static int pair_terms(const BwdParams *P, const float *face, const float *texture, const float *face_info, int fn,
                      float xp, float yp, const float g[4], const float oc[4], float softmax_sum, float softmax_max,
                      Nudge *nd, float gv[9], float *gtex) {
    const int texture_size = P->texture_size, texture_res = P->texture_res, texture_sample_type = P->texture_sample_type;
    const float near = P->near, far = P->far, sigma_val = P->sigma_val, gamma_val = P->gamma_val;
    float dis = 0, dis_x = 0, dis_y = 0, t[3] = {0, 0, 0}, w[3], w0[3], sign = 0, soft_fragment;
    int tex_written = 0;

    barycentric_coordinate(w, xp, yp, face_info);

    if (P->func_id_dist == 0) {
        soft_fragment = 1;
    } else {
        float x;
        if (P->func_id_dist == 1) {
            dis = forward_barycentric_p2f_distance(w);
            for (int k = 0; k < 3; k++) t[k] = w[k];
            x = rdiv(nd, SITE_DIV_SIGARG, -dis, sigma_val);
        } else {
            euclidean_p2f_distance(&sign, &dis_x, &dis_y, w, t, face, face_info, xp, yp, nd);
            dis = dis_x * dis_x + dis_y * dis_y;
            x = rdiv(nd, SITE_DIV_SIGARG, -sign * dis, sigma_val);
        }
        const float e = fmaxf(site(nd, SITE_EXP_SIG, expf(x), 3), 0.f);
        soft_fragment = (float)(1. / (1. + (double)e));
        if (nd && !nd->exact_tail) soft_fragment = fminf(fmaxf(site(nd, SITE_TAIL_D, soft_fragment, 2), 0.f), 1.f);
    }

    float grad_v[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    float C_grad_xy = 0;

    float C_grad_xy_alpha = g[3];
    if (P->func_id_alpha == 0) {
    } else if (P->func_id_alpha == 1) {
        C_grad_xy_alpha /= P->nf;
    } else if (P->func_id_alpha == 2) {
        C_grad_xy_alpha = (float)((double)C_grad_xy_alpha * ((double)(1 - oc[3]) / fmax((double)(1 - soft_fragment), 1e-6)));
        if (nd && !nd->exact_tail) C_grad_xy_alpha = site(nd, SITE_PROD, C_grad_xy_alpha, 4);
    }
    C_grad_xy += C_grad_xy_alpha;

    for (int k = 0; k < 3; k++) w0[k] = w[k];
    /* barycentric_clip (:49-54) and zp (:1296) */
    for (int k = 0; k < 3; k++) w[k] = (float)fmax(fmin((double)w[k], 1.), 0.);
    const float w_sum = (float)fmax((double)(w[0] + w[1] + w[2]), 1e-5);
    for (int k = 0; k < 3; k++) w[k] = rdiv(nd, SITE_DIV_CLIPW + k, w[k], w_sum);
    const float zp = (float)(1. / (double)(rdiv(nd, SITE_DIV_CLIPZ + 0, w[0], face[2]) + rdiv(nd, SITE_DIV_CLIPZ + 1, w[1], face[5]) +
                                           rdiv(nd, SITE_DIV_CLIPZ + 2, w[2], face[8])));

    if (P->func_id_rgb == 0) {
        if ((float)fn == softmax_max) { /* int vs float compare, Q10 */
            tex_written = 1;
            for (int k = 0; k < 3; k++)
                for (int j = 0; j < texture_size; j++)
                    gtex[3 * j + k] = backward_sample_texture(g[k], w, texture_res, j, texture_sample_type);
        }
    } else if (P->func_id_rgb == 1) {
        tex_written = 1;
        float C_grad_xyz_rgb = 0.f;
        const float zp_norm = (far - zp) / (far - near);
        const float e = fmaxf(site(nd, SITE_EXP_SOFT, expf((zp_norm - softmax_max) / gamma_val), 3), 0.f);
        const float zp_softmax = rdiv(nd, SITE_DIV_ZSOFT, soft_fragment * e, softmax_sum);

        for (int k = 0; k < 3; k++) {
            for (int j = 0; j < texture_size; j++)
                gtex[3 * j + k] = zp_softmax * backward_sample_texture(g[k], w, texture_res, j, texture_sample_type);
            const float color_k = forward_sample_texture_bwd(texture, w, texture_res, k, texture_sample_type);
            C_grad_xyz_rgb += g[k] * (color_k - oc[k]);
        }
        C_grad_xyz_rgb *= zp_softmax;
        C_grad_xy += rdiv(nd, SITE_DIV_COLD, C_grad_xyz_rgb, soft_fragment);

        const float C_grad_z_rgb = rdiv(nd, SITE_DIV_NMF, rdiv(nd, SITE_DIV_GAMMA, C_grad_xyz_rgb, gamma_val), near - far) * zp * zp;
        for (int k = 0; k < 3; k++)
            grad_v[k][2] = rdiv(nd, SITE_DIV_Z2 + k, rdiv(nd, SITE_DIV_Z1 + k, C_grad_z_rgb * w[k], face[3 * k + 2]), face[3 * k + 2]);
    }

    C_grad_xy *= rdiv(nd, SITE_DIV_SIGMA, soft_fragment * (1 - soft_fragment), sigma_val);
    if (P->func_id_dist == 1) {
        backward_barycentric_p2f_distance(grad_v, t, face_info, xp, yp, dis, C_grad_xy);
    } else if (P->func_id_dist == 2) {
        for (int k = 0; k < 3; k++)
            for (int l = 0; l < 2; l++)
                grad_v[k][l] = 2 * sign * C_grad_xy * (t[k] + w0[k]) * (l == 0 ? dis_x : dis_y);
    }
    for (int k = 0; k < 3; k++)
        for (int l = 0; l < 3; l++) gv[3 * k + l] = grad_v[k][l];
    return tex_written;
}

/* Walks the pairs of K6 in the reference's sequential order (pixels in ascending linear index, slots m ascending)
 * and hands each one's terms to visit(). */
typedef void (*PairVisitor)(void *ctx, const BwdParams *P, const float *face, const float *texture,
                            const float *face_info, int fn, long pair, float xp, float yp, const float g[4],
                            const float oc[4], float softmax_sum, float softmax_max, size_t gfo, size_t gto);

static void walk_pairs(const float *faces, const float *textures, const float *soft_colors, const float *faces_info,
                       const float *aggrs_info, const int32_t *faces_id_buffer, const float *grad_soft_colors,
                       const BwdParams *P, int batch_size, int image_size, int max_faces_id, float threshold,
                       int row_begin, int row_end, int row_stride, PairVisitor visit, void *ctx) {
    const int is = image_size, nf = P->nf, mf = max_faces_id, texture_size = P->texture_size;
    const long npix = (long)is * is;
    for (int bn = 0; bn < batch_size; bn++)
        for (int row = row_begin; row < row_end; row += (row_stride < 1 ? 1 : row_stride))
            for (int col = 0; col < is; col++) {
                const long pn = (long)row * is + col;
                const int yi = is - 1 - row;
                const int xi = col;
                const float yp = (float)((2. * yi + 1 - is) / is);
                const float xp = (float)((2. * xi + 1 - is) / is);
                const float softmax_sum = aggrs_info[((long)bn * 2 + 0) * npix + pn];
                const float softmax_max = aggrs_info[((long)bn * 2 + 1) * npix + pn];
                float g[4], oc[4];
                for (int k = 0; k < 4; k++) {
                    g[k] = grad_soft_colors[((long)bn * 4 + k) * npix + pn];
                    oc[k] = soft_colors[((long)bn * 4 + k) * npix + pn];
                }
                for (int m = 0; m < mf; m++) {
                    const int fn = faces_id_buffer[((long)bn * mf + m) * npix + pn];
                    if (fn == -1) break;
                    const float *face = &faces[((long)bn * nf + fn) * 9];
                    if (check_border(xp, yp, face, sqrtf(threshold))) continue;
                    visit(ctx, P, face, &textures[((long)bn * nf + fn) * texture_size * 3],
                          &faces_info[((long)bn * nf + fn) * 27], fn, ((long)bn * npix + pn) * mf + m, xp, yp, g, oc,
                          softmax_sum, softmax_max, ((size_t)bn * nf + fn) * 9, ((size_t)bn * nf + fn) * texture_size * 3);
                }
            }
}

static BwdParams bwd_params(int num_faces, int texture_size, float near, float far, float sigma_val, int func_id_dist,
                            float gamma_val, int func_id_rgb, int func_id_alpha, int texture_sample_type) {
    BwdParams P = {num_faces, texture_size, (int)sqrt((double)texture_size), func_id_dist, func_id_rgb, func_id_alpha,
                   texture_sample_type, near, far, sigma_val, gamma_val};
    return P;
}

typedef struct {
    int accumulate_double;
    double *gf, *gt;
    float *gtex;
} SumCtx;

static void acc(const SumCtx *c, double *buf, size_t idx, float val) {
    if (c->accumulate_double) buf[idx] += (double)val;
    else buf[idx] = (double)((float)buf[idx] + val);
}

static void sum_pair(void *ctx, const BwdParams *P, const float *face, const float *texture, const float *face_info,
                     int fn, long pair, float xp, float yp, const float g[4], const float oc[4], float softmax_sum,
                     float softmax_max, size_t gfo, size_t gto) {
    SumCtx *c = (SumCtx *)ctx;
    float gv[9];
    (void)pair;
    const int tw = pair_terms(P, face, texture, face_info, fn, xp, yp, g, oc, softmax_sum, softmax_max, NULL, gv, c->gtex);
    if (tw)
        for (int j = 0; j < 3 * P->texture_size; j++) acc(c, c->gt, gto + j, c->gtex[j]);
    for (int i = 0; i < 9; i++) acc(c, c->gf, gfo + i, gv[i]);
}

/* Sequential restatement: pixels in ascending linear index, slots m ascending,
 * `+=` in place of atomicAdd.  accumulate_double != 0 accumulates in double and
 * rounds once at the end (order-free centre for tolerance tests); 0 accumulates
 * in float exactly like a serialised execution of the reference.
 * faces_id_buffer layout [B, K, H, W] (the reference transposes to [B,H,W,K] on
 * the host first, soft_rasterize.py:108; the values read are the same). */
void softras_oracle_backward(const float *faces, const float *textures, const float *soft_colors,
                             const float *faces_info, const float *aggrs_info,
                             const int32_t *faces_id_buffer, const float *grad_soft_colors,
                             float *grad_faces, float *grad_textures, int batch_size,
                             int num_faces, int texture_size, int image_size, int max_faces_id,
                             float near, float far, float eps, float sigma_val, int func_id_dist,
                             float dist_eps, float gamma_val, int func_id_rgb, int func_id_alpha,
                             int texture_sample_type, int double_side, int accumulate_double,
                             int row_begin, int row_end, int row_stride) {
    (void)eps;
    (void)double_side;
    const BwdParams P = bwd_params(num_faces, texture_size, near, far, sigma_val, func_id_dist, gamma_val, func_id_rgb,
                                   func_id_alpha, texture_sample_type);
    const size_t ngf = (size_t)batch_size * num_faces * 9;
    const size_t ngt = (size_t)batch_size * num_faces * texture_size * 3;
    SumCtx c = {accumulate_double, (double *)calloc(ngf, sizeof(double)), (double *)calloc(ngt, sizeof(double)),
                (float *)malloc(sizeof(float) * 3 * (size_t)texture_size)};
    walk_pairs(faces, textures, soft_colors, faces_info, aggrs_info, faces_id_buffer, grad_soft_colors, &P, batch_size,
               image_size, max_faces_id, dist_eps * sigma_val, row_begin, row_end, row_stride, sum_pair, &c);
    for (size_t i = 0; i < ngf; i++) grad_faces[i] = (float)c.gf[i];
    for (size_t i = 0; i < ngt; i++) grad_textures[i] = (float)c.gt[i];
    free(c.gf);
    free(c.gt);
    free(c.gtex);
}

/* Per-slot statistics of the K6 terms, over slots s = grad_faces index (< B*nf*9), then B*nf*9 + grad_textures index:
 *   g64[s]  double sum of the terms (what accumulate_double = 1 rounds),
 *   A[s]    sum of |term|,
 *   N[s]    number of pairs that write a term into the slot, zero or not: at least as many as the float additions the
 *           kernel makes into it,
 *   E[s]    sum over pairs of how far the kernel's term may be from this one: the largest |term moved - term| over
 *           the moves of the pair's first six live rounding sites to the corners of their budget box and of each site
 *           alone, plus, for every further live site (tiny-numerator divisions only), its own largest move.
 *           A term is monotone in each site's value within its budget except across a clamp, so its extremes over
 *           the box lie on those points.  Sites interact (moving expf can make a division site live, and D's and
 *           1 - D's roundings compound near D = 1), so the corners are taken jointly, not site by site.
 * exact_tail: the kernel's softras_exact_tail.  nudge: 0, or +1 / -1 / 2 to compute g64 (only) with every live site
 * moved by its budget up / down / by a hashed sign per pair and site.  term_val / term_slot (NULL or term_cap
 * entries): every non-zero term and its slot, in the sequential order. */
#define MAX_CORNER_SITES 6
typedef struct {
    int exact_tail, nudge;
    size_t ngf;
    double *g64, *A, *E;
    int32_t *N;
    float *base, *moved, *dmax, *dextra;
    float *term_val;
    int64_t *term_slot;
    long term_cap, nterms;
} StatsCtx;

static void stats_pair(void *ctx, const BwdParams *P, const float *face, const float *texture, const float *face_info,
                       int fn, long pair, float xp, float yp, const float g[4], const float oc[4], float softmax_sum,
                       float softmax_max, size_t gfo, size_t gto) {
    StatsCtx *c = (StatsCtx *)ctx;
    const int ns = 9 + 3 * P->texture_size;
    Nudge nd = {c->exact_tail, 0, 0, c->nudge == 2, (uint32_t)pair, 0};
    if (c->nudge == 1) nd.up = ~0u;
    if (c->nudge == -1) nd.down = ~0u;
    const int tw = pair_terms(P, face, texture, face_info, fn, xp, yp, g, oc, softmax_sum, softmax_max, &nd, c->base, c->base + 9);
    const int nslots = tw ? ns : 9;
    for (int i = 0; i < nslots; i++) c->dmax[i] = c->dextra[i] = 0.f;
    if (!c->nudge && nd.live) {
        int live[N_SITES], L = 0;
        for (int s = 0; s < N_SITES; s++)
            if (nd.live >> s & 1u) live[L++] = s;
        const int Lc = L < MAX_CORNER_SITES ? L : MAX_CORNER_SITES;
        const long ncorner = 1L << Lc;
        for (long p = 0; p < ncorner + 2 * L; p++) {
            Nudge n2 = {c->exact_tail, 0, 0, 0, (uint32_t)pair, 0};
            if (p < ncorner) {
                for (int i = 0; i < Lc; i++) {
                    if (p >> i & 1L) n2.up |= 1u << live[i];
                    else n2.down |= 1u << live[i];
                }
            } else if ((p - ncorner) & 1L) {
                n2.up = 1u << live[(p - ncorner) >> 1];
            } else {
                n2.down = 1u << live[(p - ncorner) >> 1];
            }
            pair_terms(P, face, texture, face_info, fn, xp, yp, g, oc, softmax_sum, softmax_max, &n2, c->moved, c->moved + 9);
            float *d_out = c->dmax;
            if (p >= ncorner && (int)((p - ncorner) >> 1) >= Lc) d_out = c->dextra;   /* a site past the corners */
            for (int i = 0; i < nslots; i++) {
                const float d = fabsf(c->moved[i] - c->base[i]);
                if (!(d <= d_out[i])) d_out[i] = d;   /* NaN propagates */
            }
            if (d_out == c->dextra && ((p - ncorner) & 1L))   /* both directions of this site done */
                for (int i = 0; i < nslots; i++) {
                    c->E[i < 9 ? gfo + i : c->ngf + gto + (i - 9)] += c->dextra[i];
                    c->dextra[i] = 0.f;
                }
        }
    }
    for (int i = 0; i < nslots; i++) {
        const size_t s = i < 9 ? gfo + i : c->ngf + gto + (i - 9);
        const float v = c->base[i];
        c->g64[s] += (double)v;
        c->E[s] += c->dmax[i];
        c->N[s]++;
        if (v != 0.f) {
            c->A[s] += fabs((double)v);
            if (c->term_val && c->nterms < c->term_cap) {
                c->term_val[c->nterms] = v;
                c->term_slot[c->nterms] = (int64_t)s;
            }
            c->nterms++;
        }
    }
}

/* returns the number of non-zero terms */
long softras_oracle_backward_stats(const float *faces, const float *textures, const float *soft_colors,
                                   const float *faces_info, const float *aggrs_info,
                                   const int32_t *faces_id_buffer, const float *grad_soft_colors,
                                   double *g64, double *A, int32_t *N, double *E, int batch_size,
                                   int num_faces, int texture_size, int image_size, int max_faces_id,
                                   float near, float far, float eps, float sigma_val, int func_id_dist,
                                   float dist_eps, float gamma_val, int func_id_rgb, int func_id_alpha,
                                   int texture_sample_type, int double_side, int exact_tail, int nudge,
                                   int row_begin, int row_end, int row_stride,
                                   float *term_val, int64_t *term_slot, long term_cap) {
    (void)eps;
    (void)double_side;
    const BwdParams P = bwd_params(num_faces, texture_size, near, far, sigma_val, func_id_dist, gamma_val, func_id_rgb,
                                   func_id_alpha, texture_sample_type);
    const size_t ngf = (size_t)batch_size * num_faces * 9;
    const size_t ns = ngf + (size_t)batch_size * num_faces * texture_size * 3;
    const size_t np = 9 + 3 * (size_t)texture_size;
    StatsCtx c = {exact_tail, nudge, ngf, g64, A, E, N, (float *)malloc(sizeof(float) * np),
                  (float *)malloc(sizeof(float) * np), (float *)malloc(sizeof(float) * np), (float *)malloc(sizeof(float) * np),
                  term_val, term_slot, term_cap, 0};
    memset(g64, 0, sizeof(double) * ns);
    memset(A, 0, sizeof(double) * ns);
    memset(E, 0, sizeof(double) * ns);
    memset(N, 0, sizeof(int32_t) * ns);
    walk_pairs(faces, textures, soft_colors, faces_info, aggrs_info, faces_id_buffer, grad_soft_colors, &P, batch_size,
               image_size, max_faces_id, dist_eps * sigma_val, row_begin, row_end, row_stride, stats_pair, &c);
    free(c.base);
    free(c.moved);
    free(c.dmax);
    free(c.dextra);
    return c.nterms;
}

/* Multi-threaded timing variant for the CPU baseline (bench.py): thread t runs the sequential
 * restatement above on rows row_begin + t*stride, + nthreads*stride, ... into private
 * gradient buffers (double accumulation), which are then summed -- SURVEY.md 8(d)'s
 * "per-thread private grad buffers reduced at the end".  Not used by the parity tests. */
void softras_oracle_backward_mt(const float *faces, const float *textures, const float *soft_colors,
                                const float *faces_info, const float *aggrs_info,
                                const int32_t *faces_id_buffer, const float *grad_soft_colors,
                                float *grad_faces, float *grad_textures, int batch_size,
                                int num_faces, int texture_size, int image_size, int max_faces_id,
                                float near, float far, float eps, float sigma_val, int func_id_dist,
                                float dist_eps, float gamma_val, int func_id_rgb, int func_id_alpha,
                                int texture_sample_type, int double_side,
                                int row_begin, int row_end, int row_stride, int nthreads) {
    const size_t ngf = (size_t)batch_size * num_faces * 9;
    const size_t ngt = (size_t)batch_size * num_faces * texture_size * 3;
    if (row_stride < 1) row_stride = 1;
    if (nthreads < 1) nthreads = 1;
    float *pf = (float *)calloc(ngf * nthreads, sizeof(float));
    float *pt = (float *)calloc(ngt * nthreads, sizeof(float));
#pragma omp parallel for schedule(static, 1) num_threads(nthreads)
    for (int t = 0; t < nthreads; t++)
        softras_oracle_backward(faces, textures, soft_colors, faces_info, aggrs_info, faces_id_buffer,
                                grad_soft_colors, pf + ngf * t, pt + ngt * t, batch_size, num_faces,
                                texture_size, image_size, max_faces_id, near, far, eps, sigma_val,
                                func_id_dist, dist_eps, gamma_val, func_id_rgb, func_id_alpha,
                                texture_sample_type, double_side, 1, row_begin + t * row_stride, row_end,
                                row_stride * nthreads);
#pragma omp parallel for schedule(static) num_threads(nthreads)
    for (long i = 0; i < (long)ngf; i++) {
        double a = 0;
        for (int t = 0; t < nthreads; t++) a += pf[ngf * t + i];
        grad_faces[i] = (float)a;
    }
#pragma omp parallel for schedule(static) num_threads(nthreads)
    for (long i = 0; i < (long)ngt; i++) {
        double a = 0;
        for (int t = 0; t < nthreads; t++) a += pt[ngt * t + i];
        grad_textures[i] = (float)a;
    }
    free(pf);
    free(pt);
}

int softras_oracle_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
