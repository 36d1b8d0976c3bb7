/*
 * nmr_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement (plain C, IEEE fp32/fp64, -ffp-contract=off) of the reference's Neural
 * Mesh Renderer (dr_type='n3mr') kernels.  Only tests/, __graft_entry__.smoke() and
 * bench.py's CPU-baseline legs may load this library.
 *
 * Follows jrender/renderer/dr/n3mr/cuda/rasterize.py (paths relative to /root/reference):
 *     :30-164   forward_face_index_map_cuda_kernel     (K7)
 *     :227-298  forward_texture_sampling_cuda_kernel   (K8)
 *     :351-610  backward_pixel_map_cuda_kernel         (K9)
 *     :659-694  backward_textures_cuda_kernel          (K10)
 *     :738-788  backward_depth_map_cuda_kernel         (K11)
 * host semantics: jrender/renderer/dr/n3mr/n3mr.py:29-67 (grad), :69-123 (execute),
 * :135-148 (background mix, alpha).
 *
 * Maps are indexed [b][yi][xi] with yi UP (row 0 = bottom), exactly as the kernels write them;
 * the vertical flip happens later on the host (n3mr.py:239-247).
 *
 * Determinism: K7 resolves its per-pixel z-test under a spin lock, so for faces with EQUAL
 * depth at a pixel the winner is race-dependent in the reference.  This oracle visits faces
 * in ascending id with the kernel's strict `zp < depth` test, i.e. the lowest face id wins
 * ties; the product kernels implement the same rule.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static inline int backside(const float *face) { /* :63, :377 */
    return (face[7] - face[1]) * (face[3] - face[0]) < (face[4] - face[1]) * (face[6] - face[0]);
}

/* ---------------------------------------------------------------- K7 :30-164 + fills :176-184 */
void nmr_oracle_face_index_map(const float *faces, int32_t *face_index_map, float *weight_map,
                               float *depth_map, float *face_inv_map /* may be NULL */,
                               int batch_size, int num_faces, int image_size, float near, float far,
                               int return_depth) {
    const int is = image_size;
    const size_t npix = (size_t)batch_size * is * is;
    for (size_t i = 0; i < npix; i++) face_index_map[i] = -1;     /* thrust::fill -1 */
    memset(weight_map, 0, sizeof(float) * 3 * npix);
    for (size_t i = 0; i < npix; i++) depth_map[i] = far;         /* thrust::fill far */
    if (face_inv_map) memset(face_inv_map, 0, sizeof(float) * 9 * npix);

    for (int bn = 0; bn < batch_size; bn++)
        for (int fn = 0; fn < num_faces; fn++) {
            const float *face = &faces[((size_t)bn * num_faces + fn) * 9];
            if (backside(face)) continue;

            float p[3][2];
            for (int num = 0; num < 3; num++)
                for (int dim = 0; dim < 2; dim++)
                    p[num][dim] = (float)(0.5 * (double)(face[3 * num + dim] * is + is - 1));

            float face_inv[9] = {
                p[1][1] - p[2][1], p[2][0] - p[1][0], p[1][0] * p[2][1] - p[2][0] * p[1][1],
                p[2][1] - p[0][1], p[0][0] - p[2][0], p[2][0] * p[0][1] - p[0][0] * p[2][1],
                p[0][1] - p[1][1], p[1][0] - p[0][0], p[0][0] * p[1][1] - p[1][0] * p[0][1]};
            const float den = (p[2][0] * (p[0][1] - p[1][1]) + p[0][0] * (p[1][1] - p[2][1]) + p[1][0] * (p[2][1] - p[0][1]));
            for (int k = 0; k < 9; k++) face_inv[k] /= den;

            float x_min = (float)is, y_min = (float)is, x_max = 0, y_max = 0;
            for (int num = 0; num < 3; num++) {
                if (p[num][0] < x_min) x_min = p[num][0];
                if (p[num][0] > x_max) x_max = p[num][0];
                if (p[num][1] < y_min) y_min = p[num][1];
                if (p[num][1] > y_max) y_max = p[num][1];
            }
            int ix_min = (int)x_min > 0 ? (int)x_min : 0;
            int ix_max = (int)x_max < is - 1 ? (int)x_max : is - 1;
            int iy_min = (int)y_min > 0 ? (int)y_min : 0;
            int iy_max = (int)y_max < is - 1 ? (int)y_max : is - 1;

            for (int xi = ix_min; xi <= ix_max; xi++)
                for (int yi = iy_min; yi <= iy_max; yi++) {
                    const float yp = (float)((2. * yi + 1 - is) / is);
                    const float xp = (float)((2. * xi + 1 - is) / is);
                    if (((yp - face[1]) * (face[3] - face[0]) < (xp - face[0]) * (face[4] - face[1])) ||
                        ((yp - face[4]) * (face[6] - face[3]) < (xp - face[3]) * (face[7] - face[4])) ||
                        ((yp - face[7]) * (face[0] - face[6]) < (xp - face[6]) * (face[1] - face[7])))
                        continue;

                    const size_t i1 = (size_t)bn * is * is + (size_t)yi * is + xi;
                    float w[3];
                    w[0] = face_inv[0] * xi + face_inv[1] * yi + face_inv[2];
                    w[1] = face_inv[3] * xi + face_inv[4] * yi + face_inv[5];
                    w[2] = face_inv[6] * xi + face_inv[7] * yi + face_inv[8];
                    float w_sum = 0;
                    for (int k = 0; k < 3; k++) {
                        w[k] = (float)fmin(fmax((double)w[k], 0.), 1.);
                        w_sum += w[k];
                    }
                    for (int k = 0; k < 3; k++) w[k] /= w_sum;
                    const float zp = (float)(1. / (double)(w[0] / face[2] + w[1] / face[5] + w[2] / face[8]));
                    if (zp <= near || far <= zp) continue;
                    if (zp < depth_map[i1]) {
                        depth_map[i1] = zp;
                        face_index_map[i1] = fn;
                        for (int k = 0; k < 3; k++) weight_map[3 * i1 + k] = w[k];
                        if (return_depth && face_inv_map)
                            for (int k = 0; k < 9; k++) face_inv_map[9 * i1 + k] = face_inv[k];
                    }
                }
        }
}

/* ---------------------------------------------------------------- K8 :227-298 + memsets :311-313 */
void nmr_oracle_texture_sampling(const float *faces, const float *textures, const int32_t *face_index_map,
                                 const float *weight_map, const float *depth_map, float *rgb_map,
                                 int32_t *sampling_index_map, float *sampling_weight_map,
                                 int batch_size, int num_faces, int image_size, int texture_size, float eps) {
    const int is = image_size, nf = num_faces, ts = texture_size;
    const size_t npix = (size_t)batch_size * is * is;
    memset(rgb_map, 0, sizeof(float) * 3 * npix);
    memset(sampling_index_map, 0, sizeof(int32_t) * 8 * npix);
    memset(sampling_weight_map, 0, sizeof(float) * 8 * npix);
    for (size_t i = 0; i < npix; i++) {
        const int face_index = face_index_map[i];
        if (face_index < 0) continue;
        const int bn = (int)(i / ((size_t)is * is));
        const float *face = &faces[((size_t)bn * nf + face_index) * 9];
        const float *texture = &textures[((size_t)bn * nf + face_index) * ts * ts * ts * 3];
        const float *weight = &weight_map[i * 3];
        const float depth = depth_map[i];
        float tif3[3];
        for (int k = 0; k < 3; k++) {
            float tif = weight[k] * (ts - 1) * (depth / (face[3 * k + 2]));
            tif = (float)fmax((double)tif, 0.);
            tif = fminf(tif, ts - 1 - eps);
            tif3[k] = tif;
        }
        float new_pixel[3] = {0, 0, 0};
        for (int pn = 0; pn < 8; pn++) {
            float w = 1;
            int tii[3];
            for (int k = 0; k < 3; k++) {
                if ((pn >> k) % 2 == 0) {
                    w *= 1 - (tif3[k] - (int)tif3[k]);
                    tii[k] = (int)tif3[k];
                } else {
                    w *= tif3[k] - (int)tif3[k];
                    tii[k] = (int)tif3[k] + 1;
                }
            }
            const int isc = tii[0] * ts * ts + tii[1] * ts + tii[2];
            /* texture_size 1 (the Mesh default texture_res, SURVEY.md 8d): ts - 1 - eps < 0, so the
             * "+1" taps index past the face's own block -- the reference reads the next faces'
             * texels (and, for the last faces, past the tensor: UB).  Restated as: taps inside the
             * tensor are read as the reference reads them, taps past its end contribute 0. */
            const size_t tap = ((size_t)bn * nf + face_index) * ts * ts * ts + (size_t)isc;
            if (isc >= 0 && tap < (size_t)batch_size * nf * ts * ts * ts)
                for (int k = 0; k < 3; k++) new_pixel[k] += w * texture[isc * 3 + k];
            sampling_index_map[i * 8 + pn] = isc;
            sampling_weight_map[i * 8 + pn] = w;
        }
        for (int k = 0; k < 3; k++) rgb_map[i * 3 + k] = new_pixel[k];
    }
}

/* ---------------------------------------------------------------- K9 :351-610 (+ memset :623) */
/* Optional per (face, gradient slot) statistics of K9's sums, for error bounds on kernels that add the same terms in
 * another order and with other roundings.  Per slot s of face i (arrays [B*nf*9], zeroed here; z slots stay 0):
 *   g64[s]   the sum, in double, of the float terms -diff_grad / dist that the float path adds;
 *   T[s]     the sum of their absolute values;
 *   R[s]     sum over every pixel a scan visits -- the inward scan's owner test applies, the `diff_grad <= 0` skip
 *            does not -- of (sum_k |map_k * grad_k| + |ref_k * grad_k|) / |dist|: the scale of a diff_grad that
 *            is formed as A - sum_k ref_k * grad_k, and of the terms whose diff_grad changes sign near 0;
 *   cnt[s]   the number of terms added;
 *   chain[s] a bound on the float additions any one term of the slot goes through in k_nmr_backward_pixel_map:
 *            the most pixels of the slot one lane visits (a sample's lane for inward scans of < 64 pixels,
 *            lane (d1 - d1_from) % 32 otherwise), plus 3 per group of 32 samples (one add of the lane's own inward
 *            sum and one flush of each of the two passes feeding the slot), plus 5 levels of the warp reduction. */
/* sum_k |map_k * grad_k| + |ref_k * grad_k| at pixel idx (double, exact products of floats) */
static inline double diff_mag(const float *rgb_map, const float *alpha_map, const float *grad_rgb_map,
                              const float *grad_alpha_map, long idx, const float *rgb_ref, float alpha_ref,
                              int return_rgb, int return_alpha) {
    double m = 0;
    if (return_alpha)
        m += fabs((double)alpha_map[idx] * grad_alpha_map[idx]) + fabs((double)alpha_ref * grad_alpha_map[idx]);
    if (return_rgb)
        for (int k = 0; k < 3; k++)
            m += fabs((double)rgb_map[idx * 3 + k] * grad_rgb_map[idx * 3 + k]) + fabs((double)rgb_ref[k] * grad_rgb_map[idx * 3 + k]);
    return m;
}

typedef struct {
    double *g64, *T, *R;
    int32_t *cnt, *chain;
} k9_stats;

/* one visited pixel of a scan: float term (the reference's), statistics */
static inline void k9_visit(float *grad_slot, int slot, float diff_grad, float dist, double mag, int lane,
                            double *g64, double *T, double *R, int32_t *cnt, int32_t lanes[9][32]) {
    if (g64) {
        R[slot] += mag / fabs((double)dist);
        lanes[slot][lane]++;
    }
    if (diff_grad <= 0) return;
    const float term = diff_grad / dist;
    *grad_slot -= term;
    if (g64) {
        g64[slot] -= (double)term;
        T[slot] += fabs((double)term);
        cnt[slot]++;
    }
}

static void backward_pixel_map(const float *faces, const int32_t *face_index_map, const float *rgb_map,
                               const float *alpha_map, const float *grad_rgb_map, const float *grad_alpha_map,
                               float *grad_faces, int batch_size, int num_faces, int image_size, float eps,
                               int return_rgb, int return_alpha, const k9_stats *st) {
    const int is = image_size;
    memset(grad_faces, 0, sizeof(float) * 9 * (size_t)batch_size * num_faces);
    if (st) {
        const size_t n = 9 * (size_t)batch_size * num_faces;
        memset(st->g64, 0, sizeof(double) * n);
        memset(st->T, 0, sizeof(double) * n);
        memset(st->R, 0, sizeof(double) * n);
        memset(st->cnt, 0, sizeof(int32_t) * n);
        memset(st->chain, 0, sizeof(int32_t) * n);
    }
    for (long i = 0; i < (long)batch_size * num_faces; i++) {
        const int bn = (int)(i / num_faces);
        const int fn = (int)(i % num_faces);
        const float *face = &faces[i * 9];
        float grad_face[9] = {0};
        if (backside(face)) continue;
        double *g64 = st ? st->g64 + i * 9 : NULL, *T = st ? st->T + i * 9 : NULL, *R = st ? st->R + i * 9 : NULL;
        int32_t *cnt = st ? st->cnt + i * 9 : NULL;
        int32_t lanes[9][32];
        memset(lanes, 0, sizeof(lanes));
        int sidx = -1; /* the kernel's sample number: pass-major, every d0 of every pass */

        for (int edge_num = 0; edge_num < 3; edge_num++) {
            int pi[3];
            float pp[3][2];
            for (int num = 0; num < 3; num++) pi[num] = (edge_num + num) % 3;
            for (int num = 0; num < 3; num++)
                for (int dim = 0; dim < 2; dim++)
                    pp[num][dim] = (float)(0.5 * (double)(face[3 * pi[num] + dim] * is + is - 1));

            for (int axis = 0; axis < 2; axis++) {
                float p[3][2];
                for (int num = 0; num < 3; num++)
                    for (int dim = 0; dim < 2; dim++) p[num][dim] = pp[num][(dim + axis) % 2];

                int direction;
                if (axis == 0) direction = (p[0][0] < p[1][0]) ? -1 : 1;
                else direction = (p[0][0] < p[1][0]) ? 1 : -1;

                const int d0_from = (int)fmax((double)ceilf(fminf(p[0][0], p[1][0])), 0.);
                const int d0_to = (int)fmin((double)fmaxf(p[0][0], p[1][0]), is - 1.);
                for (int d0 = d0_from; d0 <= d0_to; d0++) {
                    sidx++;
                    int d1_in, d1_out;
                    const float d1_cross = (p[1][1] - p[0][1]) / (p[1][0] - p[0][0]) * (d0 - p[0][0]) + p[0][1];
                    if (0 < direction) d1_in = (int)floorf(d1_cross);
                    else d1_in = (int)ceilf(d1_cross);
                    d1_out = d1_in + direction;
                    if (d1_in < 0 || is <= d1_in) continue;
                    if (d1_out < 0 || is <= d1_out) continue;

                    float alpha_in = 0, alpha_out = 0;
                    const float *rgb_in = NULL, *rgb_out = NULL;
                    long map_index_in, map_index_out;
                    if (axis == 0) {
                        map_index_in = (long)bn * is * is + (long)d1_in * is + d0;
                        map_index_out = (long)bn * is * is + (long)d1_out * is + d0;
                    } else {
                        map_index_in = (long)bn * is * is + (long)d0 * is + d1_in;
                        map_index_out = (long)bn * is * is + (long)d0 * is + d1_out;
                    }
                    if (return_alpha) {
                        alpha_in = alpha_map[map_index_in];
                        alpha_out = alpha_map[map_index_out];
                    }
                    if (return_rgb) {
                        rgb_in = &rgb_map[map_index_in * 3];
                        rgb_out = &rgb_map[map_index_out * 3];
                    }

                    /* out */
                    if (face_index_map[map_index_in] == fn) {
                        const int d1_limit = (0 < direction) ? is - 1 : 0;
                        int d1_from = d1_out < d1_limit ? d1_out : d1_limit; if (d1_from < 0) d1_from = 0;
                        int d1_to = d1_out > d1_limit ? d1_out : d1_limit; if (d1_to > is - 1) d1_to = is - 1;
                        const long map_offset = (axis == 0) ? is : 1;
                        long idx = (axis == 0) ? (long)bn * is * is + (long)d1_from * is + d0
                                               : (long)bn * is * is + (long)d0 * is + d1_from;
                        for (int d1 = d1_from; d1 <= d1_to; d1++, idx += map_offset) {
                            float diff_grad = 0;
                            if (return_alpha) diff_grad += (alpha_map[idx] - alpha_in) * grad_alpha_map[idx];
                            if (return_rgb)
                                for (int k = 0; k < 3; k++) diff_grad += (rgb_map[idx * 3 + k] - rgb_in[k]) * grad_rgb_map[idx * 3 + k];
                            const double mag = st ? diff_mag(rgb_map, alpha_map, grad_rgb_map, grad_alpha_map, idx, rgb_in, alpha_in,
                                                             return_rgb, return_alpha) : 0;
                            const int lane = (d1 - d1_from) % 32;
                            if (p[1][0] != d0) {
                                float dist = (float)((double)((p[1][0] - p[0][0]) / (p[1][0] - d0) * (d1 - d1_cross)) * 2. / is);
                                dist = (0 < dist) ? dist + eps : dist - eps;
                                const int slot = pi[0] * 3 + (1 - axis);
                                k9_visit(&grad_face[slot], slot, diff_grad, dist, mag, lane, g64, T, R, cnt, lanes);
                            }
                            if (p[0][0] != d0) {
                                float dist = (float)((double)((p[1][0] - p[0][0]) / (d0 - p[0][0]) * (d1 - d1_cross)) * 2. / is);
                                dist = (0 < dist) ? dist + eps : dist - eps;
                                const int slot = pi[1] * 3 + (1 - axis);
                                k9_visit(&grad_face[slot], slot, diff_grad, dist, mag, lane, g64, T, R, cnt, lanes);
                            }
                        }
                    }

                    /* in */
                    {
                        int d1_limit;
                        float d0_cross2;
                        if ((d0 - p[0][0]) * (d0 - p[2][0]) < 0)
                            d0_cross2 = (p[2][1] - p[0][1]) / (p[2][0] - p[0][0]) * (d0 - p[0][0]) + p[0][1];
                        else
                            d0_cross2 = (p[1][1] - p[2][1]) / (p[1][0] - p[2][0]) * (d0 - p[2][0]) + p[2][1];
                        if (0 < direction) d1_limit = (int)ceilf(d0_cross2);
                        else d1_limit = (int)floorf(d0_cross2);
                        int d1_from = d1_in < d1_limit ? d1_in : d1_limit; if (d1_from < 0) d1_from = 0;
                        int d1_to = d1_in > d1_limit ? d1_in : d1_limit; if (d1_to > is - 1) d1_to = is - 1;
                        const long map_offset = (axis == 0) ? is : 1;
                        long idx = (axis == 0) ? (long)bn * is * is + (long)d1_from * is + d0
                                               : (long)bn * is * is + (long)d0 * is + d1_from;
                        const int serial = d1_to - d1_from < 64; /* walked by the sample's own lane in the kernel */
                        for (int d1 = d1_from; d1 <= d1_to; d1++, idx += map_offset) {
                            if (face_index_map[idx] != fn) continue;
                            float diff_grad = 0;
                            if (return_alpha) diff_grad += (alpha_map[idx] - alpha_out) * grad_alpha_map[idx];
                            if (return_rgb)
                                for (int k = 0; k < 3; k++) diff_grad += (rgb_map[idx * 3 + k] - rgb_out[k]) * grad_rgb_map[idx * 3 + k];
                            const double mag = st ? diff_mag(rgb_map, alpha_map, grad_rgb_map, grad_alpha_map, idx, rgb_out, alpha_out,
                                                             return_rgb, return_alpha) : 0;
                            const int lane = serial ? sidx % 32 : (d1 - d1_from) % 32;
                            if (p[1][0] != d0) {
                                float dist = (float)((double)((p[1][0] - p[0][0]) / (p[1][0] - d0) * (d1 - d1_cross)) * 2. / is);
                                dist = (0 < dist) ? dist + eps : dist - eps;
                                const int slot = pi[0] * 3 + (1 - axis);
                                k9_visit(&grad_face[slot], slot, diff_grad, dist, mag, lane, g64, T, R, cnt, lanes);
                            }
                            if (p[0][0] != d0) {
                                float dist = (float)((double)((p[1][0] - p[0][0]) / (d0 - p[0][0]) * (d1 - d1_cross)) * 2. / is);
                                dist = (0 < dist) ? dist + eps : dist - eps;
                                const int slot = pi[1] * 3 + (1 - axis);
                                k9_visit(&grad_face[slot], slot, diff_grad, dist, mag, lane, g64, T, R, cnt, lanes);
                            }
                        }
                    }
                }
            }
        }
        for (int k = 0; k < 9; k++) grad_faces[i * 9 + k] = grad_face[k];
        if (st) {
            const int groups = (sidx + 1 + 31) / 32;
            for (int k = 0; k < 9; k++) {
                int m = 0;
                for (int l = 0; l < 32; l++) m = lanes[k][l] > m ? lanes[k][l] : m;
                st->chain[i * 9 + k] = m + 3 * groups + 5;
            }
        }
    }
}

void nmr_oracle_backward_pixel_map(const float *faces, const int32_t *face_index_map, const float *rgb_map,
                                   const float *alpha_map, const float *grad_rgb_map, const float *grad_alpha_map,
                                   float *grad_faces, int batch_size, int num_faces, int image_size, float eps,
                                   int return_rgb, int return_alpha) {
    backward_pixel_map(faces, face_index_map, rgb_map, alpha_map, grad_rgb_map, grad_alpha_map, grad_faces, batch_size,
                       num_faces, image_size, eps, return_rgb, return_alpha, NULL);
}

/* The float path above plus its statistics (see k9_stats). */
void nmr_oracle_backward_pixel_map_stats(const float *faces, const int32_t *face_index_map, const float *rgb_map,
                                         const float *alpha_map, const float *grad_rgb_map, const float *grad_alpha_map,
                                         float *grad_faces, int batch_size, int num_faces, int image_size, float eps,
                                         int return_rgb, int return_alpha, double *g64, double *T, double *R,
                                         int32_t *cnt, int32_t *chain) {
    const k9_stats st = {g64, T, R, cnt, chain};
    backward_pixel_map(faces, face_index_map, rgb_map, alpha_map, grad_rgb_map, grad_alpha_map, grad_faces, batch_size,
                       num_faces, image_size, eps, return_rgb, return_alpha, &st);
}

/* ---------------------------------------------------------------- K10 :659-694 (+ memset :705) */
/* absT / cnt (optional, [B*nf*ts^3*3]): sum of |term| and number of terms per texel channel; the double sum is
 * returned in acc64 when given. */
static void backward_textures(const int32_t *face_index_map, const float *sampling_weight_map,
                              const int32_t *sampling_index_map, const float *grad_rgb_map,
                              float *grad_textures, int batch_size, int num_faces, int image_size,
                              int texture_size, double *acc64, double *absT, int32_t *cnt) {
    const int is = image_size, nf = num_faces, ts = texture_size;
    const size_t ntex = (size_t)batch_size * nf * ts * ts * ts * 3;
    double *acc = acc64 ? acc64 : (double *)calloc(ntex, sizeof(double));
    if (acc64) memset(acc64, 0, sizeof(double) * ntex);
    if (absT) memset(absT, 0, sizeof(double) * ntex);
    if (cnt) memset(cnt, 0, sizeof(int32_t) * ntex);
    const size_t npix = (size_t)batch_size * is * is;
    for (size_t i = 0; i < npix; i++) {
        const int face_index = face_index_map[i];
        if (face_index < 0) continue;
        const int bn = (int)(i / ((size_t)is * is));
        const size_t base = ((size_t)bn * nf + face_index) * ts * ts * ts * 3;
        for (int pn = 0; pn < 8; pn++) {
            const float w = sampling_weight_map[i * 8 + pn];
            const int isc = sampling_index_map[i * 8 + pn];
            if (isc < 0 || base + (size_t)isc * 3 + 2 >= ntex) continue; /* tap past the tensor (ts == 1, see K8) */
            for (int k = 0; k < 3; k++) {
                const float term = w * grad_rgb_map[i * 3 + k];
                acc[base + (size_t)isc * 3 + k] += (double)term;
                if (absT) absT[base + (size_t)isc * 3 + k] += fabs((double)term);
                if (cnt) cnt[base + (size_t)isc * 3 + k]++;
            }
        }
    }
    for (size_t j = 0; j < ntex; j++) grad_textures[j] = (float)acc[j];
    if (!acc64) free(acc);
}

void nmr_oracle_backward_textures(const int32_t *face_index_map, const float *sampling_weight_map,
                                  const int32_t *sampling_index_map, const float *grad_rgb_map,
                                  float *grad_textures, int batch_size, int num_faces, int image_size,
                                  int texture_size) {
    backward_textures(face_index_map, sampling_weight_map, sampling_index_map, grad_rgb_map, grad_textures,
                      batch_size, num_faces, image_size, texture_size, NULL, NULL, NULL);
}

void nmr_oracle_backward_textures_stats(const int32_t *face_index_map, const float *sampling_weight_map,
                                        const int32_t *sampling_index_map, const float *grad_rgb_map,
                                        float *grad_textures, int batch_size, int num_faces, int image_size,
                                        int texture_size, double *g64, double *absT, int32_t *cnt) {
    backward_textures(face_index_map, sampling_weight_map, sampling_index_map, grad_rgb_map, grad_textures,
                      batch_size, num_faces, image_size, texture_size, g64, absT, cnt);
}

/* ---------------------------------------------------------------- K11 :738-788 (accumulates INTO grad_faces) */
/* acc64 / absT / cnt (optional, [B*nf*9]): K11's own double sum, sum of |term| and number of terms per slot */
static void backward_depth_map(const float *faces, const float *depth_map, const int32_t *face_index_map,
                               const float *face_inv_map, const float *weight_map, const float *grad_depth_map,
                               float *grad_faces, int batch_size, int num_faces, int image_size, double *acc64,
                               double *absT, int32_t *cnt) {
    const int is = image_size, nf = num_faces;
    const size_t ng = (size_t)batch_size * nf * 9;
    double *acc = acc64 ? acc64 : (double *)calloc(ng, sizeof(double));
    if (acc64) memset(acc64, 0, sizeof(double) * ng);
    if (absT) memset(absT, 0, sizeof(double) * ng);
    if (cnt) memset(cnt, 0, sizeof(int32_t) * ng);
    const size_t npix = (size_t)batch_size * is * is;
    for (size_t i = 0; i < npix; i++) {
        const int fn = face_index_map[i];
        if (fn < 0) continue;
        const int bn = (int)(i / ((size_t)is * is));
        const float *face = &faces[((size_t)bn * nf + fn) * 9];
        const float depth = depth_map[i];
        const float depth2 = depth * depth;
        const float *face_inv = &face_inv_map[i * 9];
        const float *weight = &weight_map[i * 3];
        const float grad_depth = grad_depth_map[i];
        const size_t o = ((size_t)bn * nf + fn) * 9;
        double *g = &acc[o];
        float term[9];
        for (int k = 0; k < 3; k++) {
            const float z_k = face[3 * k + 2];
            term[3 * k + 2] = grad_depth * weight[k] * depth2 / (z_k * z_k);
        }
        float tmp[3] = {0, 0, 0};
        for (int k = 0; k < 3; k++)
            for (int l = 0; l < 3; l++) tmp[k] += -face_inv[3 * l + k] / face[3 * l + 2];
        for (int k = 0; k < 3; k++)
            for (int l = 0; l < 2; l++) term[3 * k + l] = -grad_depth * tmp[l] * weight[k] * depth2 * is / 2;
        for (int s = 0; s < 9; s++) {
            g[s] += (double)term[s];
            if (absT) absT[o + s] += fabs((double)term[s]);
            if (cnt) cnt[o + s]++;
        }
    }
    for (size_t j = 0; j < ng; j++) grad_faces[j] = (float)((double)grad_faces[j] + acc[j]);
    if (!acc64) free(acc);
}

void nmr_oracle_backward_depth_map(const float *faces, const float *depth_map, const int32_t *face_index_map,
                                   const float *face_inv_map, const float *weight_map, const float *grad_depth_map,
                                   float *grad_faces, int batch_size, int num_faces, int image_size) {
    backward_depth_map(faces, depth_map, face_index_map, face_inv_map, weight_map, grad_depth_map, grad_faces,
                       batch_size, num_faces, image_size, NULL, NULL, NULL);
}

void nmr_oracle_backward_depth_map_stats(const float *faces, const float *depth_map, const int32_t *face_index_map,
                                         const float *face_inv_map, const float *weight_map, const float *grad_depth_map,
                                         float *grad_faces, int batch_size, int num_faces, int image_size, double *g64,
                                         double *absT, int32_t *cnt) {
    backward_depth_map(faces, depth_map, face_index_map, face_inv_map, weight_map, grad_depth_map, grad_faces,
                       batch_size, num_faces, image_size, g64, absT, cnt);
}
