// screen_space_api.cu -- the render2 image passes that read G-buffers: screen-space ambient occlusion, directional
// occlusion and FXAA (jrender/render2/utils/cuda/SSAO_cuda.py:108-172, SSDO_cuda.py:120-206, FXAA_cuda.py:37-249).
//
//   b200r_ssao / b200r_ssdo  one launch, one thread per pixel.  The reference allocates a curandStateXORWOW_t (48 B) per
//                            pixel, runs an init kernel and synchronises the device on every call; here each thread
//                            runs curand_init(1, i, 0) into registers, so a call allocates nothing, never synchronises
//                            and can be captured in a CUDA graph.  The draws are the same: same generator, same seed,
//                            same subsequence, same order (x, y, z of each sample).
//   b200r_fxaa               one launch.  The reference's edge search is dead code (its `uv1 -= offset` / `uv2 +=
//                            offset` call free operators that return a new value), so both ends stay one pixel away,
//                            the edge offset is 0.5 - 1 / 2 = 0, and the result is the centre colour or one bilinear
//                            sample at the sub-pixel offset.  That is what fxaa_pixel computes, without the ten
//                            resamples whose results are never used.
//
// Arithmetic: this library builds with -fmad=false; the reference builds with nvcc defaults, which contract a*b+c.  Every
// fmaf / fma below stands where the reference's sm_90a SASS has an FFMA / DFMA, with its operands in the same roles, and
// every other operation is a separately rounded one in the reference's order, so the results are the reference's bit
// for bit (oracle/screen_space.py restates them in numpy).  Double precision is kept where the reference's double
// literals put it: pi, 0.01, the luma weights and the FXAA thresholds.
#include <curand_kernel.h>
#include <limits.h>
#include <math.h>

#include "../../include/b200raster.h"
#include "api_util.cuh"

namespace {

constexpr int kThreads = 256;
constexpr double kPi = 3.1415926;   // the reference's `#define pi 3.1415926`, a double

// What SSAO and SSDO share: the pixel's view-space point and its tangent frame; screen_sample then draws each sample in
// the half ball of radius r on the normal's side of that point and finds the flat index of the pixel it projects to.
struct ScreenFrame {
    float wx, wy, wz;   // wcoord
    float nx, ny, nz;   // N
    float tx, ty, tz;   // T
    float bx, by, bz;   // B = T x N
};

__device__ __forceinline__ ScreenFrame screen_frame(int i, int is, const float* __restrict__ depth,
                                                    const float* __restrict__ normals, float width) {
    ScreenFrame f;
    const float fis = (float)is;
    const float xi = (2.f * (float)(i % is) + 1.f - fis) / fis;
    const float yi = (2.f * ((float)(is - 1) - (float)(i / is)) + 1.f - fis) / fis;
    const float d = depth[i];
    f.nx = normals[i * 3 + 0];
    f.ny = normals[i * 3 + 1];
    f.nz = normals[i * 3 + 2];
    f.wx = xi * width * d;
    f.wy = yi * width * d;
    f.wz = d;
    if (fabsf(f.nx) > 0.5f || fabsf(f.ny) > 0.5f) {   // T = (-N.y, N.x, 0), normalised
        const float r = rsqrtf(fmaf(f.nx, f.nx, f.ny * f.ny) + 0.f);
        f.tx = -f.ny * r;
        f.ty = f.nx * r;
        f.tz = 0.f * r;
    } else {                                          // T = (N.z, 0, -N.x), normalised
        const float r = rsqrtf(fmaf(f.nx, f.nx, fmaf(f.nz, f.nz, 0.f)));
        f.tx = f.nz * r;
        f.ty = 0.f * r;
        f.tz = -f.nx * r;
    }
    f.bx = fmaf(f.ty, f.nz, -(f.tz * f.ny));
    f.by = fmaf(f.tz, f.nx, -(f.tx * f.nz));
    f.bz = fmaf(f.tx, f.ny, -(f.ty * f.nx));
    return f;
}

// One sample: three draws -> the point p (randp) and the flat index of the pixel it projects to.  The index follows the
// reference's integer arithmetic: round() through the saturating float-to-int conversion, the row taken from is - row,
// and row * is + column evaluated in size_t and truncated to int, so a column off either side of the image lands in the
// neighbouring row and only the flat index is range-checked (by the caller).
__device__ __forceinline__ int screen_sample(const ScreenFrame& f, curandStateXORWOW_t* s, int is, float r, float width,
                                             float* px, float* py, float* pz) {
    const float ux = curand_uniform(s);
    const float uy = curand_uniform(s);
    const float uz = curand_uniform(s);
    const float randr = sqrtf(uz / 3.f);
    const double a = 2 * kPi * (double)ux;
    const float ry = randr * uy;
    const float lx = (float)((double)ry * cos(a));
    const float ly = randr * sqrtf(fmaf(-uy, uy, 1.f));
    const float lz = (float)((double)ry * sin(a));
    const float sx = fmaf(f.bx, lz, fmaf(f.tx, lx, f.nx * ly));
    const float sy = fmaf(f.by, lz, fmaf(f.ty, lx, f.ny * ly));
    const float sz = fmaf(f.bz, lz, fmaf(f.tz, lx, f.nz * ly));
    *px = fmaf(sx, r, f.wx);
    *py = fmaf(sy, r, f.wy);
    *pz = fmaf(sz, r, f.wz);
    const float fis = (float)is;
    const int col = (int)roundf(fis * (*px / *pz / width + 1.f) * 0.5f);
    const int row = (int)(fis - roundf(fis * (*py / *pz / width + 1.f) * 0.5f));
    return (int)((unsigned)row * (unsigned)is + (unsigned)col);
}

__global__ void __launch_bounds__(kThreads)
k_ssao(const float* __restrict__ depth, const int* __restrict__ face_ind, const float* __restrict__ normals,
       float* __restrict__ occlusion, int is, int sample_num, float r, float width) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    const int np = is * is;
    if (i >= np) return;
    if (face_ind[i] == -1) {
        occlusion[i] = 0.f;
        return;
    }
    const ScreenFrame f = screen_frame(i, is, depth, normals, width);
    curandStateXORWOW_t s;
    curand_init(1, i, 0, &s);
    float occ = 0.f;
    for (int k = 0; k < sample_num; k++) {
        float px, py, pz;
        const int j = screen_sample(f, &s, is, r, width, &px, &py, &pz);
        if (j >= np || j < 0) continue;
        if (depth[j] < pz) occ = occ + 1.f;
    }
    occlusion[i] = occ / (float)sample_num;
}

__global__ void __launch_bounds__(kThreads)
k_ssdo(const float* __restrict__ color, const float* __restrict__ depth, const int* __restrict__ face_ind,
       const float* __restrict__ normals, float* __restrict__ image, int is, int sample_num, float r, float width) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    const int np = is * is;
    if (i >= np) return;
    if (face_ind[i] == -1) {
        image[3 * i + 0] = color[3 * i + 0];
        image[3 * i + 1] = color[3 * i + 1];
        image[3 * i + 2] = color[3 * i + 2];
        return;
    }
    const ScreenFrame f = screen_frame(i, is, depth, normals, width);
    curandStateXORWOW_t s;
    curand_init(1, i, 0, &s);
    const float rho = 0.2f;
    const float area = 1.f / (float)sample_num * r * r;   // light_area_per_sample
    float ambient = 0.f, ind_r = 0.f, ind_g = 0.f, ind_b = 0.f;
    for (int k = 0; k < sample_num; k++) {
        float px, py, pz;
        const int j = screen_sample(f, &s, is, r, width, &px, &py, &pz);
        if (j >= np || j < 0) continue;
        if ((double)depth[j] > (double)pz - 0.01) {
            ambient = ambient + 1.f;
            continue;
        }
        // one bounce from the sample's pixel
        float dx = px - f.wx, dy = py - f.wy, dz = pz - f.wz;
        const float d2 = fmaf(dz, dz, fmaf(dx, dx, dy * dy));
        const float dist = sqrtf(d2);
        const float rm = rsqrtf(d2);
        dx = dx * rm;
        dy = dy * rm;
        dz = dz * rm;
        const float* n = normals + 3 * j;
        const float cos_rn = (float)fmax((double)-fmaf(n[2], dz, fmaf(n[0], dx, n[1] * dy)), 0.);
        const float cos_n = (float)fmax((double)fmaf(f.nz, dz, fmaf(f.nx, dx, f.ny * dy)), 0.);
        const float w = rho * cos_rn * cos_n * area / (dist * dist);
        const float* c = color + 3 * j;
        ind_r = fmaf(c[0], w, ind_r);
        ind_g = fmaf(c[1], w, ind_g);
        ind_b = fmaf(c[2], w, ind_b);
    }
    ambient = ambient / (float)sample_num;
    image[3 * i + 0] = fmaf(ambient, color[3 * i + 0], ind_r);
    image[3 * i + 1] = fmaf(ambient, color[3 * i + 1], ind_g);
    image[3 * i + 2] = fmaf(ambient, color[3 * i + 2], ind_b);
}

struct Rgb {
    float r, g, b;
};

// tex_sample (FXAA_cuda.py:37-53): bilinear read at (xp, yp), y up, clamped to the image the reference's way (in double,
// so a NaN coordinate becomes 0).  The four taps are (x, y), (x, y + 1), (x + 1, y), (x + 1, y + 1) of the flipped row
// index; a tap past the last pixel is the reference's read past the image, at weight 0, and counts as 0 here.  A tap at
// x + 1 of the last column is the first pixel of the next row, read as the reference reads it.
__device__ __forceinline__ Rgb tex_sample(const float* __restrict__ tex, float xp, float yp, int is) {
    const double hi = (double)(float)(is - 1);
    xp = (float)fmin(fmax((double)xp, 0.), hi);
    yp = (float)fmin(fmax((double)yp, 0.), hi);
    yp = (float)(is - 1) - yp;
    const int x0 = (int)xp, y0 = (int)yp;
    const float wx1 = xp - (float)x0, wx2 = 1.f - wx1;
    const float wy1 = yp - (float)y0, wy2 = 1.f - wy1;
    const int np = is * is;
    const int p[4] = {x0 + y0 * is, x0 + (y0 + 1) * is, x0 + 1 + y0 * is, x0 + 1 + (y0 + 1) * is};
    const float wa[4] = {wx2, wx2, wx1, wx1};
    const float wb[4] = {wy2, wy1, wy2, wy1};
    float c[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        float acc = 0.f;
#pragma unroll
        for (int t = 0; t < 4; t++) {
            const float v = p[t] < np ? tex[p[t] * 3 + k] : 0.f;
            acc = fmaf(wb[t], wa[t] * v, acc);
        }
        c[k] = acc;
    }
    return {c[0], c[1], c[2]};
}

// toluma: sqrtf of the double sum x 0.299 + y 0.587 + z 0.114 (contracted to two DFMAs), rounded to float first.
__device__ __forceinline__ float toluma(const Rgb& c) {
    return sqrtf((float)fma((double)c.b, 0.114, fma((double)c.r, 0.299, (double)c.g * 0.587)));
}

__device__ __forceinline__ Rgb fxaa_pixel(const float* __restrict__ tex, int i, int is) {
    const float ux = (float)(i % is), uy = (float)(is - 1) - (float)(i / is);
    const Rgb centre = tex_sample(tex, ux, uy, is);
    const float lc = toluma(centre);
    const float ll = toluma(tex_sample(tex, ux - 1.f, uy, is));
    const float lr = toluma(tex_sample(tex, ux + 1.f, uy, is));
    const float lu = toluma(tex_sample(tex, ux, uy + 1.f, is));
    const float ld = toluma(tex_sample(tex, ux, uy - 1.f, is));
    const float lmin = fminf(lc, fminf(fminf(ld, lu), fminf(ll, lr)));
    const float lmax = fmaxf(lc, fmaxf(fmaxf(ld, lu), fmaxf(ll, lr)));
    const float range = lmax - lmin;
    if ((double)range < fmax(0.0312, (double)lmax * 0.125)) return centre;
    const float lul = toluma(tex_sample(tex, ux - 1.f, uy + 1.f, is));
    const float lur = toluma(tex_sample(tex, ux + 1.f, uy + 1.f, is));
    const float ldl = toluma(tex_sample(tex, ux - 1.f, uy - 1.f, is));
    const float ldr = toluma(tex_sample(tex, ux + 1.f, uy - 1.f, is));
    const float down_up = ld + lu, left_right = ll + lr;
    const float left_c = ldl + lul, down_c = ldl + ldr, right_c = ldr + lur, up_c = lur + lul;
    // The double sums are exact up to their one rounding each (every product is by a power of two).
    const float edge_h = (float)(fabs(-2.0 * ll + left_c) + fabs(-2.0 * lc + down_up) * 2.0 + fabs(-2.0 * lr + right_c));
    const float edge_v = (float)(fabs(-2.0 * lu + up_c) + fabs(-2.0 * lc + left_right) * 2.0 + fabs(-2.0 * ld + down_c));
    const bool horizontal = edge_h >= edge_v;
    const float g1 = (horizontal ? ld : ll) - lc;
    const float g2 = (horizontal ? lu : lr) - lc;
    const float step = fabsf(g1) >= fabsf(g2) ? -1.f : 1.f;
    // sub-pixel offset; the edge offset it is compared with is always 0
    const float avg = (float)((1.0 / 12.0) * (2.0 * (double)(down_up + left_right) + left_c + right_c));
    const float s1 = (float)fmin(fmax((double)(fabsf(avg - lc) / range), 0.0), 1.0);
    const float s2 = (float)((-2.0 * s1 + 3.0) * s1 * s1);
    const float off = fmaxf(0.f, s2 * s2 * 0.75f);
    return horizontal ? tex_sample(tex, ux, fmaf(step, off, uy), is) : tex_sample(tex, fmaf(step, off, ux), uy, is);
}

__global__ void __launch_bounds__(kThreads) k_fxaa(const float* __restrict__ tex, float* __restrict__ image, int is) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= is * is) return;
    const Rgb c = fxaa_pixel(tex, i, is);
    image[i * 3 + 0] = c.r;
    image[i * 3 + 1] = c.g;
    image[i * 3 + 2] = c.b;
}

int check_size(const char* what, int is) {
    if (is < 1 || (long long)is * is * 3 > INT_MAX)
        return b200r_fail(B200R_EINVAL, "%s: image_size %d outside [1, %d]", what, is, 26754);
    return 0;
}

unsigned blocks(int is) { return (unsigned)(((long long)is * is + kThreads - 1) / kThreads); }

}  // namespace

extern "C" int b200r_ssao(const float* depth, const int32_t* face_ind, const float* normals, float* occlusion,
                          int image_size, int sample_num, float sample_range_r, float width, void* stream) {
    if (!depth || !face_ind || !normals || !occlusion) return b200r_fail(B200R_EINVAL, "b200r_ssao: NULL pointer argument");
    if (int rc = check_size("b200r_ssao", image_size)) return rc;
    if (sample_num < 0) return b200r_fail(B200R_EINVAL, "b200r_ssao: sample_num %d < 0", sample_num);
    return b200r_launch("k_ssao", B200R_K_SSS, k_ssao, blocks(image_size), kThreads, 0, (cudaStream_t)stream, depth,
                        face_ind, normals, occlusion, image_size, sample_num, sample_range_r, width);
}

extern "C" int b200r_ssdo(const float* color, const float* depth, const int32_t* face_ind, const float* normals,
                          float* image, int image_size, int sample_num, float sample_range_r, float width, void* stream) {
    if (!color || !depth || !face_ind || !normals || !image)
        return b200r_fail(B200R_EINVAL, "b200r_ssdo: NULL pointer argument");
    if (int rc = check_size("b200r_ssdo", image_size)) return rc;
    if (sample_num < 0) return b200r_fail(B200R_EINVAL, "b200r_ssdo: sample_num %d < 0", sample_num);
    return b200r_launch("k_ssdo", B200R_K_SSS, k_ssdo, blocks(image_size), kThreads, 0, (cudaStream_t)stream, color,
                        depth, face_ind, normals, image, image_size, sample_num, sample_range_r, width);
}

extern "C" int b200r_fxaa(const float* texture, float* image, int image_size, void* stream) {
    if (!texture || !image) return b200r_fail(B200R_EINVAL, "b200r_fxaa: NULL pointer argument");
    if (int rc = check_size("b200r_fxaa", image_size)) return rc;
    return b200r_launch("k_fxaa", B200R_K_SSS, k_fxaa, blocks(image_size), kThreads, 0, (cudaStream_t)stream, texture,
                        image, image_size);
}
