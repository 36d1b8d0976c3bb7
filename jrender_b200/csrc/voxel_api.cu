// voxel_api.cu -- mesh voxelization (jrender/renderer/utils/voxelization.py:1-57, kernels in
// jrender/renderer/utils/cuda/voxelization.py).
//
//   b200r_voxelize_surface  <-  voxelize_sub1 (x3 axes, :5-16) + voxelize_sub2 (:18-22) + the OR of the four grids (:52-53)
//   b200r_voxelize_fill     <-  voxelize_sub3 / voxelize_sub4 and the host loop that relaunches sub4 until visible.sum()
//                               stops changing (:24-38), then 1 - visible
//
// Surface.  The reference gives a thread to every integer column (y, x) of every axis and tests it against every face
// (3 B vs^2 nf tests).  Here a thread takes one (batch, face) and, per axis, walks the columns of the face's projected
// bounding box only; boxes above kVoxSerialBox columns are then taken one at a time by the whole warp (k_nmr_zbuffer's
// scheme).  Every (face, column) test is the reference's float32 expression, operand for operand, unfused (-fmad=false).
// The box is only used when it provably holds every column the float test can accept (vox_box_proven); otherwise the
// face is tested against every column of that projection, as the reference does.  Result bits are therefore those of
// the all-columns loop.  One deliberate difference: the reference converts floor(z) to int before its range check, so
// a NaN depth becomes voxel 0; here the range check is done on the float, so non-finite depths write nothing.
//
// Fill.  visible = empty voxels 6-connected through empty voxels to an empty voxel on the grid boundary; the result is
// 1 - visible.  The reference iterates a racy in-place kernel with a host synchronisation per round.  Here the grid is
// packed to bits (32 voxels of a z-row per word), one CTA per image runs Gauss-Seidel sweeps in place until a sweep
// changes nothing (__syncthreads_or), and the result is unpacked: three launches, no host synchronisation.  Updates
// only ever add visible voxels that have a visible neighbour, so the sweep's fixed point is the unique answer whatever
// order rows are visited in.
#include "../../include/b200raster.h"
#include "api_util.cuh"

namespace {

constexpr int kVoxSerialBox = 16;   // columns one lane walks alone
constexpr int kVoxMaxSize = 1024;

// the reference's coordinate permutations per axis (:8-11): (y, x, z) of axis a are input coordinates kPerm[a][0..2]
__constant__ int kPerm[3][3] = {{2, 1, 0}, {0, 2, 1}, {0, 1, 2}};

struct VoxFace {
    float f0, f1, f2, y1d, x1d, z1d, y2d, x2d, z2d, det;
    int y_lo, y_hi, x_lo, x_hi;   // columns to test, inclusive (empty when lo > hi)
};

// Proof that every column the float test accepts lies in the box [floor(min), ceil(max)] of the face's projected
// vertices (DESIGN.md section 4 item 12).  With eps = 2^-24, a = y2d, b = x2d, c = y1d, d = x1d and U, V the largest
// |x - f1|, |y - f0| over the grid's columns:
//   eta   = 3 eps (|d a| + |b c|) / |det|                  relative error of the float det
//   delta = (4 eps max(|a| U + |b| V, |c| U + |d| V) + 2^-146) / (|det| (1 - eta))
//                                                          error of t1, t2 from the rounded numerators (+ underflow)
//   Delta = 2 eta + 3 delta + 8 eps                        every accepted column has barycentrics >= -Delta
// The triangle grown to barycentrics >= -Delta extends at most 2 Delta ext past its bounding box on each axis (ext =
// the box's larger side), so with (2 Delta + 4 eps) ext <= 1/4 (eta <= 1/4) an accepted integer column is within 1/2 of
// the box and lies in [floor(min), ceil(max)].  Evaluated in double with margins; NaN / inf fail the test.
__device__ bool vox_box_proven(const VoxFace& q, float ymin, float ymax, float xmin, float xmax, int vs) {
    const double eps = 5.9604644775390625e-8;
    const double a = q.y2d, b = q.x2d, c = q.y1d, d = q.x1d, det = fabs((double)q.det);
    const double U = fmax(fabs((double)q.f1), fabs((double)(vs - 1) - q.f1));
    const double V = fmax(fabs((double)q.f0), fabs((double)(vs - 1) - q.f0));
    const double eta = 3.0 * eps * (fabs(d * a) + fabs(b * c)) / det;
    if (!(eta <= 0.25)) return false;
    const double num = fmax(fabs(a) * U + fabs(b) * V, fabs(c) * U + fabs(d) * V);
    const double delta = (4.0 * eps * num + 1.2e-44) / (det * (1.0 - eta));
    const double Delta = 2.0 * eta + 3.0 * delta + 8.0 * eps;
    const double ext = fmax((double)ymax - ymin, (double)xmax - xmin);
    return (2.0 * Delta + 4.0 * eps) * ext <= 0.25;
}

// voxelize_sub1_kernel's per-face set-up (cuda/voxelization.py:49-57) for one axis, and the columns to test
__device__ void vox_setup(const float* __restrict__ face, int axis, int vs, VoxFace& q) {
    const int p0 = kPerm[axis][0], p1 = kPerm[axis][1], p2 = kPerm[axis][2];
    const float v0y = __ldg(face + p0), v0x = __ldg(face + p1);
    const float v1y = __ldg(face + 3 + p0), v1x = __ldg(face + 3 + p1);
    const float v2y = __ldg(face + 6 + p0), v2x = __ldg(face + 6 + p1);
    q.f0 = v0y;
    q.f1 = v0x;
    q.f2 = __ldg(face + p2);
    q.y1d = v1y - q.f0;
    q.x1d = v1x - q.f1;
    q.z1d = __ldg(face + 3 + p2) - q.f2;
    q.y2d = v2y - q.f0;
    q.x2d = v2x - q.f1;
    q.z2d = __ldg(face + 6 + p2) - q.f2;
    q.det = q.x1d * q.y2d - q.x2d * q.y1d;
    q.y_lo = 0, q.y_hi = -1, q.x_lo = 0, q.x_hi = -1;
    if (q.det == 0) return;                                               // :59
    const float ymin = fminf(fminf(v0y, v1y), v2y), ymax = fmaxf(fmaxf(v0y, v1y), v2y);
    const float xmin = fminf(fminf(v0x, v1x), v2x), xmax = fmaxf(fmaxf(v0x, v1x), v2x);
    if (vox_box_proven(q, ymin, ymax, xmin, xmax, vs)) {
        const float top = (float)(vs - 1);
        if (!(floorf(ymin) <= top && ceilf(ymax) >= 0.f && floorf(xmin) <= top && ceilf(xmax) >= 0.f)) return;
        q.y_lo = (int)fmaxf(floorf(ymin), 0.f), q.y_hi = (int)fminf(ceilf(ymax), top);
        q.x_lo = (int)fmaxf(floorf(xmin), 0.f), q.x_hi = (int)fminf(ceilf(xmax), top);
    } else {
        q.y_lo = 0, q.y_hi = vs - 1, q.x_lo = 0, q.x_hi = vs - 1;
    }
}

__device__ __forceinline__ size_t vox_stride(int coord, int vs) {
    return coord == 0 ? (size_t)vs * vs : coord == 1 ? (size_t)vs : 1;
}

// one (face, column) test and its four writes, cuda/voxelization.py:56-88
__device__ __forceinline__ void vox_column(const VoxFace& q, int y, int x, int vs, size_t sy, size_t sx, size_t sz,
                                           int* __restrict__ vox) {
    const float ypd = (float)y - q.f0;
    const float xpd = (float)x - q.f1;
    const float t1 = (q.y2d * xpd - q.x2d * ypd) / q.det;
    const float t2 = (-q.y1d * xpd + q.x1d * ypd) / q.det;
    if (t1 < 0) return;
    if (t2 < 0) return;
    if (1 < t1 + t2) return;
    const float zf = floorf(t1 * q.z1d + t2 * q.z2d + q.f2);
    if (!(zf >= 0.f && zf < (float)vs)) return;
    int* p = vox + (size_t)y * sy + (size_t)x * sx + (size_t)zf * sz;
    *p = 1;
    if (y > 0) *(p - sy) = 1;
    if (x > 0) *(p - sx) = 1;
    if (y > 0 && x > 0) *(p - sy - sx) = 1;
}

__global__ void __launch_bounds__(256)
k_voxelize_surface(const float* __restrict__ faces, int* __restrict__ voxels, int B, int nf, int vs) {
    const int lane = threadIdx.x & 31;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long total = (long)B * nf;
    const bool active = i < total;
    const size_t vs3 = (size_t)vs * vs * vs;
    if (active) {                                                          // voxelize_sub2_kernel, :150-160
        const float* face = faces + i * 9;
        int* vox = voxels + (size_t)(i / nf) * vs3;
        for (int k = 0; k < 3; k++) {
            const float c0 = __ldg(face + 3 * k), c1 = __ldg(face + 3 * k + 1), c2 = __ldg(face + 3 * k + 2);
            if (c0 >= 0.f && c0 < (float)vs && c1 >= 0.f && c1 < (float)vs && c2 >= 0.f && c2 < (float)vs)
                vox[((size_t)floorf(c0) * vs + (size_t)floorf(c1)) * vs + (size_t)floorf(c2)] = 1;
        }
    }
    for (int axis = 0; axis < 3; axis++) {
        // output strides of the axis's (y, x, z): input coordinate 0 is the slowest index
        const size_t sy = vox_stride(kPerm[axis][0], vs), sx = vox_stride(kPerm[axis][1], vs), sz = vox_stride(kPerm[axis][2], vs);
        VoxFace q;
        int n = 0, bw = 1;
        if (active) {
            vox_setup(faces + i * 9, axis, vs, q);
            if (q.y_lo <= q.y_hi && q.x_lo <= q.x_hi) {
                bw = q.x_hi - q.x_lo + 1;
                n = bw * (q.y_hi - q.y_lo + 1);
            }
        }
        if (n > 0 && n <= kVoxSerialBox) {
            int* vox = voxels + (size_t)(i / nf) * vs3;
            for (int j = 0; j < n; j++) vox_column(q, q.y_lo + j / bw, q.x_lo + j % bw, vs, sy, sx, sz, vox);
        }
        // large boxes and whole-grid fall-backs: the warp takes them one at a time (set-up recomputed by every lane)
        for (unsigned m = __ballot_sync(0xffffffffu, n > kVoxSerialBox); m != 0u; m &= m - 1u) {
            const long fi = i - lane + (__ffs(m) - 1);
            VoxFace r;
            vox_setup(faces + fi * 9, axis, vs, r);
            const int rw = r.x_hi - r.x_lo + 1, rn = rw * (r.y_hi - r.y_lo + 1);
            int* vox = voxels + (size_t)(fi / nf) * vs3;
            for (int j = lane; j < rn; j += 32) vox_column(r, r.y_lo + j / rw, r.x_lo + j % rw, vs, sy, sx, sz, vox);
        }
    }
}

// ---- fill.  Workspace: empty bits E then visible bits V, each [B, vs, vs, W] words, W = ceil(vs / 32); bit l of word w
// of row (b, y, x) is voxel z = 32 w + l; padding bits past vs are 0 in both.

// one warp per row: E = (voxel == 0); V = E on the grid's boundary (voxelize_sub3_kernel, :235-246)
__global__ void __launch_bounds__(256)
k_voxel_pack(const int* __restrict__ voxels, uint32_t* __restrict__ E, uint32_t* __restrict__ V, long rows, int vs, int W) {
    const long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int yx = (int)(row % ((long)vs * vs)), y = yx / vs, x = yx % vs;
    const bool edge_row = y == 0 || y == vs - 1 || x == 0 || x == vs - 1;
    const int* src = voxels + (size_t)row * vs;
    for (int w = 0; w < W; w++) {
        const int z = 32 * w + lane;
        const uint32_t e = __ballot_sync(0xffffffffu, z < vs && __ldg(src + z) == 0);
        const uint32_t ends = (w == 0 ? 1u : 0u) | (w == (vs - 1) / 32 ? 1u << ((vs - 1) & 31) : 0u);
        if (lane == 0) {
            E[(size_t)row * W + w] = e;
            V[(size_t)row * W + w] = edge_row ? e : (e & ends);
        }
    }
}

// One interior row (y, x): new visible bits are empty bits with a visible neighbour row, then each run of empty bits
// along z that holds a visible bit becomes visible (an add carries a seed to the top of its run; bit-reversed, to the
// bottom), across words.  Returns whether the row changed.
__device__ __forceinline__ bool vox_fill_row(const uint32_t* __restrict__ e_row, uint32_t* v_row, size_t sx, size_t sy, int W) {
    const uint32_t *xm = v_row - sx, *xp = v_row + sx, *ym = v_row - sy, *yp = v_row + sy;
    bool changed = false;
    uint32_t carry = 0;
    for (int w = 0; w < W; w++) {                                          // upward along z
        const uint32_t e = e_row[w], v = v_row[w];
        uint32_t s = v;
        if (e != v) {   // else every empty bit of the word is visible already
            s |= e & (xm[w] | xp[w] | ym[w] | yp[w] | carry);
            s |= ((e + s) ^ e) & e;
            if (s != v) {
                v_row[w] = s;
                changed = true;
            }
        }
        carry = s >> 31;
    }
    carry = 0;
    for (int w = W - 1; w >= 0; w--) {                                     // downward along z
        const uint32_t e = e_row[w], v = v_row[w];
        uint32_t s = v;
        if (e != v) {
            const uint32_t re = __brev(e);
            uint32_t r = __brev(v) | (re & carry);
            r |= ((re + r) ^ re) & re;
            s = __brev(r);
            if (s != v) {
                v_row[w] = s;
                changed = true;
            }
        }
        carry = s & 1u;
    }
    return changed;
}

// One CTA per image: sweeps over the interior rows (boundary rows are visible wherever empty from the start),
// alternating direction, until a sweep changes nothing.
__global__ void __launch_bounds__(1024)
k_voxel_propagate(const uint32_t* __restrict__ E, uint32_t* V, int vs, int W) {
    if (vs < 3) return;
    const size_t image = (size_t)blockIdx.x * vs * vs * W;
    const uint32_t* e_img = E + image;
    uint32_t* v_img = V + image;
    const int n = vs - 2, rows = n * n;
    const size_t sx = W, sy = (size_t)vs * W;
    for (int sweep = 0;; sweep++) {
        bool changed = false;
        for (int k = threadIdx.x; k < rows; k += blockDim.x) {
            const int r = (sweep & 1) ? rows - 1 - k : k;
            const size_t off = ((size_t)(1 + r / n) * vs + (1 + r % n)) * W;
            changed |= vox_fill_row(e_img + off, v_img + off, sx, sy, W);
        }
        if (!__syncthreads_or(changed)) break;
    }
}

// one warp per row: voxel = 1 - visible
__global__ void __launch_bounds__(256)
k_voxel_unpack(const uint32_t* __restrict__ V, int* __restrict__ voxels, long rows, int vs, int W) {
    const long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    int* dst = voxels + (size_t)row * vs;
    for (int w = 0; w < W; w++) {
        const int z = 32 * w + lane;
        if (z < vs) dst[z] = 1 - (int)((__ldg(V + (size_t)row * W + w) >> lane) & 1u);
    }
}

int check_voxel_size(const char* what, int B, int vs) {
    if (B < 1) return b200r_fail(B200R_EINVAL, "%s: batch_size %d < 1", what, B);
    if (vs < 1 || vs > kVoxMaxSize) return b200r_fail(B200R_EINVAL, "%s: voxel_size %d outside [1, %d]", what, vs, kVoxMaxSize);
    return 0;
}

}  // namespace

extern "C" size_t b200r_voxelize_workspace_bytes(int batch_size, int voxel_size) {
    if (batch_size < 1 || voxel_size < 1 || voxel_size > kVoxMaxSize) return 0;
    const size_t W = (size_t)(voxel_size + 31) / 32;
    return 2 * (size_t)batch_size * voxel_size * voxel_size * W * sizeof(uint32_t);
}

extern "C" int b200r_voxelize_surface(const float* faces, int32_t* voxels, int batch_size, int num_faces, int voxel_size,
                                      void* stream) {
    if (!faces || !voxels) return b200r_fail(B200R_EINVAL, "b200r_voxelize_surface: NULL pointer argument");
    if (int rc = check_voxel_size("b200r_voxelize_surface", batch_size, voxel_size)) return rc;
    if (num_faces < 1) return b200r_fail(B200R_EINVAL, "b200r_voxelize_surface: num_faces %d < 1", num_faces);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t vs3 = (size_t)voxel_size * voxel_size * voxel_size;
    cudaError_t e = cudaMemsetAsync(voxels, 0, (size_t)batch_size * vs3 * sizeof(int32_t), st);
    if (e != cudaSuccess) return b200r_cuda_fail(e, "b200r_voxelize_surface: memset");
    const long total = (long)batch_size * num_faces;
    {
        B200rProfScope prof(B200R_K_VOXEL_SURFACE, st);
        k_voxelize_surface<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(faces, voxels, batch_size, num_faces, voxel_size);
    }
    e = cudaGetLastError();
    if (e != cudaSuccess) return b200r_cuda_fail(e, "k_voxelize_surface");
    return 0;
}

extern "C" int b200r_voxelize_fill(int32_t* voxels, void* workspace, size_t workspace_bytes, int batch_size, int voxel_size,
                                   void* stream) {
    if (!voxels || !workspace) return b200r_fail(B200R_EINVAL, "b200r_voxelize_fill: NULL pointer argument");
    if (int rc = check_voxel_size("b200r_voxelize_fill", batch_size, voxel_size)) return rc;
    const size_t need = b200r_voxelize_workspace_bytes(batch_size, voxel_size);
    if (workspace_bytes < need)
        return b200r_fail(B200R_EWORKSPACE, "b200r_voxelize_fill: workspace %zu bytes < %zu", workspace_bytes, need);
    cudaStream_t st = (cudaStream_t)stream;
    const int vs = voxel_size, W = (vs + 31) / 32;
    const long rows = (long)batch_size * vs * vs;
    uint32_t* E = (uint32_t*)workspace;
    uint32_t* V = E + (size_t)rows * W;
    const unsigned row_blocks = (unsigned)((rows + 7) / 8);   // 8 warps of 256 threads, one row each
    {
        B200rProfScope prof(B200R_K_VOXEL_FILL, st);
        k_voxel_pack<<<row_blocks, 256, 0, st>>>(voxels, E, V, rows, vs, W);
    }
    {
        B200rProfScope prof(B200R_K_VOXEL_FILL, st);
        k_voxel_propagate<<<batch_size, 1024, 0, st>>>(E, V, vs, W);
    }
    {
        B200rProfScope prof(B200R_K_VOXEL_FILL, st);
        k_voxel_unpack<<<row_blocks, 256, 0, st>>>(V, voxels, rows, vs, W);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return b200r_cuda_fail(e, "k_voxel_fill");
    return 0;
}
