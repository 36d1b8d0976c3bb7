// preraster_api.cu -- fused pre-raster geometry stage (SURVEY.md section 8f rank 1).
//
// One launch replaces the tensor-op chain the reference runs between `Mesh.vertices` (world
// space) and the rasterizer's `face_vertices` input:
//   look_at   jrender/renderer/transform/look_at.py:24-38   (axes, v - eye, v @ r^T)
//   look      jrender/renderer/transform/look.py:30-53      (same with a fixed direction)
//   perspective / orthogonal   transform/perspective.py:11-16, transform/orthogonal.py:12-15
//   face_vertices gather       structures/utils/faces_vertices.py:14-19
// and, in the backward, the scatter-add of grad_face_vertices to grad_vertices that the
// reference's autograd derives from the gather, plus the Jacobians of projection and rotation.
//
// Arithmetic follows the reference expressions in source order (separately rounded fp32 ops,
// -fmad=false): v - eye; sum_k v_k r[i][k] in k order; x / z / width.  Parity against the
// reference's own Python (run through a numpy-backed jittor stub, tests/golden/ref_host_*.npz)
// is a float comparison: jittor's reduction order inside matmul / normalize is not specified.
#include "../../include/b200raster.h"
#include "api_util.cuh"

namespace {

struct CamParams {
    float at_or_dir[3];  // look_at: `at`; look: `direction`
    float up[3];
    float width;         // perspective: tan(angle); orthogonal: scale
    int mode;            // B200R_CAM_LOOK_AT / LOOK_RIGHT / LOOK_LEFT
    int projection;      // B200R_PROJ_PERSPECTIVE / ORTHOGONAL
    int B, nv, nf, vertices_batch, faces_batch, eye_batch;
};

__device__ __forceinline__ void normalize3(float* v, float eps) {
    // jt.normalize(x, eps): x / max(||x||_2, eps)
    const float n = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    const float d = fmaxf(n, eps);
    v[0] = v[0] / d; v[1] = v[1] / d; v[2] = v[2] / d;
}

__device__ __forceinline__ void cross3(float* o, const float* a, const float* b) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

// rows of r = camera x, y, z axes (look_at.py:24-30, look.py:30-47)
__device__ __forceinline__ void camera_axes(const CamParams& C, const float* eye, float r[3][3]) {
    float z[3], up[3] = {C.up[0], C.up[1], C.up[2]};
    if (C.mode == B200R_CAM_LOOK_AT) {
        z[0] = C.at_or_dir[0] - eye[0]; z[1] = C.at_or_dir[1] - eye[1]; z[2] = C.at_or_dir[2] - eye[2];
        normalize3(z, 1e-5f);
    } else {
        z[0] = C.at_or_dir[0]; z[1] = C.at_or_dir[1]; z[2] = C.at_or_dir[2];
        normalize3(z, 1e-5f);    // look.py:23
        normalize3(up, 1e-5f);   // look.py:24
    }
    float x[3], y[3];
    if (C.mode == B200R_CAM_LOOK_LEFT) {
        cross3(x, z, up); normalize3(x, 1e-5f);  // look.py:42-43
        cross3(y, x, z);  normalize3(y, 1e-5f);
    } else {
        cross3(x, up, z); normalize3(x, 1e-5f);  // look_at.py:28-29, look.py:39-40
        cross3(y, z, x);  normalize3(y, 1e-5f);
    }
#pragma unroll
    for (int k = 0; k < 3; k++) { r[0][k] = x[k]; r[1][k] = y[k]; r[2][k] = z[k]; }
}

__device__ __forceinline__ void to_camera(const float* v, const float* eye, const float r[3][3], float* cam) {
    const float d0 = v[0] - eye[0], d1 = v[1] - eye[1], d2 = v[2] - eye[2];  // look_at.py:36
#pragma unroll
    for (int i = 0; i < 3; i++) cam[i] = d0 * r[i][0] + d1 * r[i][1] + d2 * r[i][2];  // matmul(v, r^T) :38
}

// thread = one (batch, face, corner): 12-byte stores are contiguous across the warp
__global__ void __launch_bounds__(256)
k_project_faces_fwd(const CamParams C, const float* __restrict__ vertices, const int32_t* __restrict__ faces,
                    const float* __restrict__ eyes, float* __restrict__ face_vertices) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long per_b = (long long)C.nf * 3;
    if (i >= per_b * C.B) return;
    const int b = (int)(i / per_b);
    const long long fc = i - (long long)b * per_b;
    const int idx = __ldg(faces + (C.faces_batch > 1 ? (long long)b * per_b : 0) + fc);
    float* out = face_vertices + i * 3;
    if ((unsigned)idx >= (unsigned)C.nv) {  // the reference would read out of bounds; poison the face instead
        out[0] = out[1] = out[2] = __int_as_float(0x7fc00000);
        return;
    }
    const float* v = vertices + ((C.vertices_batch > 1 ? (long long)b * C.nv : 0) + idx) * 3;
    const float* ep = eyes + (C.eye_batch > 1 ? b * 3 : 0);
    const float eye[3] = {__ldg(ep), __ldg(ep + 1), __ldg(ep + 2)};
    const float vv[3] = {__ldg(v), __ldg(v + 1), __ldg(v + 2)};
    float r[3][3], cam[3];
    camera_axes(C, eye, r);
    to_camera(vv, eye, r, cam);
    if (C.projection == B200R_PROJ_PERSPECTIVE) {
        out[0] = cam[0] / cam[2] / C.width;  // perspective.py:14-15
        out[1] = cam[1] / cam[2] / C.width;
    } else {
        out[0] = cam[0] * C.width;           // orthogonal.py:13-14
        out[1] = cam[1] * C.width;
    }
    out[2] = cam[2];
}

// Backward: d(loss)/d(world vertex) accumulated over every (face, corner) that references the
// vertex (and over the batch when the vertices are shared).  grad_vertices is zeroed by the caller
// of the kernel (b200r_zero in the entry point).
__global__ void __launch_bounds__(256)
k_project_faces_bwd(const CamParams C, const float* __restrict__ vertices, const int32_t* __restrict__ faces,
                    const float* __restrict__ eyes, const float* __restrict__ grad_face_vertices,
                    float* __restrict__ grad_vertices) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long per_b = (long long)C.nf * 3;
    if (i >= per_b * C.B) return;
    const int b = (int)(i / per_b);
    const long long fc = i - (long long)b * per_b;
    const int idx = __ldg(faces + (C.faces_batch > 1 ? (long long)b * per_b : 0) + fc);
    if ((unsigned)idx >= (unsigned)C.nv) return;
    const float* g = grad_face_vertices + i * 3;
    const float gx = __ldg(g), gy = __ldg(g + 1), gz = __ldg(g + 2);
    if (gx == 0.f && gy == 0.f && gz == 0.f) return;  // faces the rasterizer never touched
    const long long vrow = (C.vertices_batch > 1 ? (long long)b * C.nv : 0) + idx;
    const float* v = vertices + vrow * 3;
    const float* ep = eyes + (C.eye_batch > 1 ? b * 3 : 0);
    const float eye[3] = {__ldg(ep), __ldg(ep + 1), __ldg(ep + 2)};
    const float vv[3] = {__ldg(v), __ldg(v + 1), __ldg(v + 2)};
    float r[3][3], cam[3], dc[3];
    camera_axes(C, eye, r);
    to_camera(vv, eye, r, cam);
    if (C.projection == B200R_PROJ_PERSPECTIVE) {
        // x = X / Z / w, y = Y / Z / w, z = Z
        const float zw = cam[2] * C.width;
        dc[0] = gx / zw;
        dc[1] = gy / zw;
        dc[2] = gz - (gx * cam[0] + gy * cam[1]) / (cam[2] * zw);
    } else {
        dc[0] = gx * C.width;
        dc[1] = gy * C.width;
        dc[2] = gz;
    }
    float* o = grad_vertices + vrow * 3;
#pragma unroll
    for (int k = 0; k < 3; k++) atomicAdd(o + k, dc[0] * r[0][k] + dc[1] * r[1][k] + dc[2] * r[2][k]);
}

int check_args(const char* who, const void* vertices, const void* faces, const void* eye, const void* io,
               const float* at_or_dir, const float* up, int B, int nv, int nf, int vb, int fb, int eb, int mode, int proj) {
    if (!vertices || !faces || !eye || !io || !at_or_dir || !up) return b200r_fail(B200R_EINVAL, "%s: NULL pointer", who);
    if (B <= 0 || nv <= 0 || nf <= 0) return b200r_fail(B200R_EINVAL, "%s: B=%d nv=%d nf=%d must be positive", who, B, nv, nf);
    if ((vb != 1 && vb != B) || (fb != 1 && fb != B) || (eb != 1 && eb != B))
        return b200r_fail(B200R_EINVAL, "%s: vertices/faces/eye batch (%d, %d, %d) must be 1 or B=%d", who, vb, fb, eb, B);
    if (mode < B200R_CAM_LOOK_AT || mode > B200R_CAM_LOOK_LEFT) return b200r_fail(B200R_EINVAL, "%s: camera mode %d", who, mode);
    if (proj != B200R_PROJ_PERSPECTIVE && proj != B200R_PROJ_ORTHOGONAL) return b200r_fail(B200R_EINVAL, "%s: projection %d", who, proj);
    if ((long long)B * nf * 3 > 0x7fffffffLL * 64) return b200r_fail(B200R_EINVAL, "%s: too many corners", who);
    return 0;
}

CamParams make_params(const float* at_or_dir, const float* up, float width, int mode, int proj, int B, int nv, int nf,
                      int vb, int fb, int eb) {
    CamParams C;
    for (int k = 0; k < 3; k++) { C.at_or_dir[k] = at_or_dir[k]; C.up[k] = up[k]; }
    C.width = width; C.mode = mode; C.projection = proj;
    C.B = B; C.nv = nv; C.nf = nf; C.vertices_batch = vb; C.faces_batch = fb; C.eye_batch = eb;
    return C;
}

}  // namespace

extern "C" {

B200R_API int b200r_project_faces_forward(const float* vertices, const int32_t* faces, const float* eye,
                                          float* face_vertices,
                                          const float* at_or_direction, const float* up, float width_or_scale,
                                          int camera_mode, int projection, int batch_size, int num_vertices,
                                          int num_faces, int vertices_batch, int faces_batch, int eye_batch, void* stream) {
    int rc = check_args("b200r_project_faces_forward", vertices, faces, eye, face_vertices, at_or_direction, up, batch_size,
                        num_vertices, num_faces, vertices_batch, faces_batch, eye_batch, camera_mode, projection);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const CamParams C = make_params(at_or_direction, up, width_or_scale, camera_mode, projection, batch_size, num_vertices,
                                    num_faces, vertices_batch, faces_batch, eye_batch);
    const long long n = (long long)batch_size * num_faces * 3;
    return b200r_launch("k_project_faces_fwd", B200R_K_PROJECT_FWD, k_project_faces_fwd, (unsigned)((n + 255) / 256), 256, 0, st, C,
                        vertices, faces, eye, face_vertices);
}

B200R_API int b200r_project_faces_backward(const float* vertices, const int32_t* faces, const float* eye,
                                           const float* grad_face_vertices, float* grad_vertices,
                                           const float* at_or_direction, const float* up, float width_or_scale,
                                           int camera_mode, int projection, int batch_size, int num_vertices,
                                           int num_faces, int vertices_batch, int faces_batch, int eye_batch, void* stream) {
    int rc = check_args("b200r_project_faces_backward", vertices, faces, eye, grad_vertices, at_or_direction, up, batch_size,
                        num_vertices, num_faces, vertices_batch, faces_batch, eye_batch, camera_mode, projection);
    if (rc) return rc;
    if (!grad_face_vertices) return b200r_fail(B200R_EINVAL, "b200r_project_faces_backward: grad_face_vertices is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    const CamParams C = make_params(at_or_direction, up, width_or_scale, camera_mode, projection, batch_size, num_vertices,
                                    num_faces, vertices_batch, faces_batch, eye_batch);
    const long long n = (long long)batch_size * num_faces * 3;
    if (int rc = b200r_zero(grad_vertices, sizeof(float) * 3 * (size_t)vertices_batch * num_vertices, st,
                            "b200r_project_faces_backward: memset"))
        return rc;
    return b200r_launch("k_project_faces_bwd", B200R_K_PROJECT_BWD, k_project_faces_bwd, (unsigned)((n + 255) / 256), 256, 0, st, C,
                        vertices, faces, eye, grad_face_vertices, grad_vertices);
}

}  // extern "C"
