// camera.cuh -- the look_at / look camera of the fused projection (preraster_api.cu), shared with the depth G-buffer
// (gbuffer_api.cu) so that both form the same float32 camera axes and camera-space coordinates.
#pragma once
#include "../../include/b200raster.h"

namespace b200r_camera {

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

}  // namespace b200r_camera
