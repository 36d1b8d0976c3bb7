// gbuffer_api.cu -- normal and depth G-buffers of the surface lighting branches (Lighting(Gbuffer='normal' | 'depth')).
//
//   b200r_gbuffer_lighting_forward / _backward  <-  Lighting.execute, light_mode='surface', no normal map, no SSS
//        jrender/renderer/lighting/lighting.py:180-204   (textures = ones; clamp(ones * diffuse + ones * specular))
//        jrender/renderer/lighting/directional_lighting.py:136-144
//            'normal': specular *= 0, diffuse = normals * 0.5 + 0.5
//            'depth':  specular *= 0, diffuse = z / max(z) in all three channels, z the camera depth of the face
//                      centroid (transform.tranpos), the max over every (batch, face)
//   b200r_normal_mapped_gbuffer_forward / _backward  <-  the same branch with mesh.normal_textures, 'normal' only
//
// The light terms are the fused lighting kernels' own (lighting_math.cuh): the specular term s of the Cook-Torrance
// branch is evaluated because the reference multiplies it by 0 rather than dropping it, so a non-finite s turns the
// texel into NaN, and a -0.0 depth becomes +0.0.  The camera is the fused projection's (camera.cuh).
//
// Depth takes two launches forward: k_gb_depth_z writes each face's z and one partial max per block (at most
// GB_PARTIALS blocks, grid-stride); k_gb_fwd<DEPTH> has every block fold the partials to M in the same order, block 0
// stores M, and each thread writes one face's texels.  Backward likewise: k_gb_bwd_depth_fold folds the upstream
// gradient per face, G_f = sum_{t,c} g * mask, and writes one partial of sum_f G_f z_f per block; k_gb_bwd_depth_scatter
// folds those to dM = -sum / (M M), and scatters dz_f = G_f / M (+ dM where z_f == M: the reduce-max gradient as the
// mask x == max, every tied face getting all of it) through dz/dv = z_axis / 3.  No host synchronisation anywhere.
#include <math.h>

#include "../../include/b200raster.h"
#include "api_util.cuh"
#include "lighting_math.cuh"
#include "camera.cuh"

using namespace b200r;

namespace {

enum { GB_NORMAL = 0, GB_DEPTH = 1 };
constexpr int GB_THREADS = 256;
constexpr int GB_PARTIALS = 1024;   // blocks of the grid-stride depth passes, and so partials per reduction

struct GbArgs {
    const float* vertices;
    const int32_t* faces;
    const float* metallic;
    const float* roughness;
    const float* eye;       // specular eye, nullptr without the Cook-Torrance branch
    const float* cam_eye;   // camera eye (depth)
    int B, Bv, Bf, Be, Bc, nv, nf, T, Tm;
};

// The face's vertex indices and corners; its float64 normal (returns |c|) and centroid as the lighting kernels form them,
// except that a NaN |c| makes the whole normal NaN: each component is written to its own channel here, not dotted.
__device__ __forceinline__ double face_setup(const GbArgs& A, int b, int f, int idx[3], float v[9], float N[3], float pos[3]) {
    const int32_t* fi = A.faces + ((size_t)(A.Bf == 1 ? 0 : b) * A.nf + f) * 3;
    const float* vb = A.vertices + (size_t)(A.Bv == 1 ? 0 : b) * A.nv * 3;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        idx[k] = __ldg(fi + k);
        const float* q = vb + (size_t)idx[k] * 3;
        v[3 * k] = __ldg(q); v[3 * k + 1] = __ldg(q + 1); v[3 * k + 2] = __ldg(q + 2);
    }
    const double len = normal_f64(v, N);
    if (len != len) N[0] = N[1] = N[2] = __int_as_float(0x7fffffff);   // F.normalize's clamp_min keeps a NaN norm
#pragma unroll
    for (int k = 0; k < 3; k++) pos[k] = ((v[k] + v[3 + k]) + v[6 + k]) / 3.0f;   // torch.sum(face_vertices, dim=2) / 3.0
    return len;
}

// The specular term's inputs of face i: the branch flag (in Lf), the face's mean metallic / roughness and the eye.
__device__ __forceinline__ bool face_material(const GbArgs& A, const LightParams& L, long i, int b, LightParams& Lf, float& m,
                                              float& r, const float*& ey) {
    const bool spec = L.with_specular && A.metallic != nullptr && A.roughness != nullptr && A.eye != nullptr;
    Lf = L;
    Lf.with_specular = spec ? 1 : 0;
    m = spec ? mean_tm(A.metallic + (size_t)i * A.Tm, A.Tm) : 0.f;
    r = spec ? mean_tm(A.roughness + (size_t)i * A.Tm, A.Tm) : 1.f;
    ey = spec ? A.eye + (size_t)(A.Be == 1 ? 0 : b) * 3 : nullptr;
    return spec;
}

// camera z of a point, and the camera axes r (rows x, y, z) of batch element b
__device__ __forceinline__ float camera_depth(const GbArgs& A, const b200r_camera::CamParams& C, int b, const float pos[3],
                                              float r[3][3]) {
    const float* ep = A.cam_eye + (size_t)(A.Bc == 1 ? 0 : b) * 3;
    const float eye[3] = {__ldg(ep), __ldg(ep + 1), __ldg(ep + 2)};
    float cam[3];
    b200r_camera::camera_axes(C, eye, r);
    b200r_camera::to_camera(pos, eye, r, cam);
    return cam[2];
}

// numpy's max: NaN as soon as either is NaN
__device__ __forceinline__ float nan_max(float a, float b) { return a != a ? a : (b != b ? b : (b > a ? b : a)); }

// Every thread of the block gets the fold of its threads' x: max (MAX) or sum, in one fixed tree order.
template <bool MAX>
__device__ __forceinline__ float block_fold(float x) {
    __shared__ float sh[GB_THREADS];
    __syncthreads();   // sh may still be read by a previous fold
    sh[threadIdx.x] = x;
    __syncthreads();
    for (int s = GB_THREADS / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) sh[threadIdx.x] = MAX ? nan_max(sh[threadIdx.x], sh[threadIdx.x + s]) : sh[threadIdx.x] + sh[threadIdx.x + s];
        __syncthreads();
    }
    return sh[0];
}

// partials[0 .. n) folded the same way in every block (thread k takes k, k + 256, ... in order, then the tree)
template <bool MAX>
__device__ __forceinline__ float fold_partials(const float* __restrict__ partials, int n) {
    float x = MAX ? -INFINITY : 0.f;
    for (int k = threadIdx.x; k < n; k += GB_THREADS) x = MAX ? nan_max(x, partials[k]) : x + partials[k];
    return block_fold<MAX>(x);
}

__global__ void __launch_bounds__(GB_THREADS)
k_gb_depth_z(GbArgs A, b200r_camera::CamParams C, float* __restrict__ face_z, float* __restrict__ partials) {
    const long n = (long)A.B * A.nf;
    float m = -INFINITY;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const int b = (int)(i / A.nf), f = (int)(i % A.nf);
        int idx[3];
        float v[9], pos[3], r[3][3];
#pragma unroll
        for (int k = 0; k < 3; k++) {   // the centroid alone, as face_centroid forms it
            idx[k] = __ldg(A.faces + ((size_t)(A.Bf == 1 ? 0 : b) * A.nf + f) * 3 + k);
            const float* q = A.vertices + ((size_t)(A.Bv == 1 ? 0 : b) * A.nv + idx[k]) * 3;
            v[3 * k] = __ldg(q); v[3 * k + 1] = __ldg(q + 1); v[3 * k + 2] = __ldg(q + 2);
        }
#pragma unroll
        for (int k = 0; k < 3; k++) pos[k] = ((v[k] + v[3 + k]) + v[6 + k]) / 3.0f;
        const float z = camera_depth(A, C, b, pos, r);
        face_z[i] = z;
        m = nan_max(m, z);
    }
    m = block_fold<true>(m);
    if (threadIdx.x == 0) partials[blockIdx.x] = m;
}

// One thread per (batch, face): the face's value (N * 0.5 + 0.5, or z / M) plus specular * 0 over its T texels.
template <int MODE>
__global__ void __launch_bounds__(GB_THREADS)
k_gb_fwd(GbArgs A, LightParams L, const float* __restrict__ face_z, const float* __restrict__ partials, int nparts,
         float* __restrict__ depth_max, float* __restrict__ out) {
    float M = 0.f;
    if (MODE == GB_DEPTH) {
        M = fold_partials<true>(partials, nparts);
        if (blockIdx.x == 0 && threadIdx.x == 0) *depth_max = M;
    }
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)A.B * A.nf) return;
    const int b = (int)(i / A.nf), f = (int)(i % A.nf);
    int idx[3];
    float v[9], N[3], pos[3], d[3], s[3], m, r;
    const float* ey;
    LightParams Lf;
    face_setup(A, b, f, idx, v, N, pos);
    face_material(A, L, i, b, Lf, m, r, ey);
    face_light<float>(N, pos, Lf, ey, m, r, d, s);
    float val[3], S[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        val[c] = MODE == GB_NORMAL ? N[c] * 0.5f + 0.5f : face_z[i] / M;
        S[c] = (0.0f + s[c]) * 0.0f;   // specularLight (zeros + s) *= 0.0
    }
    float* o = out + (size_t)i * A.T * 3;
    for (int t = 0; t < A.T; t++)
#pragma unroll
        for (int c = 0; c < 3; c++) o[t * 3 + c] = clamp01(1.0f * val[c] + 1.0f * S[c]);   // ones * diffuse + ones * specular
}

// Backward of one face, both modes: the masked upstream gradient per channel, the material gradients (through
// specular * 0: zero, or NaN where a partial of s is not finite), and the vertex gradient of everything but the depth
// value (the normal's Jacobian, and specular * 0).  Returns G_f = sum_c Gs[c].
template <int MODE>
__device__ __forceinline__ float gb_bwd_face(const GbArgs& A, const LightParams& L, long i, float zval, const float* __restrict__ grad_out,
                                             float* __restrict__ grad_vertices, float* __restrict__ grad_metallic,
                                             float* __restrict__ grad_roughness) {
    const int b = (int)(i / A.nf), f = (int)(i % A.nf);
    int idx[3];
    float v[9], N[3], pos[3], d[3], s[3], m, r;
    const float* ey;
    LightParams Lf;
    const double len = face_setup(A, b, f, idx, v, N, pos);
    const bool spec = face_material(A, L, i, b, Lf, m, r, ey);
    face_light<float>(N, pos, Lf, ey, m, r, d, s);
    float val[3], S[3], Gs[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int c = 0; c < 3; c++) {
        val[c] = MODE == GB_NORMAL ? N[c] * 0.5f + 0.5f : zval;
        S[c] = (0.0f + s[c]) * 0.0f;
    }
    const float* go = grad_out + (size_t)i * A.T * 3;
    for (int t = 0; t < A.T; t++)
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const float x = 1.0f * val[c] + 1.0f * S[c];
            Gs[c] += (x >= 0.0f && x <= 1.0f) ? __ldg(go + t * 3 + c) : 0.f;   // torch.clamp passes the gradient on [0, 1]
        }
    if (grad_metallic != nullptr || grad_roughness != nullptr) {
        float gm = 0.f, gr = 0.f;
        if (spec) {
            Dual<2> dm[3], sm[3];
            face_light<float, Dual<2>>(N, pos, Lf, ey, dvar<2>(m, 0), dvar<2>(r, 1), dm, sm);
#pragma unroll
            for (int c = 0; c < 3; c++) {
                gm += (Gs[c] * 0.0f) * sm[c].d[0];
                gr += (Gs[c] * 0.0f) * sm[c].d[1];
            }
            gm = gm / (float)A.Tm;
            gr = gr / (float)A.Tm;
        }
        if (grad_metallic != nullptr)
            for (int t = 0; t < A.Tm; t++) grad_metallic[(size_t)i * A.Tm + t] = gm;
        if (grad_roughness != nullptr)
            for (int t = 0; t < A.Tm; t++) grad_roughness[(size_t)i * A.Tm + t] = gr;
    }
    if (grad_vertices != nullptr && (MODE == GB_NORMAL || spec)) {
        typedef Dual<9> D;
        D Nd[3];
        normal_duals(v, N, len, Nd);
        if (len != len)   // the mirror divides by the NaN norm: every partial is NaN (normal_f64 clamps it to 1e-12)
#pragma unroll
            for (int j = 0; j < 3; j++)
#pragma unroll
                for (int k = 0; k < 9; k++) Nd[j].d[k] = __int_as_float(0x7fffffff);
        float acc[9];
#pragma unroll
        for (int k = 0; k < 9; k++) acc[k] = 0.f;
        if (MODE == GB_NORMAL) {
#pragma unroll
            for (int k = 0; k < 9; k++)
#pragma unroll
                for (int c = 0; c < 3; c++) acc[k] += (Gs[c] * 0.5f) * Nd[c].d[k];
        }
        if (spec) {
            D pd[3], dd[3], sd[3];
#pragma unroll
            for (int k = 0; k < 3; k++) pd[k] = ((dvar<9>(v[k], k) + dvar<9>(v[3 + k], 3 + k)) + dvar<9>(v[6 + k], 6 + k)) / 3.0f;
            face_light<D>(Nd, pd, Lf, ey, m, r, dd, sd);
#pragma unroll
            for (int k = 0; k < 9; k++)
#pragma unroll
                for (int c = 0; c < 3; c++) acc[k] += (Gs[c] * 0.0f) * sd[c].d[k];
        }
        float* gv = grad_vertices + (size_t)(A.Bv == 1 ? 0 : b) * A.nv * 3;
#pragma unroll
        for (int k = 0; k < 9; k++)
            if (acc[k] != 0.f) atomicAdd(gv + (size_t)idx[k / 3] * 3 + (k % 3), acc[k]);
    }
    return (Gs[0] + Gs[1]) + Gs[2];
}

__global__ void __launch_bounds__(GB_THREADS)
k_gb_bwd_normal(GbArgs A, LightParams L, const float* __restrict__ grad_out, float* __restrict__ grad_vertices,
                float* __restrict__ grad_metallic, float* __restrict__ grad_roughness) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)A.B * A.nf) return;
    gb_bwd_face<GB_NORMAL>(A, L, i, 0.f, grad_out, grad_vertices, grad_metallic, grad_roughness);
}

// depth backward, pass 1 (grid-stride, <= GB_PARTIALS blocks): G_f per face, and one partial of sum_f G_f z_f per block
__global__ void __launch_bounds__(GB_THREADS)
k_gb_bwd_depth_fold(GbArgs A, LightParams L, const float* __restrict__ face_z, const float* __restrict__ depth_max,
                    const float* __restrict__ grad_out, float* __restrict__ face_G, float* __restrict__ partials,
                    float* __restrict__ grad_vertices, float* __restrict__ grad_metallic, float* __restrict__ grad_roughness) {
    const long n = (long)A.B * A.nf;
    const float M = __ldg(depth_max);
    float acc = 0.f;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const float z = face_z[i];
        const float G = gb_bwd_face<GB_DEPTH>(A, L, i, z / M, grad_out, grad_vertices, grad_metallic, grad_roughness);
        face_G[i] = G;
        acc += G * z;
    }
    acc = block_fold<false>(acc);
    if (threadIdx.x == 0) partials[blockIdx.x] = acc;
}

// depth backward, pass 2: dz_f = G_f / M (+ dM where z_f == M), scattered as dz_f z_axis / 3 to the face's vertices
__global__ void __launch_bounds__(GB_THREADS)
k_gb_bwd_depth_scatter(GbArgs A, b200r_camera::CamParams C, const float* __restrict__ face_z, const float* __restrict__ depth_max,
                       const float* __restrict__ face_G, const float* __restrict__ partials, int nparts,
                       float* __restrict__ grad_vertices) {
    const float M = __ldg(depth_max);
    const float dM = -fold_partials<false>(partials, nparts) / (M * M);
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)A.B * A.nf) return;
    const int b = (int)(i / A.nf), f = (int)(i % A.nf);
    const float z = face_z[i];
    float dz = face_G[i] / M;
    // The max's gradient is dM * (z == M), a product, as the mirror forms it: a NaN dM reaches every face.  When the
    // vertices, faces and camera are all shared over the batch, the depths are one [1, nf] set broadcast over B (the
    // reference's positions have the vertices' batch), so each face's tie counts once, at b = 0.
    const bool shared = A.Bv == 1 && A.Bf == 1 && A.Bc == 1;
    if (!shared || b == 0) dz = dz + dM * (z == M ? 1.0f : 0.0f);
    if (dz == 0.f) return;
    const float* ep = A.cam_eye + (size_t)(A.Bc == 1 ? 0 : b) * 3;
    const float eye[3] = {__ldg(ep), __ldg(ep + 1), __ldg(ep + 2)};
    float r[3][3];
    b200r_camera::camera_axes(C, eye, r);
    const int32_t* fi = A.faces + ((size_t)(A.Bf == 1 ? 0 : b) * A.nf + f) * 3;
    float* gv = grad_vertices + (size_t)(A.Bv == 1 ? 0 : b) * A.nv * 3;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float g = (dz * r[2][k]) / 3.0f;   // z = (pos - eye) . z_axis, pos = sum of the corners / 3
        if (g != 0.f)
#pragma unroll
            for (int j = 0; j < 3; j++) atomicAdd(gv + (size_t)__ldg(fi + j) * 3 + k, g);
    }
}

// ---- normal-mapped normal G-buffer: one normal per texel, N = normalize(n_t . TBN) ---------------------------------

struct NmArgs {
    GbArgs g;
    const float* normal_textures;
    const float* tbn;
    int Bn, Bt;
};

// one thread per (batch, face, texel)
__global__ void __launch_bounds__(GB_THREADS)
k_nm_gb_fwd(NmArgs A, LightParams L, float* __restrict__ out) {
    const GbArgs& G = A.g;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)G.B * G.nf * G.T) return;
    const long bf = i / G.T;
    const int t = (int)(i % G.T), b = (int)(bf / G.nf), f = (int)(bf % G.nf);
    float pos[3], nt[3], N[3], d[3], s[3];
    face_centroid(G.vertices, G.faces, b, f, G.Bv, G.Bf, G.nv, G.nf, pos);
    const float* np_ = A.normal_textures + (((size_t)(A.Bn == 1 ? 0 : b) * G.nf + f) * G.T + t) * 3;
#pragma unroll
    for (int k = 0; k < 3; k++) nt[k] = __ldg(np_ + k);
    texel_normal(nt, A.tbn + ((size_t)(A.Bt == 1 ? 0 : b) * G.nf + f) * 9, N);
    const bool spec = L.with_specular && G.metallic != nullptr && G.roughness != nullptr && G.eye != nullptr;
    LightParams Lf = L;
    Lf.with_specular = spec ? 1 : 0;
    const float m = spec ? __ldg(G.metallic + i) : 0.f;
    const float r = spec ? __ldg(G.roughness + i) : 1.f;
    face_light<float>(N, pos, Lf, spec ? G.eye + (size_t)(G.Be == 1 ? 0 : b) * 3 : nullptr, m, r, d, s);
#pragma unroll
    for (int c = 0; c < 3; c++) out[(size_t)i * 3 + c] = clamp01(1.0f * (N[c] * 0.5f + 0.5f) + 1.0f * ((0.0f + s[c]) * 0.0f));
}

// One thread per (normal-texture batch, face, texel); with a batch-1 normal texture the thread runs every batch element
// in turn and sums its texel's grad_normal_textures without atomics.  Dual<6> over the tangent-space normal and the
// centroid; the centroid reaches the result only through specular * 0, so its atomics fire only on a NaN.
__global__ void __launch_bounds__(GB_THREADS)
k_nm_gb_bwd(NmArgs A, LightParams L, const float* __restrict__ grad_out, float* __restrict__ grad_normal_textures,
            float* __restrict__ grad_vertices, float* __restrict__ grad_metallic, float* __restrict__ grad_roughness) {
    typedef Dual<6> D;
    const GbArgs& G = A.g;
    const long w = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= (long)A.Bn * G.nf * G.T) return;
    const long bnf = w / G.T;
    const int t = (int)(w % G.T), bn = (int)(bnf / G.nf), f = (int)(bnf % G.nf);
    const int b0 = A.Bn == 1 ? 0 : bn, b1 = A.Bn == 1 ? G.B : bn + 1;
    const bool spec = L.with_specular && G.metallic != nullptr && G.roughness != nullptr && G.eye != nullptr;
    LightParams Lf = L;
    Lf.with_specular = spec ? 1 : 0;
    float nt[3];
#pragma unroll
    for (int k = 0; k < 3; k++) nt[k] = __ldg(A.normal_textures + (size_t)w * 3 + k);
    float gn[3] = {0.f, 0.f, 0.f};
    for (int b = b0; b < b1; b++) {
        const size_t i = ((size_t)b * G.nf + f) * G.T + t;
        float pos[3], N[3], d[3], s[3], Gs[3];
        face_centroid(G.vertices, G.faces, b, f, G.Bv, G.Bf, G.nv, G.nf, pos);
        const float* tb = A.tbn + ((size_t)(A.Bt == 1 ? 0 : b) * G.nf + f) * 9;
        const float* ey = spec ? G.eye + (size_t)(G.Be == 1 ? 0 : b) * 3 : nullptr;
        texel_normal(nt, tb, N);
        const float m = spec ? __ldg(G.metallic + i) : 0.f;
        const float r = spec ? __ldg(G.roughness + i) : 1.f;
        face_light<float>(N, pos, Lf, ey, m, r, d, s);
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const float x = 1.0f * (N[c] * 0.5f + 0.5f) + 1.0f * ((0.0f + s[c]) * 0.0f);
            Gs[c] = (x >= 0.0f && x <= 1.0f) ? __ldg(grad_out + i * 3 + c) : 0.f;
        }
        if (grad_metallic != nullptr || grad_roughness != nullptr) {
            float gm = 0.f, gr = 0.f;
            if (spec) {
                Dual<2> dm[3], sm[3];
                face_light<float, Dual<2>>(N, pos, Lf, ey, dvar<2>(m, 0), dvar<2>(r, 1), dm, sm);
#pragma unroll
                for (int c = 0; c < 3; c++) {
                    gm += (Gs[c] * 0.0f) * sm[c].d[0];
                    gr += (Gs[c] * 0.0f) * sm[c].d[1];
                }
            }
            if (grad_metallic != nullptr) grad_metallic[i] = gm;
            if (grad_roughness != nullptr) grad_roughness[i] = gr;
        }
        if (grad_normal_textures == nullptr && (grad_vertices == nullptr || !spec)) continue;
        D ntd[3], Nd[3], pd[3], dd[3], sd[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            ntd[k] = dvar<6>(nt[k], k);
            pd[k] = dvar<6>(pos[k], 3 + k);
        }
        texel_normal(ntd, tb, Nd);
        float gk[6];
#pragma unroll
        for (int k = 0; k < 6; k++) {
            float acc = 0.f;
#pragma unroll
            for (int c = 0; c < 3; c++) acc += (Gs[c] * 0.5f) * Nd[c].d[k];
            gk[k] = acc;
        }
        if (spec) {
            face_light<D>(Nd, pd, Lf, ey, m, r, dd, sd);
#pragma unroll
            for (int k = 0; k < 6; k++)
#pragma unroll
                for (int c = 0; c < 3; c++) gk[k] += (Gs[c] * 0.0f) * sd[c].d[k];
        }
#pragma unroll
        for (int k = 0; k < 3; k++) gn[k] += gk[k];
        if (grad_vertices != nullptr) {
            const int32_t* fi = G.faces + ((size_t)(G.Bf == 1 ? 0 : b) * G.nf + f) * 3;
            float* gv = grad_vertices + (size_t)(G.Bv == 1 ? 0 : b) * G.nv * 3;
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const float g = gk[3 + k] / 3.0f;
                if (g != 0.f)
#pragma unroll
                    for (int j = 0; j < 3; j++) atomicAdd(gv + (size_t)__ldg(fi + j) * 3 + k, g);
            }
        }
    }
    if (grad_normal_textures != nullptr)
#pragma unroll
        for (int k = 0; k < 3; k++) grad_normal_textures[(size_t)w * 3 + k] = gn[k];
}

int check_gb(const char* fn, const GbArgs& A, int mode, const void* dir_c, const void* dir) {
    if (!A.vertices || !A.faces || !dir_c || !dir) return b200r_fail(B200R_EINVAL, "%s: NULL pointer argument", fn);
    if (mode != GB_NORMAL && mode != GB_DEPTH) return b200r_fail(B200R_EINVAL, "%s: mode %d is neither normal (0) nor depth (1)", fn, mode);
    if (A.B <= 0 || A.nv <= 0 || A.nf <= 0 || A.T <= 0 || A.Tm < 0) return b200r_fail(B200R_EINVAL, "%s: non-positive size", fn);
    if ((A.Bv != 1 && A.Bv != A.B) || (A.Bf != 1 && A.Bf != A.B) || (A.Be != 0 && A.Be != 1 && A.Be != A.B))
        return b200r_fail(B200R_EINVAL, "%s: vertices / faces / eye batch must be 1 or B", fn);
    if (A.eye != nullptr && (A.metallic == nullptr || A.roughness == nullptr || A.Tm == 0))
        return b200r_fail(B200R_EINVAL, "%s: the specular branch needs metallic, roughness and Tm > 0", fn);
    return 0;
}

int check_depth(const char* fn, const GbArgs& A, const void* workspace, size_t workspace_floats, const void* depth_max,
                const float* at, const float* up, int camera_mode) {
    if (!A.cam_eye || !workspace || !depth_max || !at || !up) return b200r_fail(B200R_EINVAL, "%s: depth needs the camera eye, "
                                                                                 "a workspace and depth_max", fn);
    if (A.Bc != 1 && A.Bc != A.B) return b200r_fail(B200R_EINVAL, "%s: camera eye batch must be 1 or B", fn);
    if (camera_mode < B200R_CAM_LOOK_AT || camera_mode > B200R_CAM_LOOK_LEFT) return b200r_fail(B200R_EINVAL, "%s: camera mode %d", fn, camera_mode);
    if (workspace_floats < (size_t)A.B * A.nf + GB_PARTIALS)
        return b200r_fail(B200R_EWORKSPACE, "%s: workspace of %zu floats, needs %zu", fn, workspace_floats, (size_t)A.B * A.nf + GB_PARTIALS);
    return 0;
}

GbArgs gb_args(const float* vertices, const int32_t* faces, const float* metallic, const float* roughness, const float* eye,
               const float* cam_eye, int B, int vb, int fb, int eb, int cb, int nv, int nf, int T, int Tm) {
    GbArgs A;
    A.vertices = vertices; A.faces = faces; A.metallic = metallic; A.roughness = roughness;
    A.eye = eb ? eye : nullptr; A.cam_eye = cam_eye;
    A.B = B; A.Bv = vb; A.Bf = fb; A.Be = eb ? eb : 1; A.Bc = cb; A.nv = nv; A.nf = nf; A.T = T; A.Tm = Tm;
    return A;
}

b200r_camera::CamParams cam_params(const float* at, const float* up, int camera_mode) {
    b200r_camera::CamParams C = {};
    for (int k = 0; k < 3; k++) { C.at_or_dir[k] = at[k]; C.up[k] = up[k]; }
    C.mode = camera_mode;
    return C;
}

const float zero3[3] = {0.f, 0.f, 0.f};

unsigned depth_grid(long n) { return (unsigned)(n / GB_THREADS + 1 < GB_PARTIALS ? n / GB_THREADS + 1 : GB_PARTIALS); }

}  // namespace

extern "C" {

size_t b200r_gbuffer_workspace_floats(int batch_size, int num_faces) {
    if (batch_size <= 0 || num_faces <= 0) return 0;
    return (size_t)batch_size * num_faces + GB_PARTIALS;
}

int b200r_gbuffer_lighting_forward(const float* vertices, const int32_t* faces, const float* metallic, const float* roughness,
                                   const float* eye, const float* camera_eye, float* out_textures, float* workspace,
                                   size_t workspace_floats, float* depth_max, int mode, int B, int vertices_batch,
                                   int faces_batch, int eye_batch, int camera_eye_batch, int nv, int nf, int T, int Tm,
                                   float directional_intensity, const float* directional_color, const float* direction,
                                   int with_specular, const float* camera_at_or_direction, const float* camera_up,
                                   int camera_mode, void* stream) {
    const char* fn = "b200r_gbuffer_lighting_forward";
    const GbArgs A = gb_args(vertices, faces, metallic, roughness, eye, camera_eye, B, vertices_batch, faces_batch, eye_batch,
                             camera_eye_batch, nv, nf, T, Tm);
    if (int rc = check_gb(fn, A, mode, directional_color, direction)) return rc;
    if (!out_textures) return b200r_fail(B200R_EINVAL, "%s: NULL pointer argument", fn);
    cudaStream_t st = (cudaStream_t)stream;
    const LightParams L = make(0.f, zero3, directional_intensity, directional_color, direction, with_specular);
    const long n = (long)B * nf;
    const unsigned grid = (unsigned)((n + GB_THREADS - 1) / GB_THREADS);
    if (mode == GB_NORMAL)
        return b200r_launch("k_gb_fwd<normal>", B200R_K_LIGHTING, k_gb_fwd<GB_NORMAL>, grid, GB_THREADS, 0, st, A, L,
                            (const float*)nullptr, (const float*)nullptr, 0, (float*)nullptr, out_textures);
    if (int rc = check_depth(fn, A, workspace, workspace_floats, depth_max, camera_at_or_direction, camera_up, camera_mode)) return rc;
    const b200r_camera::CamParams C = cam_params(camera_at_or_direction, camera_up, camera_mode);
    const unsigned parts = depth_grid(n);
    float* face_z = workspace;
    float* partials = workspace + n;
    if (int rc = b200r_launch("k_gb_depth_z", B200R_K_LIGHTING, k_gb_depth_z, parts, GB_THREADS, 0, st, A, C, face_z, partials))
        return rc;
    return b200r_launch("k_gb_fwd<depth>", B200R_K_LIGHTING, k_gb_fwd<GB_DEPTH>, grid, GB_THREADS, 0, st, A, L,
                        (const float*)face_z, (const float*)partials, (int)parts, depth_max, out_textures);
}

int b200r_gbuffer_lighting_backward(const float* vertices, const int32_t* faces, const float* metallic, const float* roughness,
                                    const float* eye, const float* camera_eye, const float* grad_out, const float* face_depth,
                                    const float* depth_max, float* workspace, size_t workspace_floats, float* grad_vertices,
                                    float* grad_metallic, float* grad_roughness, int mode, int B, int vertices_batch,
                                    int faces_batch, int eye_batch, int camera_eye_batch, int nv, int nf, int T, int Tm,
                                    float directional_intensity, const float* directional_color, const float* direction,
                                    int with_specular, const float* camera_at_or_direction, const float* camera_up,
                                    int camera_mode, void* stream) {
    const char* fn = "b200r_gbuffer_lighting_backward";
    const GbArgs A = gb_args(vertices, faces, metallic, roughness, eye, camera_eye, B, vertices_batch, faces_batch, eye_batch,
                             camera_eye_batch, nv, nf, T, Tm);
    if (int rc = check_gb(fn, A, mode, directional_color, direction)) return rc;
    if (!grad_out) return b200r_fail(B200R_EINVAL, "%s: NULL pointer argument", fn);
    if ((grad_metallic || grad_roughness) && (!metallic || !roughness || Tm == 0))
        return b200r_fail(B200R_EINVAL, "%s: material gradients need metallic, roughness and Tm > 0", fn);
    cudaStream_t st = (cudaStream_t)stream;
    if (grad_vertices != nullptr) {
        if (int rc = b200r_zero(grad_vertices, sizeof(float) * 3 * (size_t)vertices_batch * nv, st, "memset grad_vertices")) return rc;
    }
    const LightParams L = make(0.f, zero3, directional_intensity, directional_color, direction, with_specular);
    const long n = (long)B * nf;
    const unsigned grid = (unsigned)((n + GB_THREADS - 1) / GB_THREADS);
    if (mode == GB_NORMAL)
        return b200r_launch("k_gb_bwd_normal", B200R_K_LIGHTING, k_gb_bwd_normal, grid, GB_THREADS, 0, st, A, L, grad_out,
                            grad_vertices, grad_metallic, grad_roughness);
    if (int rc = check_depth(fn, A, workspace, workspace_floats, depth_max, camera_at_or_direction, camera_up, camera_mode)) return rc;
    if (!face_depth) return b200r_fail(B200R_EINVAL, "%s: depth needs the forward's face depths", fn);
    const b200r_camera::CamParams C = cam_params(camera_at_or_direction, camera_up, camera_mode);
    const unsigned parts = depth_grid(n);
    float* face_G = workspace;
    float* partials = workspace + n;
    if (int rc = b200r_launch("k_gb_bwd_depth_fold", B200R_K_LIGHTING, k_gb_bwd_depth_fold, parts, GB_THREADS, 0, st, A, L,
                              face_depth, depth_max, grad_out, face_G, partials, grad_vertices, grad_metallic, grad_roughness))
        return rc;
    if (grad_vertices == nullptr) return 0;
    return b200r_launch("k_gb_bwd_depth_scatter", B200R_K_LIGHTING, k_gb_bwd_depth_scatter, grid, GB_THREADS, 0, st, A, C,
                        face_depth, depth_max, (const float*)face_G, (const float*)partials, (int)parts, grad_vertices);
}

int b200r_normal_mapped_gbuffer_forward(const float* vertices, const int32_t* faces, const float* normal_textures,
                                        const float* tbn, const float* metallic, const float* roughness, const float* eye,
                                        float* out_textures, int B, int vertices_batch, int faces_batch, int eye_batch,
                                        int normal_batch, int tbn_batch, int nv, int nf, int T, float directional_intensity,
                                        const float* directional_color, const float* direction, int with_specular,
                                        void* stream) {
    const char* fn = "b200r_normal_mapped_gbuffer_forward";
    NmArgs A;
    A.g = gb_args(vertices, faces, metallic, roughness, eye, nullptr, B, vertices_batch, faces_batch, eye_batch, 1, nv, nf, T,
                  eye_batch ? 1 : 0);
    A.normal_textures = normal_textures; A.tbn = tbn; A.Bn = normal_batch; A.Bt = tbn_batch;
    if (int rc = check_gb(fn, A.g, GB_NORMAL, directional_color, direction)) return rc;
    if (!normal_textures || !tbn || !out_textures) return b200r_fail(B200R_EINVAL, "%s: NULL pointer argument", fn);
    if ((normal_batch != 1 && normal_batch != B) || (tbn_batch != 1 && tbn_batch != B))
        return b200r_fail(B200R_EINVAL, "%s: normal_textures / tbn batch must be 1 or B", fn);
    const LightParams L = make(0.f, zero3, directional_intensity, directional_color, direction, with_specular);
    const long n = (long)B * nf * T;
    return b200r_launch("k_nm_gb_fwd", B200R_K_LIGHTING, k_nm_gb_fwd, (unsigned)((n + GB_THREADS - 1) / GB_THREADS), GB_THREADS, 0,
                        (cudaStream_t)stream, A, L, out_textures);
}

int b200r_normal_mapped_gbuffer_backward(const float* vertices, const int32_t* faces, const float* normal_textures,
                                         const float* tbn, const float* metallic, const float* roughness, const float* eye,
                                         const float* grad_out, float* grad_normal_textures, float* grad_vertices,
                                         float* grad_metallic, float* grad_roughness, int B, int vertices_batch,
                                         int faces_batch, int eye_batch, int normal_batch, int tbn_batch, int nv, int nf,
                                         int T, float directional_intensity, const float* directional_color,
                                         const float* direction, int with_specular, void* stream) {
    const char* fn = "b200r_normal_mapped_gbuffer_backward";
    NmArgs A;
    A.g = gb_args(vertices, faces, metallic, roughness, eye, nullptr, B, vertices_batch, faces_batch, eye_batch, 1, nv, nf, T,
                  eye_batch ? 1 : 0);
    A.normal_textures = normal_textures; A.tbn = tbn; A.Bn = normal_batch; A.Bt = tbn_batch;
    if (int rc = check_gb(fn, A.g, GB_NORMAL, directional_color, direction)) return rc;
    if (!normal_textures || !tbn || !grad_out) return b200r_fail(B200R_EINVAL, "%s: NULL pointer argument", fn);
    if ((normal_batch != 1 && normal_batch != B) || (tbn_batch != 1 && tbn_batch != B))
        return b200r_fail(B200R_EINVAL, "%s: normal_textures / tbn batch must be 1 or B", fn);
    if ((grad_metallic || grad_roughness) && (!metallic || !roughness))
        return b200r_fail(B200R_EINVAL, "%s: material gradients need metallic and roughness", fn);
    cudaStream_t st = (cudaStream_t)stream;
    if (grad_vertices != nullptr) {
        if (int rc = b200r_zero(grad_vertices, sizeof(float) * 3 * (size_t)vertices_batch * nv, st, "memset grad_vertices")) return rc;
    }
    const LightParams L = make(0.f, zero3, directional_intensity, directional_color, direction, with_specular);
    const long n = (long)normal_batch * nf * T;
    return b200r_launch("k_nm_gb_bwd", B200R_K_LIGHTING, k_nm_gb_bwd, (unsigned)((n + GB_THREADS - 1) / GB_THREADS), GB_THREADS, 0, st,
                        A, L, grad_out, grad_normal_textures, grad_vertices, grad_metallic, grad_roughness);
}

}  // extern "C"
