// lighting_api.cu -- fused surface-mode lighting of the pre-raster stage (SURVEY.md section 8f rank 1).
//
//   b200r_surface_lighting_forward / _backward  <-  Lighting.execute, light_mode='surface', no normal map, no SSS
//        jrender/renderer/lighting/lighting.py:186-204         (zeros -> ambient -> directional -> clamp(tex * diffuse + specular))
//        jrender/renderer/lighting/ambient_lighting.py:4-9
//        jrender/renderer/lighting/directional_lighting.py:54-135 (diffuse branch and the Cook-Torrance branch the
//                                                                reference takes by default: Mesh.with_specular = True)
//        jrender/structures/mesh.py:213-229                    (surface normals: float64 cross product, normalised)
//
// One thread per (batch, face): gathers the face's three world-space vertices, forms the normal and the centroid,
// evaluates the two light terms (6 floats) and streams the face's T texels through  clamp(tex * diffuse + specular, 0, 1).
// The reference runs this as ~30 tensor ops over [B, nf, 3] intermediates (and as many again backward); in the
// launch-bound demo loops that was ~230 launches per iteration.  Backward: the same expression re-evaluated in
// forward-mode automatic differentiation over the 9 vertex coordinates (dual.cuh) -- the exact gradient of the
// expression the forward evaluates, including the path through the normal, with 9 atomics per face into grad_vertices --
// and, only when material gradients are requested, once more over the face's mean metallic and roughness (Dual<2>,
// geometry constant), which keeps the vertex-only evaluation's code and registers as they were.
#include "../../include/b200raster.h"
#include "api_util.cuh"
#include "dual.cuh"

using namespace b200r;

namespace {

struct LightParams {
    float amb_i, amb_c[3];
    float dir_i, dir_c[3], dir[3];   // dir: normalised on the host exactly like F.normalize(light_direction, eps=1e-12)
    int with_specular;               // Cook-Torrance branch (needs eye + metallic + roughness)
};

// R: the result type of an expression mixing geometry of type S with material scalars of type M -- float when both are
// float, Dual<N> when either is (face_light never mixes two Dual types).  lift<R>(x) widens a float or an R to an R.
template <class S, class M> struct Promote { typedef S type; };
template <int N> struct Promote<float, Dual<N>> { typedef Dual<N> type; };
template <class R> struct Lift { __device__ __forceinline__ static R of(float x) { return x; } };
template <int N> struct Lift<Dual<N>> {
    __device__ __forceinline__ static Dual<N> of(float x) { return dconst<N>(x); }
    __device__ __forceinline__ static Dual<N> of(const Dual<N>& x) { return x; }
};
template <class R, class X> __device__ __forceinline__ R lift(const X& x) { return Lift<R>::of(x); }

template <class S>
__device__ __forceinline__ S dot3(const S a[3], const S b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }   // torch.sum(a * b, dim): x, y, z order
template <class S>
__device__ __forceinline__ S dot3f(const S a[3], const float b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// x / max(||x||, eps)   (F.normalize / jt.normalize)
template <class S>
__device__ __forceinline__ void normalize3(S x[3], float eps) {
    const S n = dmax(dsqrt(dot3(x, x)), eps);
#pragma unroll
    for (int k = 0; k < 3; k++) x[k] = x[k] / n;
}

// diffuse[3], specular[3] of one face from its normal N and centroid pos (directional_lighting.py:63-135, 3-D normals).
// S is the geometry's type and M the material scalars' (metallic, roughness): <float, float> evaluates, <Dual<9>, float>
// differentiates w.r.t. the vertices, <float, Dual<2>> w.r.t. metallic and roughness with the geometry held constant.
template <class S, class M, class R = typename Promote<S, M>::type>
__device__ __forceinline__ void face_light(const S N[3], const S pos[3], const LightParams& L, const float* eye, M metallic,
                                           M roughness, R diffuse[3], R specular[3]) {
    const S cosine = dmax(dot3f(N, L.dir), 0.f);   // relu(sum(normals * light_direction)) :66
#pragma unroll
    for (int c = 0; c < 3; c++) diffuse[c] = lift<R>(0.f + L.amb_i * L.amb_c[c]);   // zeros + ambient (ambient_lighting.py:8)
    if (L.with_specular && eye != nullptr) {
        S V[3] = {eye[0] - pos[0], eye[1] - pos[1], eye[2] - pos[2]};
        normalize3(V, 1e-12f);
        S H[3] = {V[0] + L.dir[0], V[1] + L.dir[1], V[2] + L.dir[2]};
        normalize3(H, 1e-12f);
        const M a = roughness * roughness, a2 = a * a;
        const S NdotH = dmax(dot3(N, H), 0.f);
        R den = (NdotH * NdotH) * (a2 - 1.0f) + 1.0f;          // GGX :17
        den = (den * 3.1415f) * den;                            // 3.1415 * denom * denom :18
        const R NDF = lift<R>(a2) / den;
        const M r1 = roughness + 1.0f, k = (r1 * r1) / 8.0f;
        const S NdotV = dmax(dot3(N, V), 0.f), NdotL = dmax(dot3f(N, L.dir), 0.f);
        const R G = (lift<R>(NdotL) / (NdotL * (1.0f - k) + k)) * (lift<R>(NdotV) / (NdotV * (1.0f - k) + k));   // GeometrySmith :34-46
        const S hv = 1.0f - dmax(dot3(H, V), 0.f);
        const S hv2 = hv * hv;
        const S p5 = (hv2 * hv2) * hv;                          // pow(1 - cosTheta, 5)
        S den4 = dmax((NdotV * 4.0f) * NdotL, 0.01f);          // clamp(4 N.V N.L, 0.01) :125-128
        const R ndf_g = NDF * G;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const M F0 = 0.4f * (1.f - metallic) + 1.0f * metallic;   // :103
            const R Fr = F0 + (1.0f - F0) * p5;                           // fresnelSchlick :48-53
            const S radiance = (cosine * L.dir_c[c]) * L.dir_i;           // :105
            const R KD = (1.0f - Fr) * (1.0f - metallic);                 // :117-119
            diffuse[c] = diffuse[c] + KD * radiance;
            specular[c] = ((ndf_g * Fr) / den4) * radiance;               // :122-129
        }
    } else {
#pragma unroll
        for (int c = 0; c < 3; c++) {
            diffuse[c] = diffuse[c] + (cosine * L.dir_c[c]) * L.dir_i;    // :131-135
            specular[c] = lift<R>(0.f);
        }
    }
}

__device__ __forceinline__ float mean_tm(const float* p, int Tm) {   // torch.sum(x, dim=2) / total
    float s = 0.f;
    for (int t = 0; t < Tm; t++) s += __ldg(p + t);
    return s / (float)Tm;
}

// surface normal the way the mirror forms it: float64 cross product of float32 edge vectors, normalised, back to float32
__device__ __forceinline__ void normal_f64(const float v[9], float N[3]) {
    const double ax = (double)(v[0] - v[3]), ay = (double)(v[1] - v[4]), az = (double)(v[2] - v[5]);   // v10 = v0 - v1
    const double bx = (double)(v[6] - v[3]), by = (double)(v[7] - v[4]), bz = (double)(v[8] - v[5]);   // v12 = v2 - v1
    const double cx = by * az - bz * ay, cy = bz * ax - bx * az, cz = bx * ay - by * ax;               // cross(v12, v10)
    const double n = fmax(sqrt(cx * cx + cy * cy + cz * cz), 1e-12);
    N[0] = (float)(cx / n); N[1] = (float)(cy / n); N[2] = (float)(cz / n);
}

__global__ void __launch_bounds__(128)
k_surface_lighting_fwd(const float* __restrict__ vertices, const int32_t* __restrict__ faces, const float* __restrict__ textures,
                       const float* __restrict__ metallic, const float* __restrict__ roughness, const float* __restrict__ eye,
                       float* __restrict__ out, LightParams L, int B, int Bv, int Bf, int Be, int nv, int nf, int T, int Tm) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * nf) return;
    const int b = (int)(i / nf), f = (int)(i % nf);
    const int32_t* fi = faces + ((size_t)(Bf == 1 ? 0 : b) * nf + f) * 3;
    const float* vb = vertices + (size_t)(Bv == 1 ? 0 : b) * nv * 3;
    float v[9];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float* q = vb + (size_t)__ldg(fi + k) * 3;
        v[3 * k] = __ldg(q); v[3 * k + 1] = __ldg(q + 1); v[3 * k + 2] = __ldg(q + 2);
    }
    float N[3], pos[3], d[3], s[3];
    normal_f64(v, N);
#pragma unroll
    for (int k = 0; k < 3; k++) pos[k] = ((v[k] + v[3 + k]) + v[6 + k]) / 3.0f;   // torch.sum(face_vertices, dim=2) / 3.0
    const bool spec = L.with_specular && metallic != nullptr && roughness != nullptr && eye != nullptr;
    LightParams Lf = L;
    Lf.with_specular = spec ? 1 : 0;
    const float m = spec ? mean_tm(metallic + (size_t)i * Tm, Tm) : 0.f;
    const float r = spec ? mean_tm(roughness + (size_t)i * Tm, Tm) : 1.f;
    face_light<float>(N, pos, Lf, spec ? eye + (size_t)(Be == 1 ? 0 : b) * 3 : nullptr, m, r, d, s);
    const float* tx = textures + (size_t)i * T * 3;
    float* o = out + (size_t)i * T * 3;
    for (int t = 0; t < T; t++)
#pragma unroll
        for (int c = 0; c < 3; c++) o[t * 3 + c] = fminf(fmaxf(__ldg(tx + t * 3 + c) * d[c] + 1.0f * s[c], 0.0f), 1.0f);   // lighting.py:199-204
}

__global__ void __launch_bounds__(128)
k_surface_lighting_bwd(const float* __restrict__ vertices, const int32_t* __restrict__ faces, const float* __restrict__ textures,
                       const float* __restrict__ metallic, const float* __restrict__ roughness, const float* __restrict__ eye,
                       const float* __restrict__ grad_out, float* __restrict__ grad_textures, float* __restrict__ grad_vertices,
                       float* __restrict__ grad_metallic, float* __restrict__ grad_roughness, LightParams L, int B, int Bv, int Bf,
                       int Be, int nv, int nf, int T, int Tm) {
    typedef Dual<9> D;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * nf) return;
    const int b = (int)(i / nf), f = (int)(i % nf);
    const int32_t* fi = faces + ((size_t)(Bf == 1 ? 0 : b) * nf + f) * 3;
    const size_t vbase = (size_t)(Bv == 1 ? 0 : b) * nv * 3;
    int idx[3];
    float v[9];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        idx[k] = __ldg(fi + k);
        const float* q = vertices + vbase + (size_t)idx[k] * 3;
        v[3 * k] = __ldg(q); v[3 * k + 1] = __ldg(q + 1); v[3 * k + 2] = __ldg(q + 2);
    }
    const bool spec = L.with_specular && metallic != nullptr && roughness != nullptr && eye != nullptr;
    LightParams Lf = L;
    Lf.with_specular = spec ? 1 : 0;
    const float m = spec ? mean_tm(metallic + (size_t)i * Tm, Tm) : 0.f;
    const float r = spec ? mean_tm(roughness + (size_t)i * Tm, Tm) : 1.f;
    const float* ey = spec ? eye + (size_t)(Be == 1 ? 0 : b) * 3 : nullptr;
    // values exactly as the forward formed them (masks of the clamp, d out / d tex)
    float N[3], pos[3], d[3], s[3];
    normal_f64(v, N);
#pragma unroll
    for (int k = 0; k < 3; k++) pos[k] = ((v[k] + v[3 + k]) + v[6 + k]) / 3.0f;
    face_light<float>(N, pos, Lf, ey, m, r, d, s);
    // upstream gradient folded over the texels: Gd[c] = sum_t g * mask * tex, Gs[c] = sum_t g * mask
    float Gd[3] = {0.f, 0.f, 0.f}, Gs[3] = {0.f, 0.f, 0.f};
    const float* tx = textures + (size_t)i * T * 3;
    const float* go = grad_out + (size_t)i * T * 3;
    float* gt = grad_textures + (size_t)i * T * 3;
    for (int t = 0; t < T; t++)
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const float x = __ldg(tx + t * 3 + c), val = x * d[c] + 1.0f * s[c];
            const float g = (val >= 0.0f && val <= 1.0f) ? __ldg(go + t * 3 + c) : 0.f;   // torch.clamp passes the gradient on [min, max]
            gt[t * 3 + c] = g * d[c];
            Gd[c] += g * x;
            Gs[c] += g;
        }
    if (grad_metallic != nullptr || grad_roughness != nullptr) {
        // derivatives of (diffuse, specular) w.r.t. the face's mean metallic and roughness, geometry held constant; each
        // is spread evenly over the face's Tm texels (the gradient of the mean).  0 without the specular branch.
        float gm = 0.f, gr = 0.f;
        if (spec) {
            Dual<2> dm[3], sm[3];
            face_light<float, Dual<2>>(N, pos, Lf, ey, dvar<2>(m, 0), dvar<2>(r, 1), dm, sm);
#pragma unroll
            for (int c = 0; c < 3; c++) {
                gm += Gd[c] * dm[c].d[0] + Gs[c] * sm[c].d[0];
                gr += Gd[c] * dm[c].d[1] + Gs[c] * sm[c].d[1];
            }
            gm = gm / (float)Tm;
            gr = gr / (float)Tm;
        }
        if (grad_metallic != nullptr)
            for (int t = 0; t < Tm; t++) grad_metallic[(size_t)i * Tm + t] = gm;
        if (grad_roughness != nullptr)
            for (int t = 0; t < Tm; t++) grad_roughness[(size_t)i * Tm + t] = gr;
    }
    if (grad_vertices == nullptr) return;
    // derivatives of (diffuse, specular) w.r.t. the 9 vertex coordinates
    D dv[9];
#pragma unroll
    for (int k = 0; k < 9; k++) dv[k] = dvar<9>(v[k], k);
    D a[3] = {dv[0] - dv[3], dv[1] - dv[4], dv[2] - dv[5]};    // v10
    D bb[3] = {dv[6] - dv[3], dv[7] - dv[4], dv[8] - dv[5]};   // v12
    D Nd[3] = {bb[1] * a[2] - bb[2] * a[1], bb[2] * a[0] - bb[0] * a[2], bb[0] * a[1] - bb[1] * a[0]};
    normalize3(Nd, 1e-12f);
    D pd[3];
#pragma unroll
    for (int k = 0; k < 3; k++) pd[k] = ((dv[k] + dv[3 + k]) + dv[6 + k]) / 3.0f;
    D dd[3], sd[3];
    face_light<D>(Nd, pd, Lf, ey, m, r, dd, sd);
    float* gv = grad_vertices + vbase;
#pragma unroll
    for (int k = 0; k < 9; k++) {
        float acc = 0.f;
#pragma unroll
        for (int c = 0; c < 3; c++) acc += Gd[c] * dd[c].d[k] + Gs[c] * sd[c].d[k];
        if (acc != 0.f) atomicAdd(gv + (size_t)idx[k / 3] * 3 + (k % 3), acc);
    }
}

int check_args(const char* fn, const void* vertices, const void* faces, const void* textures, int B, int Bv, int Bf, int Be, int nv,
               int nf, int T, int Tm) {
    if (!vertices || !faces || !textures) return b200r_fail(B200R_EINVAL, "%s: NULL pointer argument", fn);
    if (B <= 0 || nv <= 0 || nf <= 0 || T <= 0 || Tm < 0) return b200r_fail(B200R_EINVAL, "%s: non-positive size", fn);
    if ((Bv != 1 && Bv != B) || (Bf != 1 && Bf != B) || (Be != 0 && Be != 1 && Be != B))
        return b200r_fail(B200R_EINVAL, "%s: vertices / faces / eye batch must be 1 or B", fn);
    return 0;
}

LightParams make(float amb_i, const float* amb_c, float dir_i, const float* dir_c, const float* dir, int with_specular) {
    LightParams L;
    L.amb_i = amb_i; L.dir_i = dir_i; L.with_specular = with_specular;
    for (int k = 0; k < 3; k++) { L.amb_c[k] = amb_c[k]; L.dir_c[k] = dir_c[k]; L.dir[k] = dir[k]; }
    return L;
}

}  // namespace

extern "C" {

int b200r_surface_lighting_forward(const float* vertices, const int32_t* faces, const float* textures, const float* metallic,
                                   const float* roughness, const float* eye, float* out_textures, int B, int vertices_batch,
                                   int faces_batch, int eye_batch, int nv, int nf, int T, int Tm, float ambient_intensity,
                                   const float* ambient_color, float directional_intensity, const float* directional_color,
                                   const float* direction, int with_specular, void* stream) {
    int rc = check_args("b200r_surface_lighting_forward", vertices, faces, textures, B, vertices_batch, faces_batch, eye_batch, nv, nf, T, Tm);
    if (rc) return rc;
    if (!out_textures || !ambient_color || !directional_color || !direction)
        return b200r_fail(B200R_EINVAL, "b200r_surface_lighting_forward: NULL pointer argument");
    cudaStream_t st = (cudaStream_t)stream;
    const LightParams L = make(ambient_intensity, ambient_color, directional_intensity, directional_color, direction, with_specular);
    const long total = (long)B * nf;
    return b200r_launch("k_surface_lighting_fwd", B200R_K_LIGHTING, k_surface_lighting_fwd, (unsigned)((total + 127) / 128), 128, 0, st,
                        vertices, faces, textures, metallic, roughness, eye_batch ? eye : nullptr, out_textures, L, B,
                        vertices_batch, faces_batch, eye_batch ? eye_batch : 1, nv, nf, T, Tm);
}

int b200r_surface_lighting_backward(const float* vertices, const int32_t* faces, const float* textures, const float* metallic,
                                    const float* roughness, const float* eye, const float* grad_out, float* grad_textures,
                                    float* grad_vertices, float* grad_metallic, float* grad_roughness, int B, int vertices_batch,
                                    int faces_batch, int eye_batch, int nv, int nf, int T, int Tm, float ambient_intensity,
                                    const float* ambient_color, float directional_intensity, const float* directional_color,
                                    const float* direction, int with_specular, void* stream) {
    int rc = check_args("b200r_surface_lighting_backward", vertices, faces, textures, B, vertices_batch, faces_batch, eye_batch, nv, nf, T, Tm);
    if (rc) return rc;
    if (!grad_out || !grad_textures || !ambient_color || !directional_color || !direction)
        return b200r_fail(B200R_EINVAL, "b200r_surface_lighting_backward: NULL pointer argument");
    if ((grad_metallic || grad_roughness) && (!metallic || !roughness || Tm == 0))
        return b200r_fail(B200R_EINVAL, "b200r_surface_lighting_backward: material gradients need metallic, roughness and Tm > 0");
    cudaStream_t st = (cudaStream_t)stream;
    if (grad_vertices != nullptr) {
        if (int rc = b200r_zero(grad_vertices, sizeof(float) * 3 * (size_t)vertices_batch * nv, st, "memset grad_vertices")) return rc;
    }
    const LightParams L = make(ambient_intensity, ambient_color, directional_intensity, directional_color, direction, with_specular);
    const long total = (long)B * nf;
    return b200r_launch("k_surface_lighting_bwd", B200R_K_LIGHTING, k_surface_lighting_bwd, (unsigned)((total + 127) / 128), 128, 0, st,
                        vertices, faces, textures, metallic, roughness, eye_batch ? eye : nullptr, grad_out, grad_textures,
                        grad_vertices, grad_metallic, grad_roughness, L, B, vertices_batch, faces_batch,
                        eye_batch ? eye_batch : 1, nv, nf, T, Tm);
}

}  // extern "C"
