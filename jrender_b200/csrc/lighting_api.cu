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
//
//   b200r_normal_mapped_lighting_forward / _backward  <-  the same branch with mesh.normal_textures (one normal per texel,
//        structures/mesh.py:276-284 surface_ResNormals; directional_lighting.py's 4-D branch, per-texel materials)
//
// One thread per texel forward; one warp per face backward (see k_nm_lighting_bwd).
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

// x / max(||x||, eps)   (F.normalize / jt.normalize: clamp_min, so the norm's derivative passes at ||x|| == eps)
template <class S>
__device__ __forceinline__ void normalize3(S x[3], float eps) {
    const S n = dclamp_min(dsqrt(dot3(x, x)), eps);
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
        S den4 = dclamp_min((NdotV * 4.0f) * NdotL, 0.01f);    // clamp(4 N.V N.L, min=0.01) :125-128
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

// torch.clamp(x, 0, 1): NaN stays NaN (fmaxf alone would return 0 for it)
__device__ __forceinline__ float clamp01(float x) { return x != x ? x : fminf(fmaxf(x, 0.0f), 1.0f); }

// surface normal the way the mirror forms it: float64 cross product of float32 edge vectors, normalised, back to float32.
// Returns the unclamped norm |c| (NaN for a non-finite face).
__device__ __forceinline__ double normal_f64(const float v[9], float N[3]) {
    const double ax = (double)(v[0] - v[3]), ay = (double)(v[1] - v[4]), az = (double)(v[2] - v[5]);   // v10 = v0 - v1
    const double bx = (double)(v[6] - v[3]), by = (double)(v[7] - v[4]), bz = (double)(v[8] - v[5]);   // v12 = v2 - v1
    const double cx = by * az - bz * ay, cy = bz * ax - bx * az, cz = bx * ay - by * ax;               // cross(v12, v10)
    const double len = sqrt(cx * cx + cy * cy + cz * cz);
    const double n = fmax(len, 1e-12);
    N[0] = (float)(cx / n); N[1] = (float)(cy / n); N[2] = (float)(cz / n);
    return len;
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
        for (int c = 0; c < 3; c++) o[t * 3 + c] = clamp01(__ldg(tx + t * 3 + c) * d[c] + 1.0f * s[c]);   // lighting.py:199-204
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
    const double len = normal_f64(v, N);
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
                gr += Gs[c] * sm[c].d[1];   // diffuse does not depend on roughness: no Gd term (a NaN Gd stays out)
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
    const D c[3] = {bb[1] * a[2] - bb[2] * a[1], bb[2] * a[0] - bb[0] * a[2], bb[0] * a[1] - bb[1] * a[0]};
    // The normal's value and norm are the forward's float64 ones: on a sliver the float32 cross product and its norm
    // cancel, and the derivative would be taken at another normal (and the relu branches chosen there).  Only c's
    // partials come from the float32 duals; each is a sum of edge components, free of that cancellation.  They pass
    // through normalize's Jacobian (I - N N^T) / |c|, or I / 1e-12 on its eps path, where the norm is the constant
    // (clamp_min's rule: |c| == 1e-12 exactly still differentiates through the norm).
    const float n = (float)fmax(len, 1e-12), inv = 1.f / n;
    const bool on_eps = !(len >= 1e-12);
    D Nd[3];
#pragma unroll
    for (int j = 0; j < 3; j++) Nd[j].v = N[j];
#pragma unroll
    for (int k = 0; k < 9; k++) {
        const float Ndc = on_eps ? 0.f : (N[0] * c[0].d[k] + N[1] * c[1].d[k]) + N[2] * c[2].d[k];
#pragma unroll
        for (int j = 0; j < 3; j++) Nd[j].d[k] = (c[j].d[k] - N[j] * Ndc) * inv;
    }
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

// ---- normal-mapped surface lighting: one normal per texel (Lighting.execute with mesh.normal_textures) --------------
//
// N = normalize(n_t . TBN) per texel (mesh.py:276-284, surface_ResNormals: a 1x3 by 3x3 matmul, rows T, B, N), the face
// centroid as position, the texel's own metallic and roughness (directional_lighting.py's 4-D branch does not average
// them).  The TBN is fixed at load time, so the vertices reach the result only through the centroid.

// face centroid exactly as the flat kernel forms it: torch.sum(face_vertices, dim=2) / 3.0
__device__ __forceinline__ void face_centroid(const float* __restrict__ vertices, const int32_t* __restrict__ faces, int b, int f,
                                              int Bv, int Bf, int nv, int nf, float pos[3]) {
    const int32_t* fi = faces + ((size_t)(Bf == 1 ? 0 : b) * nf + f) * 3;
    const float* vb = vertices + (size_t)(Bv == 1 ? 0 : b) * nv * 3;
    const float* q0 = vb + (size_t)__ldg(fi) * 3;
    const float* q1 = vb + (size_t)__ldg(fi + 1) * 3;
    const float* q2 = vb + (size_t)__ldg(fi + 2) * 3;
#pragma unroll
    for (int k = 0; k < 3; k++) pos[k] = ((__ldg(q0 + k) + __ldg(q1 + k)) + __ldg(q2 + k)) / 3.0f;
}

// normalize(n_t . TBN, eps=1e-12): N_j = (n0 * TBN[0][j] + n1 * TBN[1][j]) + n2 * TBN[2][j]
template <class S>
__device__ __forceinline__ void texel_normal(const S nt[3], const float* __restrict__ tbn, S N[3]) {
#pragma unroll
    for (int j = 0; j < 3; j++) N[j] = (nt[0] * __ldg(tbn + j) + nt[1] * __ldg(tbn + 3 + j)) + nt[2] * __ldg(tbn + 6 + j);
    normalize3(N, 1e-12f);
}

// one thread per (batch, face, texel): consecutive threads read consecutive texels of every stream
__global__ void __launch_bounds__(256)
k_nm_lighting_fwd(const float* __restrict__ vertices, const int32_t* __restrict__ faces, const float* __restrict__ textures,
                  const float* __restrict__ normal_textures, const float* __restrict__ tbn, const float* __restrict__ metallic,
                  const float* __restrict__ roughness, const float* __restrict__ eye, float* __restrict__ out, LightParams L,
                  int B, int Bv, int Bf, int Be, int Bn, int Bt, int nv, int nf, int T) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * nf * T) return;
    const long bf = i / T;
    const int t = (int)(i % T), b = (int)(bf / nf), f = (int)(bf % nf);
    float pos[3], nt[3], N[3], d[3], s[3];
    face_centroid(vertices, faces, b, f, Bv, Bf, nv, nf, pos);
    const float* np_ = normal_textures + (((size_t)(Bn == 1 ? 0 : b) * nf + f) * T + t) * 3;
#pragma unroll
    for (int k = 0; k < 3; k++) nt[k] = __ldg(np_ + k);
    texel_normal(nt, tbn + ((size_t)(Bt == 1 ? 0 : b) * nf + f) * 9, N);
    const bool spec = L.with_specular && metallic != nullptr && roughness != nullptr && eye != nullptr;
    LightParams Lf = L;
    Lf.with_specular = spec ? 1 : 0;
    const float m = spec ? __ldg(metallic + i) : 0.f;
    const float r = spec ? __ldg(roughness + i) : 1.f;
    face_light<float>(N, pos, Lf, spec ? eye + (size_t)(Be == 1 ? 0 : b) * 3 : nullptr, m, r, d, s);
    const float* tx = textures + (size_t)i * 3;
#pragma unroll
    for (int c = 0; c < 3; c++) out[(size_t)i * 3 + c] = clamp01(__ldg(tx + c) * d[c] + 1.0f * s[c]);
}

// One warp per (normal-texture batch, face); lanes stride over the face's texels.  With a batch-1 normal texture the warp
// runs every batch element in turn, so each lane owns its texels' grad_normal_textures across the batch and sums it
// without atomics.  Three evaluations per texel: float values (clamp mask, grad_textures), Dual<6> over the tangent-space
// normal and the centroid (grad_normal_textures, grad_vertices), Dual<2> over the texel's metallic and roughness.  The
// centroid derivative is reduced over the warp and spread as d pos / d v = 1/3: 9 atomics per (batch, face).
__global__ void __launch_bounds__(128)
k_nm_lighting_bwd(const float* __restrict__ vertices, const int32_t* __restrict__ faces, const float* __restrict__ textures,
                  const float* __restrict__ normal_textures, const float* __restrict__ tbn, const float* __restrict__ metallic,
                  const float* __restrict__ roughness, const float* __restrict__ eye, const float* __restrict__ grad_out,
                  float* __restrict__ grad_textures, float* __restrict__ grad_normal_textures, float* __restrict__ grad_vertices,
                  float* __restrict__ grad_metallic, float* __restrict__ grad_roughness, LightParams L, int B, int Bv, int Bf,
                  int Be, int Bn, int Bt, int nv, int nf, int T) {
    typedef Dual<6> D;
    const long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= (long)Bn * nf) return;   // warp-uniform
    const int bn = (int)(w / nf), f = (int)(w % nf);
    const int b0 = Bn == 1 ? 0 : bn, b1 = Bn == 1 ? B : bn + 1;
    const bool spec = L.with_specular && metallic != nullptr && roughness != nullptr && eye != nullptr;
    LightParams Lf = L;
    Lf.with_specular = spec ? 1 : 0;
    const bool want_geom = grad_normal_textures != nullptr || grad_vertices != nullptr;
    const float* nface = normal_textures + ((size_t)bn * nf + f) * T * 3;
    float* gnface = grad_normal_textures != nullptr ? grad_normal_textures + ((size_t)bn * nf + f) * T * 3 : nullptr;
    for (int b = b0; b < b1; b++) {
        float pos[3];
        face_centroid(vertices, faces, b, f, Bv, Bf, nv, nf, pos);
        const float* tb = tbn + ((size_t)(Bt == 1 ? 0 : b) * nf + f) * 9;
        const float* ey = spec ? eye + (size_t)(Be == 1 ? 0 : b) * 3 : nullptr;
        const size_t base = ((size_t)b * nf + f) * T;
        float gpos[3] = {0.f, 0.f, 0.f};
        for (int t = lane; t < T; t += 32) {
            const size_t i = base + t;
            float nt[3], N[3], d[3], s[3], Gd[3], Gs[3];
#pragma unroll
            for (int k = 0; k < 3; k++) nt[k] = __ldg(nface + (size_t)t * 3 + k);
            texel_normal(nt, tb, N);
            const float m = spec ? __ldg(metallic + i) : 0.f;
            const float r = spec ? __ldg(roughness + i) : 1.f;
            face_light<float>(N, pos, Lf, ey, m, r, d, s);
#pragma unroll
            for (int c = 0; c < 3; c++) {
                const float x = __ldg(textures + i * 3 + c), val = x * d[c] + 1.0f * s[c];
                const float g = (val >= 0.0f && val <= 1.0f) ? __ldg(grad_out + i * 3 + c) : 0.f;   // torch.clamp's mask
                if (grad_textures != nullptr) grad_textures[i * 3 + c] = g * d[c];
                Gd[c] = g * x;
                Gs[c] = g;
            }
            if (grad_metallic != nullptr || grad_roughness != nullptr) {
                float gm = 0.f, gr = 0.f;
                if (spec) {
                    Dual<2> dm[3], sm[3];
                    face_light<float, Dual<2>>(N, pos, Lf, ey, dvar<2>(m, 0), dvar<2>(r, 1), dm, sm);
#pragma unroll
                    for (int c = 0; c < 3; c++) {
                        gm += Gd[c] * dm[c].d[0] + Gs[c] * sm[c].d[0];
                        gr += Gs[c] * sm[c].d[1];   // as in the flat kernel: no Gd term
                    }
                }
                if (grad_metallic != nullptr) grad_metallic[i] = gm;
                if (grad_roughness != nullptr) grad_roughness[i] = gr;
            }
            if (want_geom) {
                D ntd[3], Nd[3], pd[3], dd[3], sd[3];
#pragma unroll
                for (int k = 0; k < 3; k++) {
                    ntd[k] = dvar<6>(nt[k], k);
                    pd[k] = dvar<6>(pos[k], 3 + k);
                }
                texel_normal(ntd, tb, Nd);
                face_light<D>(Nd, pd, Lf, ey, m, r, dd, sd);
                float gk[6];
#pragma unroll
                for (int k = 0; k < 6; k++) {
                    float acc = 0.f;
#pragma unroll
                    for (int c = 0; c < 3; c++) acc += Gd[c] * dd[c].d[k] + Gs[c] * sd[c].d[k];
                    gk[k] = acc;
                }
                if (gnface != nullptr) {
                    float* gn = gnface + (size_t)t * 3;
#pragma unroll
                    for (int k = 0; k < 3; k++) gn[k] = b == b0 ? gk[k] : gn[k] + gk[k];   // this lane owns texel t
                }
#pragma unroll
                for (int k = 0; k < 3; k++) gpos[k] += gk[3 + k];
            }
        }
        if (grad_vertices != nullptr) {
#pragma unroll
            for (int k = 0; k < 3; k++)
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) gpos[k] += __shfl_xor_sync(0xffffffffu, gpos[k], o);
            if (lane == 0) {
                const int32_t* fi = faces + ((size_t)(Bf == 1 ? 0 : b) * nf + f) * 3;
                float* gv = grad_vertices + (size_t)(Bv == 1 ? 0 : b) * nv * 3;
#pragma unroll
                for (int k = 0; k < 3; k++) {
                    const float g = gpos[k] / 3.0f;   // d pos_k / d v_jk = 1/3 for each of the three vertices
                    if (g != 0.f)
#pragma unroll
                        for (int j = 0; j < 3; j++) atomicAdd(gv + (size_t)__ldg(fi + j) * 3 + k, g);
                }
            }
        }
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

int check_nm_args(const char* fn, const void* vertices, const void* faces, const void* textures, const void* normal_textures,
                  const void* tbn, const void* ambient_color, const void* directional_color, const void* direction, int B, int Bv,
                  int Bf, int Be, int Bn, int n_nf, int n_T, int Bt, int t_nf, int nv, int nf, int T) {
    if (!vertices || !faces || !textures || !normal_textures || !tbn || !ambient_color || !directional_color || !direction)
        return b200r_fail(B200R_EINVAL, "%s: NULL pointer argument", fn);
    if (B <= 0 || nv <= 0 || nf <= 0 || T <= 0) return b200r_fail(B200R_EINVAL, "%s: non-positive size", fn);
    if ((Bv != 1 && Bv != B) || (Bf != 1 && Bf != B) || (Be != 0 && Be != 1 && Be != B) || (Bn != 1 && Bn != B) ||
        (Bt != 1 && Bt != B))
        return b200r_fail(B200R_EINVAL, "%s: vertices / faces / eye / normal_textures / tbn batch must be 1 or B", fn);
    if (n_nf != nf || n_T != T || t_nf != nf)
        return b200r_fail(B200R_EINVAL, "%s: normal_textures [%d faces, %d texels] / tbn [%d faces] do not match textures [%d, %d]",
                          fn, n_nf, n_T, t_nf, nf, T);
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

int b200r_normal_mapped_lighting_forward(const float* vertices, const int32_t* faces, const float* textures,
                                         const float* normal_textures, const float* tbn, const float* metallic,
                                         const float* roughness, const float* eye, float* out_textures, int B, int vertices_batch,
                                         int faces_batch, int eye_batch, int normal_batch, int normal_faces, int normal_texels,
                                         int tbn_batch, int tbn_faces, int nv, int nf, int T, float ambient_intensity,
                                         const float* ambient_color, float directional_intensity, const float* directional_color,
                                         const float* direction, int with_specular, void* stream) {
    const char* fn = "b200r_normal_mapped_lighting_forward";
    int rc = check_nm_args(fn, vertices, faces, textures, normal_textures, tbn, ambient_color, directional_color, direction, B,
                           vertices_batch, faces_batch, eye_batch, normal_batch, normal_faces, normal_texels, tbn_batch, tbn_faces,
                           nv, nf, T);
    if (rc) return rc;
    if (!out_textures) return b200r_fail(B200R_EINVAL, "%s: NULL pointer argument", fn);
    const LightParams L = make(ambient_intensity, ambient_color, directional_intensity, directional_color, direction, with_specular);
    const long total = (long)B * nf * T;
    return b200r_launch("k_nm_lighting_fwd", B200R_K_LIGHTING, k_nm_lighting_fwd, (unsigned)((total + 255) / 256), 256, 0,
                        (cudaStream_t)stream, vertices, faces, textures, normal_textures, tbn, metallic, roughness,
                        eye_batch ? eye : nullptr, out_textures, L, B, vertices_batch, faces_batch, eye_batch ? eye_batch : 1,
                        normal_batch, tbn_batch, nv, nf, T);
}

int b200r_normal_mapped_lighting_backward(const float* vertices, const int32_t* faces, const float* textures,
                                          const float* normal_textures, const float* tbn, const float* metallic,
                                          const float* roughness, const float* eye, const float* grad_out, float* grad_textures,
                                          float* grad_normal_textures, float* grad_vertices, float* grad_metallic,
                                          float* grad_roughness, int B, int vertices_batch, int faces_batch, int eye_batch,
                                          int normal_batch, int normal_faces, int normal_texels, int tbn_batch, int tbn_faces,
                                          int nv, int nf, int T, float ambient_intensity, const float* ambient_color,
                                          float directional_intensity, const float* directional_color, const float* direction,
                                          int with_specular, void* stream) {
    const char* fn = "b200r_normal_mapped_lighting_backward";
    int rc = check_nm_args(fn, vertices, faces, textures, normal_textures, tbn, ambient_color, directional_color, direction, B,
                           vertices_batch, faces_batch, eye_batch, normal_batch, normal_faces, normal_texels, tbn_batch, tbn_faces,
                           nv, nf, T);
    if (rc) return rc;
    if (!grad_out) return b200r_fail(B200R_EINVAL, "%s: NULL pointer argument", fn);
    if ((grad_metallic || grad_roughness) && (!metallic || !roughness))
        return b200r_fail(B200R_EINVAL, "%s: material gradients need metallic and roughness", fn);
    cudaStream_t st = (cudaStream_t)stream;
    if (grad_vertices != nullptr) {
        if (int rc = b200r_zero(grad_vertices, sizeof(float) * 3 * (size_t)vertices_batch * nv, st, "memset grad_vertices")) return rc;
    }
    const LightParams L = make(ambient_intensity, ambient_color, directional_intensity, directional_color, direction, with_specular);
    const long threads = (long)normal_batch * nf * 32;
    return b200r_launch("k_nm_lighting_bwd", B200R_K_LIGHTING, k_nm_lighting_bwd, (unsigned)((threads + 127) / 128), 128, 0, st,
                        vertices, faces, textures, normal_textures, tbn, metallic, roughness, eye_batch ? eye : nullptr, grad_out,
                        grad_textures, grad_normal_textures, grad_vertices, grad_metallic, grad_roughness, L, B, vertices_batch,
                        faces_batch, eye_batch ? eye_batch : 1, normal_batch, tbn_batch, nv, nf, T);
}

}  // extern "C"
