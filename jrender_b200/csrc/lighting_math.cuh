// lighting_math.cuh -- the per-face and per-texel light arithmetic of the fused lighting kernels (lighting_api.cu) and
// the G-buffer kernels (gbuffer_api.cu): one statement of face_light, the float64 flat normal, the face centroid and the
// texel normal, so that both files evaluate the same float32 operation sequence.
#pragma once
#include "dual.cuh"

namespace b200r {

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

// d(N_j)/d(v_k) of normal_f64's normal, N's value and len as normal_f64 returned them.
// The normal's value and norm are the forward's float64 ones: on a sliver the float32 cross product and its norm
// cancel, and the derivative would be taken at another normal (and the relu branches chosen there).  Only c's
// partials come from the float32 duals; each is a sum of edge components, free of that cancellation.  They pass
// through normalize's Jacobian (I - N N^T) / |c|, or I / 1e-12 on its eps path, where the norm is the constant
// (clamp_min's rule: |c| == 1e-12 exactly still differentiates through the norm).
__device__ __forceinline__ void normal_duals(const float v[9], const float N[3], double len, Dual<9> Nd[3]) {
    typedef Dual<9> D;
    D dv[9];
#pragma unroll
    for (int k = 0; k < 9; k++) dv[k] = dvar<9>(v[k], k);
    const D a[3] = {dv[0] - dv[3], dv[1] - dv[4], dv[2] - dv[5]};    // v10
    const D bb[3] = {dv[6] - dv[3], dv[7] - dv[4], dv[8] - dv[5]};   // v12
    const D c[3] = {bb[1] * a[2] - bb[2] * a[1], bb[2] * a[0] - bb[0] * a[2], bb[0] * a[1] - bb[1] * a[0]};
    const float n = (float)fmax(len, 1e-12), inv = 1.f / n;
    const bool on_eps = !(len >= 1e-12);
#pragma unroll
    for (int j = 0; j < 3; j++) Nd[j].v = N[j];
#pragma unroll
    for (int k = 0; k < 9; k++) {
        const float Ndc = on_eps ? 0.f : (N[0] * c[0].d[k] + N[1] * c[1].d[k]) + N[2] * c[2].d[k];
#pragma unroll
        for (int j = 0; j < 3; j++) Nd[j].d[k] = (c[j].d[k] - N[j] * Ndc) * inv;
    }
}

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

inline LightParams make(float amb_i, const float* amb_c, float dir_i, const float* dir_c, const float* dir, int with_specular) {
    LightParams L;
    L.amb_i = amb_i; L.dir_i = dir_i; L.with_specular = with_specular;
    for (int k = 0; k < 3; k++) { L.amb_c[k] = amb_c[k]; L.dir_c[k] = dir_c[k]; L.dir[k] = dir[k]; }
    return L;
}

}  // namespace b200r
