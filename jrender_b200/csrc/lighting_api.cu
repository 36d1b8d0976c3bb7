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
#include "lighting_math.cuh"

using namespace b200r;

namespace {

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
    D Nd[3];
    normal_duals(v, N, len, Nd);
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
