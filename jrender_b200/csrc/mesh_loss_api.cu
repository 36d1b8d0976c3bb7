// mesh_loss_api.cu -- fused mesh regularisers of the fitting loop (SURVEY.md section 8f rank 4).
//
//   b200r_flatten_loss    <- jrender/loss/flatten_loss.py:38-79   (FlattenLoss.execute)
//   b200r_laplacian_loss  <- jrender/loss/laplacian_loss.py:29-36 (LaplacianLoss.execute)
//
// Each entry point evaluates the loss AND its gradient w.r.t. the vertices in one launch, so the
// autograd backward is a single scale (grad * upstream).  The reference runs ~60 (flatten) and
// ~8 (laplacian) tensor ops forward and as many again backward; in the launch-bound demo2 loop
// these were more than half of all launches.
//
// FlattenLoss: one thread per (batch, edge).  The expression of flatten_loss.py:48-73 is evaluated
// in forward-mode automatic differentiation over the 12 coordinates of the edge's four vertices
// (a value + 12 partials per intermediate), which reproduces the reference's arithmetic for the
// value exactly in source order and yields the exact derivative of that same expression -- no
// hand-derived formula to get wrong.  LaplacianLoss: one thread per (batch, vertex) computes
// y_i = diag_i x_i + sum_k w_ik x_nbr(i,k) and scatters 2 y_i (diag_i, w_ik) with atomics.
#include "../../include/b200raster.h"
#include "api_util.cuh"

namespace {

constexpr int ND = 12;

struct Dual {
    float v;
    float d[ND];
};

__device__ __forceinline__ Dual mk(float v) {
    Dual r; r.v = v;
#pragma unroll
    for (int i = 0; i < ND; i++) r.d[i] = 0.f;
    return r;
}
__device__ __forceinline__ Dual var(float v, int i) { Dual r = mk(v); r.d[i] = 1.f; return r; }
__device__ __forceinline__ Dual operator+(const Dual& a, const Dual& b) {
    Dual r; r.v = a.v + b.v;
#pragma unroll
    for (int i = 0; i < ND; i++) r.d[i] = a.d[i] + b.d[i];
    return r;
}
__device__ __forceinline__ Dual operator-(const Dual& a, const Dual& b) {
    Dual r; r.v = a.v - b.v;
#pragma unroll
    for (int i = 0; i < ND; i++) r.d[i] = a.d[i] - b.d[i];
    return r;
}
__device__ __forceinline__ Dual operator*(const Dual& a, const Dual& b) {
    Dual r; r.v = a.v * b.v;
#pragma unroll
    for (int i = 0; i < ND; i++) r.d[i] = a.d[i] * b.v + a.v * b.d[i];
    return r;
}
__device__ __forceinline__ Dual operator/(const Dual& a, const Dual& b) {
    Dual r; r.v = a.v / b.v;
    const float ib = 1.f / b.v;
#pragma unroll
    for (int i = 0; i < ND; i++) r.d[i] = (a.d[i] - r.v * b.d[i]) * ib;
    return r;
}
__device__ __forceinline__ Dual operator+(const Dual& a, float s) { Dual r = a; r.v = a.v + s; return r; }
__device__ __forceinline__ Dual rsub(float s, const Dual& a) {  // s - a
    Dual r; r.v = s - a.v;
#pragma unroll
    for (int i = 0; i < ND; i++) r.d[i] = -a.d[i];
    return r;
}
__device__ __forceinline__ Dual dsqrt(const Dual& a) {
    Dual r; r.v = sqrtf(a.v);
    const float h = 0.5f / r.v;
#pragma unroll
    for (int i = 0; i < ND; i++) r.d[i] = a.d[i] * h;
    return r;
}

struct Dual3 { Dual x, y, z; };
__device__ __forceinline__ Dual3 sub3(const Dual3& a, const Dual3& b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ Dual dot3(const Dual3& a, const Dual3& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }  // .sum(-1) in x, y, z order
__device__ __forceinline__ Dual3 scale3(const Dual3& a, const Dual& s) { return {a.x * s, a.y * s, a.z * s}; }

// flatten_loss.py:48-59 (and :61-72): returns cb = b - a * (ab / (|a|^2 + eps)) and |cb| estimate b_l1 * sin
__device__ __forceinline__ void half_plane(const Dual3& a, const Dual3& b, float eps, Dual3& cb, Dual& cbl1) {
    const Dual al2 = dot3(a, a);
    const Dual bl2 = dot3(b, b);
    const Dual al1 = dsqrt(al2 + eps);
    const Dual bl1 = dsqrt(bl2 + eps);
    const Dual ab = dot3(a, b);
    const Dual cosv = ab / (al1 * bl1 + eps);
    const Dual sinv = dsqrt(rsub(1.f, cosv * cosv) + eps);
    const Dual3 c = scale3(a, ab / (al2 + eps));
    cb = sub3(b, c);
    cbl1 = bl1 * sinv;
}

__global__ void __launch_bounds__(128)
k_flatten_loss(const float* __restrict__ vertices, const int32_t* __restrict__ v0s, const int32_t* __restrict__ v1s,
               const int32_t* __restrict__ v2s, const int32_t* __restrict__ v3s, float* __restrict__ loss,
               float* __restrict__ grad_vertices, int nv, int E, float eps) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    float term = 0.f;
    if (e < E) {
        const int idx[4] = {__ldg(v0s + e), __ldg(v1s + e), __ldg(v2s + e), __ldg(v3s + e)};
        const float* vb = vertices + (size_t)b * nv * 3;
        Dual3 p[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const float* q = vb + (size_t)idx[k] * 3;
            p[k].x = var(__ldg(q), 3 * k); p[k].y = var(__ldg(q + 1), 3 * k + 1); p[k].z = var(__ldg(q + 2), 3 * k + 2);
        }
        const Dual3 a = sub3(p[1], p[0]);
        Dual3 cb1, cb2;
        Dual l1, l2;
        half_plane(a, sub3(p[2], p[0]), eps, cb1, l1);
        half_plane(a, sub3(p[3], p[0]), eps, cb2, l2);
        const Dual cosv = dot3(cb1, cb2) / (l1 * l2 + eps);   // :74
        const Dual c1 = cosv + 1.f;
        const Dual t = c1 * c1;                                // (cos + 1).pow(2) :77
        term = t.v;
        float* gb = grad_vertices + (size_t)b * nv * 3;
#pragma unroll
        for (int k = 0; k < 4; k++)
#pragma unroll
            for (int c = 0; c < 3; c++) atomicAdd(gb + (size_t)idx[k] * 3 + c, t.d[3 * k + c]);
    }
    // block sum -> one atomic per block
    __shared__ float s_part[4];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) term += __shfl_xor_sync(0xffffffffu, term, d);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = term;
    __syncthreads();
    if (threadIdx.x == 0) atomicAdd(loss + b, (s_part[0] + s_part[1]) + (s_part[2] + s_part[3]));
}

__global__ void __launch_bounds__(128)
k_laplacian_loss(const float* __restrict__ vertices, const int32_t* __restrict__ nbr, const float* __restrict__ nbr_w,
                 const float* __restrict__ diag, float* __restrict__ loss, float* __restrict__ grad_vertices,
                 int nv, int maxdeg) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    float term = 0.f;
    if (i < nv) {
        const float* vb = vertices + (size_t)b * nv * 3;
        float* gb = grad_vertices + (size_t)b * nv * 3;
        const float dg = __ldg(diag + i);
        float y[3] = {__ldg(vb + (size_t)i * 3) * dg, __ldg(vb + (size_t)i * 3 + 1) * dg, __ldg(vb + (size_t)i * 3 + 2) * dg};
        for (int k = 0; k < maxdeg; k++) {
            const float w = __ldg(nbr_w + (size_t)i * maxdeg + k);
            if (w == 0.f) continue;   // padding of the neighbour table
            const float* q = vb + (size_t)__ldg(nbr + (size_t)i * maxdeg + k) * 3;
#pragma unroll
            for (int c = 0; c < 3; c++) y[c] += __ldg(q + c) * w;
        }
        term = y[0] * y[0] + y[1] * y[1] + y[2] * y[2];
#pragma unroll
        for (int c = 0; c < 3; c++) atomicAdd(gb + (size_t)i * 3 + c, 2.f * y[c] * dg);
        for (int k = 0; k < maxdeg; k++) {
            const float w = __ldg(nbr_w + (size_t)i * maxdeg + k);
            if (w == 0.f) continue;
            float* q = gb + (size_t)__ldg(nbr + (size_t)i * maxdeg + k) * 3;
#pragma unroll
            for (int c = 0; c < 3; c++) atomicAdd(q + c, 2.f * y[c] * w);
        }
    }
    __shared__ float s_part[4];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) term += __shfl_xor_sync(0xffffffffu, term, d);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = term;
    __syncthreads();
    if (threadIdx.x == 0) atomicAdd(loss + b, (s_part[0] + s_part[1]) + (s_part[2] + s_part[3]));
}

int zero_outputs(const char* who, float* loss, float* grad, int B, int nv, cudaStream_t st) {
    if (int rc = b200r_zero(loss, sizeof(float) * (size_t)B, st, who)) return rc;
    return b200r_zero(grad, sizeof(float) * 3 * (size_t)B * nv, st, who);
}

}  // namespace

extern "C" {

B200R_API int b200r_flatten_loss(const float* vertices, const int32_t* v0s, const int32_t* v1s, const int32_t* v2s,
                                 const int32_t* v3s, float* loss, float* grad_vertices, int batch_size,
                                 int num_vertices, int num_edges, float eps, void* stream) {
    if (!vertices || !v0s || !v1s || !v2s || !v3s || !loss || !grad_vertices)
        return b200r_fail(B200R_EINVAL, "b200r_flatten_loss: NULL pointer");
    if (batch_size <= 0 || num_vertices <= 0 || num_edges < 0 || batch_size > 65535)
        return b200r_fail(B200R_EINVAL, "b200r_flatten_loss: B=%d nv=%d E=%d", batch_size, num_vertices, num_edges);
    cudaStream_t st = (cudaStream_t)stream;
    int rc = zero_outputs("b200r_flatten_loss: memset", loss, grad_vertices, batch_size, num_vertices, st);
    if (rc || num_edges == 0) return rc;
    return b200r_launch("k_flatten_loss", B200R_K_FLATTEN_LOSS, k_flatten_loss, dim3((num_edges + 127) / 128, batch_size), 128, 0, st,
                        vertices, v0s, v1s, v2s, v3s, loss, grad_vertices, num_vertices, num_edges, eps);
}

B200R_API int b200r_laplacian_loss(const float* vertices, const int32_t* neighbours, const float* neighbour_weights,
                                   const float* diag, float* loss, float* grad_vertices, int batch_size,
                                   int num_vertices, int max_degree, void* stream) {
    if (!vertices || !neighbours || !neighbour_weights || !diag || !loss || !grad_vertices)
        return b200r_fail(B200R_EINVAL, "b200r_laplacian_loss: NULL pointer");
    if (batch_size <= 0 || num_vertices <= 0 || max_degree <= 0 || batch_size > 65535)
        return b200r_fail(B200R_EINVAL, "b200r_laplacian_loss: B=%d nv=%d maxdeg=%d", batch_size, num_vertices, max_degree);
    cudaStream_t st = (cudaStream_t)stream;
    int rc = zero_outputs("b200r_laplacian_loss: memset", loss, grad_vertices, batch_size, num_vertices, st);
    if (rc) return rc;
    return b200r_launch("k_laplacian_loss", B200R_K_LAPLACIAN_LOSS, k_laplacian_loss, dim3((num_vertices + 127) / 128, batch_size), 128,
                        0, st, vertices, neighbours, neighbour_weights, diag, loss, grad_vertices, num_vertices, max_degree);
}

}  // extern "C"
