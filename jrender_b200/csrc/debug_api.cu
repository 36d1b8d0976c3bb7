// debug_api.cu -- test-only entry point that checks exact_math.cuh against the plain C
// expressions on the GPU (called by tests/test_exact_math_gpu.py).
#include "../../include/b200raster.h"
#include "api_util.cuh"
#include "exact_math.cuh"

using namespace b200r;

namespace {

__device__ __forceinline__ bool same_f(float x, float y) {
    return __float_as_uint(x) == __float_as_uint(y) || (isnan(x) && isnan(y));
}
__device__ __forceinline__ bool same_d(double x, double y) {
    return __double_as_longlong(x) == __double_as_longlong(y) || (isnan(x) && isnan(y));
}

// mismatch[0] fast_div, [1] f2d_mid, [2] d2f_mid, [3] d2f_mid on exact ties, [4] sigmoid_tail,
// [5] alpha_prod, [6] number of pairs that took the fast_div fast path
__global__ void k_debug_exact_math(const float* __restrict__ a, const float* __restrict__ b, int n, int* mismatch) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = a[i], y = b[i];
    {
        const float r = rcp_refined(y);
        const bool safe = midrange(y);
        const float q1 = fast_div(x, y, r, safe);
        const float q2 = __fdiv_rn(x, y);
        if (!same_f(q1, q2)) atomicAdd(&mismatch[0], 1);
        if (safe && midrange(x)) atomicAdd(&mismatch[6], 1);
        // branch-free optimistic forms (DivGuard): whenever the guard stays up they must equal `/` too
        DivGuard g;
        g.ok = true;
        const float q3 = optimistic_div_exact(x, y, r, safe, g);
        if (g.ok && !same_f(q3, q2)) atomicAdd(&mismatch[0], 1);
        g.ok = true;
        const float q4 = optimistic_rcp(y, g);
        if (g.ok && !same_f(q4, __fdiv_rn(1.f, y))) atomicAdd(&mismatch[0], 1);
        g.ok = true;
        const float q5 = optimistic_div(x, y, r, safe, g);   // relaxed range: exact whenever |x| >= 2^-60 as well
        if (g.ok && midrange(x) && !same_f(q5, q2)) atomicAdd(&mismatch[0], 1);
    }
    if (midrange(x)) {
        if (!same_d(f2d_mid(x), (double)x)) atomicAdd(&mismatch[1], 1);
        const double d = (double)x * (double)y;
        if (d_midrange(d) && !same_f(d2f_mid(d), (float)d)) atomicAdd(&mismatch[2], 1);
        // exact tie: x + half an ulp of x
        const double dx = (double)x;
        const double tie = __hiloint2double(__double2hiint(dx), __double2loint(dx) | 0x10000000);
        if (d_midrange(tie) && !same_f(d2f_mid(tie), (float)tie)) atomicAdd(&mismatch[3], 1);
    }
    {
        const float e = fabsf(x);
        if (!same_f(sigmoid_tail(e), (float)(1.0 / (1.0 + (double)e)))) atomicAdd(&mismatch[4], 1);
        const float al = fminf(fabsf(x), 1.f), D = fminf(fabsf(y), 1.f);
        if (!same_f(alpha_prod(al, D), (float)((double)al * (1.0 - (double)D)))) atomicAdd(&mismatch[5], 1);
    }
}

}  // namespace

extern "C" B200R_API int b200r_debug_exact_math(const float* a, const float* b, int n, int* mismatch7, void* stream) {
    if (!a || !b || !mismatch7 || n <= 0) return b200r_fail(B200R_EINVAL, "b200r_debug_exact_math: bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = b200r_zero(mismatch7, 7 * sizeof(int), st, "memset mismatch counts")) return rc;
    return b200r_launch("k_debug_exact_math", B200R_K_DEBUG, k_debug_exact_math, (n + 255) / 256, 256, 0, st, a, b, n, mismatch7);
}
