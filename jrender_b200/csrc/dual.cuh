// dual.cuh -- forward-mode automatic differentiation in registers: a value and N partial derivatives per intermediate.
// Used where a per-element expression of the reference (a few dozen flops over <= 12 inputs) needs its exact gradient
// in the same launch: no hand-derived formula to get wrong, no saved intermediates.
#pragma once
#include <cuda_runtime.h>

namespace b200r {

template <int N>
struct Dual {
    float v;
    float d[N];
};

template <int N>
__device__ __forceinline__ Dual<N> dconst(float v) {
    Dual<N> r;
    r.v = v;
#pragma unroll
    for (int i = 0; i < N; i++) r.d[i] = 0.f;
    return r;
}
template <int N>
__device__ __forceinline__ Dual<N> dvar(float v, int i) {
    Dual<N> r = dconst<N>(v);
    r.d[i] = 1.f;
    return r;
}
template <int N>
__device__ __forceinline__ Dual<N> operator+(const Dual<N>& a, const Dual<N>& b) {
    Dual<N> r;
    r.v = a.v + b.v;
#pragma unroll
    for (int i = 0; i < N; i++) r.d[i] = a.d[i] + b.d[i];
    return r;
}
template <int N>
__device__ __forceinline__ Dual<N> operator-(const Dual<N>& a, const Dual<N>& b) {
    Dual<N> r;
    r.v = a.v - b.v;
#pragma unroll
    for (int i = 0; i < N; i++) r.d[i] = a.d[i] - b.d[i];
    return r;
}
template <int N>
__device__ __forceinline__ Dual<N> operator*(const Dual<N>& a, const Dual<N>& b) {
    Dual<N> r;
    r.v = a.v * b.v;
#pragma unroll
    for (int i = 0; i < N; i++) r.d[i] = a.d[i] * b.v + a.v * b.d[i];
    return r;
}
template <int N>
__device__ __forceinline__ Dual<N> operator/(const Dual<N>& a, const Dual<N>& b) {
    Dual<N> r;
    r.v = a.v / b.v;
    const float ib = 1.f / b.v;
#pragma unroll
    for (int i = 0; i < N; i++) r.d[i] = (a.d[i] - r.v * b.d[i]) * ib;
    return r;
}
template <int N>
__device__ __forceinline__ Dual<N> operator+(const Dual<N>& a, float s) { Dual<N> r = a; r.v = a.v + s; return r; }
template <int N>
__device__ __forceinline__ Dual<N> operator+(float s, const Dual<N>& a) { return a + s; }
template <int N>
__device__ __forceinline__ Dual<N> operator*(const Dual<N>& a, float s) {
    Dual<N> r;
    r.v = a.v * s;
#pragma unroll
    for (int i = 0; i < N; i++) r.d[i] = a.d[i] * s;
    return r;
}
template <int N>
__device__ __forceinline__ Dual<N> operator*(float s, const Dual<N>& a) { return a * s; }
template <int N>
__device__ __forceinline__ Dual<N> operator-(float s, const Dual<N>& a) {
    Dual<N> r;
    r.v = s - a.v;
#pragma unroll
    for (int i = 0; i < N; i++) r.d[i] = -a.d[i];
    return r;
}
template <int N>
__device__ __forceinline__ Dual<N> operator-(const Dual<N>& a, float s) { Dual<N> r = a; r.v = a.v - s; return r; }
template <int N>
__device__ __forceinline__ Dual<N> operator/(const Dual<N>& a, float s) { return a * (1.f / s); }

// plain-float overloads so that one templated expression serves value-only and value+gradient evaluation
__device__ __forceinline__ float dsqrt(float a) { return sqrtf(a); }
template <int N>
__device__ __forceinline__ Dual<N> dsqrt(const Dual<N>& a) {
    Dual<N> r;
    r.v = sqrtf(a.v);
    const float h = 0.5f / r.v;
#pragma unroll
    for (int i = 0; i < N; i++) r.d[i] = a.d[i] * h;
    return r;
}
// max(a, lo) as torch.relu: the derivative passes where a > lo, not at the kink (relu'(0) = 0).  NaN propagates as
// torch does: the value stays NaN and its derivative is 0 (the mask `a > lo` is false).
__device__ __forceinline__ float dmax(float a, float lo) { return a <= lo ? lo : a; }
template <int N>
__device__ __forceinline__ Dual<N> dmax(const Dual<N>& a, float lo) {
    if (a.v > lo) return a;
    return dconst<N>(a.v <= lo ? lo : a.v);
}
// max(a, lo) as torch.clamp(min=lo) / clamp_min (and so F.normalize's eps): the derivative passes where a >= lo,
// at equality included.  NaN as in dmax: value NaN, derivative 0.
__device__ __forceinline__ float dclamp_min(float a, float lo) { return a <= lo ? lo : a; }
template <int N>
__device__ __forceinline__ Dual<N> dclamp_min(const Dual<N>& a, float lo) {
    if (a.v >= lo) return a;
    return dconst<N>(a.v <= lo ? lo : a.v);
}
__device__ __forceinline__ float dvalue(float a) { return a; }
template <int N>
__device__ __forceinline__ float dvalue(const Dual<N>& a) { return a.v; }

}  // namespace b200r
