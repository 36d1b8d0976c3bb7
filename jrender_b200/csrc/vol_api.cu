// vol_api.cu -- NeRF volume rendering (jrender_vol/integrator/{integrator,sample}.py, rayMarching/rayMarching.py).
//
//   b200r_vol_composite_forward   <-  integrator(), integrator.py:18-39 (raw2alpha, the exclusive cumprod, the four sums)
//   b200r_vol_composite_backward  <-  autograd of the same ops, to raw only
//   b200r_vol_resample            <-  sample_pdf(), sample.py:28-57, and the fine stage of render_rays (rayMarching.py:67-71:
//                                     mids, sample_pdf of weights[..., 1:-1], argsort of the concat)
//
// Thread mapping: one warp per ray.  A ray's samples are walked in tiles of 32, lane l taking sample 32 k + l of tile k;
// the exclusive transmittance product is a shuffle scan within the tile times the product carried from the tiles before,
// and the sums are per-lane partials over the tiles reduced by an xor butterfly at the end.  No atomics, no shared
// memory in the compositing kernels.  At the training shape (1024 rays) this still gives 1024 warps -- 8 per SM -- where a
// thread per ray would occupy 8 of 132 SMs; at render chunks the grid is simply larger.  The resampler keeps one ray's
// cdf, bins and the (S + Ni)-value sort buffer in shared memory per warp and sorts with a warp bitonic network.
//
// Arithmetic is the reference's float32 expressions unfused (-fmad=false), only the order of the products and sums within a
// ray is the scan / butterfly order above; oracle/volume.py restates that order in numpy.
#include <math.h>

#include "../../include/b200raster.h"
#include "api_util.cuh"

namespace {

constexpr int kVolMaxSamples = B200R_VOL_MAX_SAMPLES;
constexpr int kCompositeWarps = 8;   // rays per 256-thread block
constexpr int kResampleWarps = 4;    // rays per 128-thread block: <= 4 x 12 KB of shared memory at the bound
constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ float warp_sum(float v) {
    for (int o = 16; o > 0; o >>= 1) v = v + __shfl_xor_sync(kFull, v, o);
    return v;
}

// Hillis-Steele inclusive scans over the 32 lanes
__device__ __forceinline__ float warp_incl_prod(float v, int lane) {
    for (int d = 1; d < 32; d <<= 1) {
        const float o = __shfl_up_sync(kFull, v, d);
        if (lane >= d) v = v * o;
    }
    return v;
}
__device__ __forceinline__ float warp_incl_sum(float v, int lane) {
    for (int d = 1; d < 32; d <<= 1) {
        const float o = __shfl_up_sync(kFull, v, d);
        if (lane >= d) v = v + o;
    }
    return v;
}

struct VolSample {
    float z, x, e, dist, alpha, t;   // x = sigma + noise, e = exp(-relu(x) * dist), t = (1 - alpha) + 1e-10
};

// integrator.py:18-28 for sample s of a ray (s < S): dists (:20-22), alpha = raw2alpha(raw[..., 3] + noise, dists)
__device__ __forceinline__ VolSample vol_sample(const float* __restrict__ zr, const float* __restrict__ rawr,
                                                const float* __restrict__ noiser, int s, int S, int C, float norm) {
    VolSample q;
    q.z = __ldg(zr + s);
    q.dist = (s + 1 < S ? __ldg(zr + s + 1) - q.z : 1e10f) * norm;
    q.x = __ldg(rawr + (size_t)s * C + 3);
    if (noiser) q.x = q.x + __ldg(noiser + s);
    const float r = q.x > 0.f ? q.x : 0.f;
    q.e = expf(-r * q.dist);
    q.alpha = 1.f - q.e;
    q.t = (1.f - q.alpha) + 1e-10f;
    return q;
}

__device__ __forceinline__ float vol_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ float ray_norm(const float* __restrict__ d) {
    const float dx = __ldg(d), dy = __ldg(d + 1), dz = __ldg(d + 2);
    return sqrtf(dx * dx + dy * dy + dz * dz);
}

// jt.maximum(1e-10, depth / acc) read as std::max(1e-10, q): the constant unless 1e-10 < q, so a NaN q gives 1e-10
__device__ __forceinline__ bool disp_takes_q(float q) { return 1e-10f < q; }

__global__ void __launch_bounds__(32 * kCompositeWarps)
k_vol_composite_fwd(const float* __restrict__ raw, const float* __restrict__ z_vals, const float* __restrict__ rays_d,
                    const float* __restrict__ noise, float* __restrict__ rgb_map, float* __restrict__ disp_map,
                    float* __restrict__ acc_map, float* __restrict__ weights, float* __restrict__ depth_map, int N, int S,
                    int C, int white_bkgd) {
    const int lane = threadIdx.x & 31;
    const long ray = (long)blockIdx.x * kCompositeWarps + (threadIdx.x >> 5);
    if (ray >= N) return;
    const float* zr = z_vals + ray * S;
    const float* rawr = raw + ray * S * C;
    const float* noiser = noise ? noise + ray * S : nullptr;
    const float norm = ray_norm(rays_d + ray * 3);
    float carry = 1.f, pr = 0.f, pg = 0.f, pb = 0.f, pacc = 0.f, pdep = 0.f;
    for (int base = 0; base < S; base += 32) {
        const int s = base + lane;
        VolSample q{};
        q.t = 1.f;
        if (s < S) q = vol_sample(zr, rawr, noiser, s, S, C, norm);
        const float incl = warp_incl_prod(q.t, lane);
        const float excl = __shfl_up_sync(kFull, incl, 1);
        const float T = carry * (lane == 0 ? 1.f : excl);
        carry = carry * __shfl_sync(kFull, incl, 31);
        if (s < S) {
            const float w = q.alpha * T;
            weights[ray * S + s] = w;
            const float* c = rawr + (size_t)s * C;
            pr = pr + w * vol_sigmoid(__ldg(c));
            pg = pg + w * vol_sigmoid(__ldg(c + 1));
            pb = pb + w * vol_sigmoid(__ldg(c + 2));
            pacc = pacc + w;
            pdep = pdep + w * q.z;
        }
    }
    pr = warp_sum(pr), pg = warp_sum(pg), pb = warp_sum(pb), pacc = warp_sum(pacc), pdep = warp_sum(pdep);
    if (lane == 0) {
        const float q = pdep / pacc;
        disp_map[ray] = 1.f / (disp_takes_q(q) ? q : 1e-10f);
        acc_map[ray] = pacc;
        depth_map[ray] = pdep;
        if (white_bkgd) {
            const float bg = 1.f - pacc;
            pr = pr + bg, pg = pg + bg, pb = pb + bg;
        }
        rgb_map[ray * 3] = pr, rgb_map[ray * 3 + 1] = pg, rgb_map[ray * 3 + 2] = pb;
    }
}

// Backward.  With t_k = (1 - a_k) + 1e-10, T_i = prod_{k<i} t_k, w_i = a_i T_i and G_i = dL/dw_i (every output is
// linear in the w_i, apart from disp through depth / acc, whose derivative is a per-ray constant):
//   dL/da_i = G_i T_i - sum_{j>i} G_j w_j / t_i = T_i (G_i - R_i),  R_i = sum_{j>i} G_j a_j prod_{i<k<j} t_k,
// with R from the suffix recurrence R_{i-1} = t_i R_i + G_i a_i -- no division by t_i, so an opaque sample (t_i = 1e-10)
// leaves the gradients of the samples in front of it finite.  Pass 1 walks the tiles front to back for the transmittance
// at each tile's start (tile k's in lane k: S <= 1024 is at most 32 tiles); pass 2 walks them back to front with the
// recurrence as a scan of affine maps x -> t x + G a.
__global__ void __launch_bounds__(32 * kCompositeWarps)
k_vol_composite_bwd(const float* __restrict__ raw, const float* __restrict__ z_vals, const float* __restrict__ rays_d,
                    const float* __restrict__ noise, const float* __restrict__ acc_map, const float* __restrict__ depth_map,
                    const float* __restrict__ g_rgb, const float* __restrict__ g_disp, const float* __restrict__ g_acc,
                    const float* __restrict__ g_weights, const float* __restrict__ g_depth, float* __restrict__ grad_raw,
                    int N, int S, int C, int white_bkgd) {
    const int lane = threadIdx.x & 31;
    const long ray = (long)blockIdx.x * kCompositeWarps + (threadIdx.x >> 5);
    if (ray >= N) return;
    const float* zr = z_vals + ray * S;
    const float* rawr = raw + ray * S * C;
    const float* noiser = noise ? noise + ray * S : nullptr;
    float* gr = grad_raw + ray * S * C;
    const float norm = ray_norm(rays_d + ray * 3);

    // dL/dw_i = g0 + gz z_i + g_weights_i + sum_c g_rgb_c sigmoid(raw_ic)
    const float c0 = g_rgb ? __ldg(g_rgb + ray * 3) : 0.f, c1 = g_rgb ? __ldg(g_rgb + ray * 3 + 1) : 0.f,
                c2 = g_rgb ? __ldg(g_rgb + ray * 3 + 2) : 0.f;
    float g0 = g_acc ? __ldg(g_acc + ray) : 0.f;
    if (white_bkgd) g0 = g0 - (c0 + c1 + c2);
    float gz = g_depth ? __ldg(g_depth + ray) : 0.f;
    if (g_disp) {
        const float acc = __ldg(acc_map + ray), dep = __ldg(depth_map + ray), q = dep / acc;
        if (disp_takes_q(q)) {   // disp = 1 / q: d/dq = -1 / q^2; q = depth / acc
            const float gq = -__ldg(g_disp + ray) / (q * q);
            gz = gz + gq / acc;
            g0 = g0 - gq * dep / (acc * acc);
        }
    }

    float tstart = 1.f;   // lane k: transmittance in front of tile k
    {
        float carry = 1.f;
        for (int base = 0, k = 0; base < S; base += 32, k++) {
            if (lane == k) tstart = carry;
            const int s = base + lane;
            const float t = s < S ? vol_sample(zr, rawr, noiser, s, S, C, norm).t : 1.f;
            carry = carry * __shfl_sync(kFull, warp_incl_prod(t, lane), 31);
        }
    }
    float carryR = 0.f;   // R-recurrence value entering the tile from behind (Q of the next tile's first sample)
    for (int k = (S - 1) / 32; k >= 0; k--) {
        const int s = 32 * k + lane;
        const bool valid = s < S;
        VolSample q{};
        q.t = 1.f;
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, G = 0.f;
        if (valid) {
            q = vol_sample(zr, rawr, noiser, s, S, C, norm);
            const float* c = rawr + (size_t)s * C;
            s0 = vol_sigmoid(__ldg(c)), s1 = vol_sigmoid(__ldg(c + 1)), s2 = vol_sigmoid(__ldg(c + 2));
            G = g0 + gz * q.z + (c0 * s0 + c1 * s1 + c2 * s2);
            if (g_weights) G = G + __ldg(g_weights + ray * S + s);
        }
        const float incl = warp_incl_prod(q.t, lane);
        const float excl = __shfl_up_sync(kFull, incl, 1);
        const float T = __shfl_sync(kFull, tstart, k) * (lane == 0 ? 1.f : excl);
        // suffix scan of the maps x -> m x + b (composition towards the tile's end)
        float m = q.t, b = valid ? G * q.alpha : 0.f;
        for (int d = 1; d < 32; d <<= 1) {
            const float m2 = __shfl_down_sync(kFull, m, d), b2 = __shfl_down_sync(kFull, b, d);
            if (lane + d < 32) {
                b = m * b2 + b;
                m = m * m2;
            }
        }
        const float Q = m * carryR + b;
        const float Qn = __shfl_down_sync(kFull, Q, 1);
        const float R = lane == 31 ? carryR : Qn;
        carryR = __shfl_sync(kFull, Q, 0);
        if (valid) {
            const float dLda = T * (G - R);
            const float w = q.alpha * T;
            float* o = gr + (size_t)s * C;
            o[0] = c0 * w * (s0 * (1.f - s0));
            o[1] = c1 * w * (s1 * (1.f - s1));
            o[2] = c2 * w * (s2 * (1.f - s2));
            o[3] = q.x > 0.f ? dLda * q.e * q.dist : 0.f;   // alpha = 1 - exp(-relu(x) dist)
            for (int ch = 4; ch < C; ch++) o[ch] = 0.f;
        }
    }
}

// jt.linspace(0., 1., steps=n)[k] as jittor forms it: k * (end - start) / (steps - 1) + start
__device__ __forceinline__ float linspace01(int k, int n) { return n > 1 ? (float)k * 1.f / (float)(n - 1) + 0.f : 0.f; }

// One warp per ray.  Shared memory per warp: cdf[nb], bins[nb], then (fine stage) the sort buffer of P = pow2 >= S + Ni.
//   fine stage (z_vals != NULL): bins = mids of z_vals (nb = S - 1), pdf weights = weights[ray, 1 : S - 1] of [N, S];
//   sample_pdf (z_vals == NULL): bins [N, nb], weights [N, nb - 1].
__global__ void __launch_bounds__(32 * kResampleWarps)
k_vol_resample(const float* __restrict__ z_vals, const float* __restrict__ bins_in, const float* __restrict__ weights,
               const float* __restrict__ u_in, float* __restrict__ z_samples, float* __restrict__ z_vals_fine, int N,
               int S, int nb, int Ni, int P) {
    extern __shared__ float smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long ray = (long)blockIdx.x * kResampleWarps + warp;
    float* cdf = smem + (size_t)warp * (2 * nb + P);
    float* bins = cdf + nb;
    float* buf = bins + nb;
    if (ray >= N) return;
    const int nw = nb - 1;                     // pdf weights
    const float* wr = z_vals ? weights + ray * S + 1 : weights + ray * nw;
    if (z_vals) {
        const float* zr = z_vals + ray * S;
        for (int k = lane; k < S; k += 32) buf[k] = __ldg(zr + k);
        for (int k = S + Ni + lane; k < P; k += 32) buf[k] = NAN;   // sorts behind every value, NaN included
        __syncwarp();
        for (int k = lane; k < nb; k += 32) bins[k] = .5f * (buf[k + 1] + buf[k]);   // rayMarching.py:67
    } else {
        for (int k = lane; k < nb; k += 32) bins[k] = __ldg(bins_in + ray * nb + k);
    }
    // weights + 1e-5; pdf = w / sum(w); cdf = [0, cumsum(pdf)]   (sample.py:30-33)
    float psum = 0.f;
    for (int base = 0; base < nw; base += 32)
        if (base + lane < nw) psum = psum + (__ldg(wr + base + lane) + 1e-5f);
    const float wsum = warp_sum(psum);
    float carry = 0.f;
    if (lane == 0) cdf[0] = 0.f;
    for (int base = 0; base < nw; base += 32) {
        const int k = base + lane;
        const float pdf = k < nw ? (__ldg(wr + k) + 1e-5f) / wsum : 0.f;
        const float incl = carry + warp_incl_sum(pdf, lane);
        if (k < nw) cdf[k + 1] = incl;
        carry = __shfl_sync(kFull, incl, 31);
    }
    __syncwarp();
    for (int j = lane; j < Ni; j += 32) {
        const float u = u_in ? __ldg(u_in + ray * Ni + j) : linspace01(j, Ni);
        int inds = 0;                                           // searchsorted(cdf, u, right=True): #{cdf <= u}
        for (int k = 0; k < nb; k++) inds += cdf[k] <= u;
        const int below = max(0, inds - 1), above = min(nb - 1, inds);
        const float cdf0 = cdf[below], cdf1 = cdf[above], bin0 = bins[below], bin1 = bins[above];
        float denom = cdf1 - cdf0;
        if (denom < 1e-5f) denom = 1.f;
        const float t = (u - cdf0) / denom;
        const float sample = bin0 + t * (bin1 - bin0);
        z_samples[ray * Ni + j] = sample;
        if (z_vals) buf[S + j] = sample;
    }
    if (!z_vals) return;
    __syncwarp();
    // bitonic sort of buf[0, P) ascending; NaN sorts last, as torch.sort puts it.  The padding past S + Ni is NaN too, so
    // the first S + Ni are torch.sort's: the real values in order, then as many NaNs as the merge held
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = lane; i < P / 2; i += 32) {
                const int lo = 2 * i - (i & (stride - 1));
                const int hi = lo + stride;
                const bool up = (lo & size) == 0;
                const float a = buf[lo], b = buf[hi];
                const bool gt = !(a <= b) && b == b;   // a > b, or a NaN and b not
                if (gt == up) buf[lo] = b, buf[hi] = a;
            }
            __syncwarp();
        }
    }
    float* out = z_vals_fine + ray * (S + Ni);
    for (int k = lane; k < S + Ni; k += 32) out[k] = buf[k];
}

int check_rays(const char* what, int N, int S) {
    if (N < 0 || S < 1) return b200r_fail(B200R_EINVAL, "%s: num_rays %d < 0 or num_samples %d < 1", what, N, S);
    if (S > kVolMaxSamples)
        return b200r_fail(B200R_EUNSUPPORTED, "%s: %d samples per ray > %d, the bound of this kernel", what, S, kVolMaxSamples);
    return 0;
}

unsigned composite_blocks(int N) { return (unsigned)((N + kCompositeWarps - 1) / kCompositeWarps); }

}  // namespace

extern "C" int b200r_vol_composite_forward(const float* raw, const float* z_vals, const float* rays_d, const float* noise,
                                           float* rgb_map, float* disp_map, float* acc_map, float* weights, float* depth_map,
                                           int num_rays, int num_samples, int raw_channels, int white_bkgd, void* stream) {
    if (int rc = check_rays("b200r_vol_composite_forward", num_rays, num_samples)) return rc;
    if (raw_channels < 4) return b200r_fail(B200R_EINVAL, "b200r_vol_composite_forward: raw has %d < 4 channels", raw_channels);
    if (num_rays == 0) return 0;
    if (!raw || !z_vals || !rays_d || !rgb_map || !disp_map || !acc_map || !weights || !depth_map)
        return b200r_fail(B200R_EINVAL, "b200r_vol_composite_forward: NULL pointer argument");
    return b200r_launch("k_vol_composite_fwd", B200R_K_VOL_COMPOSITE_FWD, k_vol_composite_fwd, composite_blocks(num_rays),
                        32 * kCompositeWarps, 0, (cudaStream_t)stream, raw, z_vals, rays_d, noise, rgb_map, disp_map, acc_map,
                        weights, depth_map, num_rays, num_samples, raw_channels, white_bkgd);
}

extern "C" int b200r_vol_composite_backward(const float* raw, const float* z_vals, const float* rays_d, const float* noise,
                                            const float* acc_map, const float* depth_map, const float* grad_rgb_map,
                                            const float* grad_disp_map, const float* grad_acc_map, const float* grad_weights,
                                            const float* grad_depth_map, float* grad_raw, int num_rays, int num_samples,
                                            int raw_channels, int white_bkgd, void* stream) {
    if (int rc = check_rays("b200r_vol_composite_backward", num_rays, num_samples)) return rc;
    if (raw_channels < 4) return b200r_fail(B200R_EINVAL, "b200r_vol_composite_backward: raw has %d < 4 channels", raw_channels);
    if (num_rays == 0) return 0;
    if (!raw || !z_vals || !rays_d || !grad_raw)
        return b200r_fail(B200R_EINVAL, "b200r_vol_composite_backward: NULL pointer argument");
    if (grad_disp_map && (!acc_map || !depth_map))
        return b200r_fail(B200R_EINVAL, "b200r_vol_composite_backward: grad_disp_map needs acc_map and depth_map");
    return b200r_launch("k_vol_composite_bwd", B200R_K_VOL_COMPOSITE_BWD, k_vol_composite_bwd, composite_blocks(num_rays),
                        32 * kCompositeWarps, 0, (cudaStream_t)stream, raw, z_vals, rays_d, noise, acc_map, depth_map,
                        grad_rgb_map, grad_disp_map, grad_acc_map, grad_weights, grad_depth_map, grad_raw, num_rays,
                        num_samples, raw_channels, white_bkgd);
}

extern "C" int b200r_vol_resample(const float* z_vals, const float* bins, const float* weights, const float* u,
                                  float* z_samples, float* z_vals_fine, int num_rays, int num_bins, int num_importance,
                                  void* stream) {
    const char* what = "b200r_vol_resample";
    if (num_rays < 0 || num_importance < 1)
        return b200r_fail(B200R_EINVAL, "%s: num_rays %d < 0 or num_importance %d < 1", what, num_rays, num_importance);
    if (num_bins + num_importance > kVolMaxSamples)
        return b200r_fail(B200R_EUNSUPPORTED, "%s: %d + %d samples per ray > %d, the bound of this kernel", what, num_bins,
                          num_importance, kVolMaxSamples);
    if (num_rays == 0) return 0;   // (empty tensors may pass NULL for every pointer)
    if ((z_vals == nullptr) == (bins == nullptr) || (z_vals == nullptr) != (z_vals_fine == nullptr))
        return b200r_fail(B200R_EINVAL, "%s: give z_vals and z_vals_fine (fine stage) or bins (sample_pdf), not both", what);
    // fine stage: num_bins = S coarse samples, nb = S - 1 mids; sample_pdf: nb = num_bins
    const int nb = z_vals ? num_bins - 1 : num_bins;
    if (nb < 1)
        return b200r_fail(B200R_EINVAL, "%s: %s %d leaves no bins", what, z_vals ? "num_samples" : "num_bins", num_bins);
    if (!weights || !z_samples) return b200r_fail(B200R_EINVAL, "%s: NULL pointer argument", what);
    int P = 0;
    if (z_vals) {
        P = 1;
        while (P < num_bins + num_importance) P <<= 1;
    }
    const size_t smem = (size_t)kResampleWarps * (2 * nb + P) * sizeof(float);
    return b200r_launch("k_vol_resample", B200R_K_VOL_RESAMPLE, k_vol_resample,
                        (unsigned)((num_rays + kResampleWarps - 1) / kResampleWarps), 32 * kResampleWarps, smem,
                        (cudaStream_t)stream, z_vals, bins, weights, u, z_samples, z_vals_fine, num_rays,
                        z_vals ? num_bins : 0, nb, num_importance, P);
}
