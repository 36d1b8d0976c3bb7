"""Build oracle/_ref/libjrender_ref_screen.so from the reference's OWN render2 screen-space kernels (TEST
INFRASTRUCTURE): SSAO_cuda, SSDO_cuda and FXAA_cuda (jrender/render2/utils/cuda/{SSAO,SSDO,FXAA}_cuda.py).

Same recipe as oracle/build_ref.py: each op's `cuda_header` is captured through build_ref._capture (read in place in the
reference checkout, build_ref.REFERENCE; never copied into this repo), launchers restating its `cuda_src` are appended,
and the result is compiled for sm_90a with nvcc defaults (fmad on, as a stock nvcc / Jittor build would).

One textual patch, and only this one: the headers' `Vector3&` / `Vector2&` / `float2&` / `float3&` operators, `cross`
and `tex_sample` return references to temporaries, which nvcc 12.9 rejects ("initial value of reference to non-const
must be an lvalue").  PATCH turns those return types into by-value returns, which is what the code means; every
expression and every call is left as written.  Each header goes into its own namespace (the three define the same
classes and the same `_curand_init`), after the system headers it includes, so its own #includes are no-ops.

Launchers, all on the stream `st` unless stated:
  ref_ssao / ref_ssdo            the whole op as cuda_src states it: cudaMalloc of one curandStateXORWOW_t per pixel,
                                 _curand_init, cudaDeviceSynchronize, the kernel, cudaFree (legacy default stream, as
                                 the op runs); the per-call cost the product removes
  ref_screen_curand_init         _curand_init alone, into caller-owned states (ref_screen_state_bytes() per pixel)
  ref_ssao_kernel / _ssdo_kernel the kernel alone on such states (which it advances: re-initialise for the same draws)
  ref_fxaa                       FXAA_cuda; `texture` must be padded with zeros: at the last row the kernel reads the
                                 row past the image, and at the last pixel one pixel further (both with weight 0);
                                 fxaa() below pads two rows
  ref_screen_draws               the uniform draws a pixel's stream gives: curand_init(1, i, 0), then n
                                 curand_uniform, the order SSAO_cuda / SSDO_cuda take them in (x, y, z per sample)

    python -m oracle.build_ref_screen

Outputs only into oracle/_ref/ (git-ignored).  Used by oracle/make_ref_screen_golden.py, tests/test_screen_space_gpu.py
and tools/time_screen_space.py.
"""
import os
import re
import subprocess
import sys
import types
from unittest import mock

from . import build_ref

LIB = os.path.join(build_ref.OUT, "libjrender_ref_screen.so")
SRC = "jrender/render2/utils/cuda"
OPS = (("SSAO_cuda.py", "SSAO_cuda", 6, "ref_ssao_ns"), ("SSDO_cuda.py", "SSDO_cuda", 7, "ref_ssdo_ns"),
       ("FXAA_cuda.py", "FXAA_cuda", 1, "ref_fxaa_ns"))
PATCH = (re.compile(r"\b(Vector3|Vector2|float2|float3)&(\s+)(operator\s*[-+*]=?|cross|tex_sample)\s*\("), r"\1\2\3(")

PRE = build_ref.PREAMBLE + "#include <cuda.h>\n#include <cuda_runtime.h>\n#include <curand_kernel.h>\n#include <math.h>\n"

LAUNCH = r'''
// ---- launchers: restate cuda_src of SSAO_cuda.py:175-212, SSDO_cuda.py:208-247 and FXAA_cuda.py:251-262 (1024
// threads per block, one thread per pixel)
namespace {
__global__ void ref_draws_kernel(float* out, size_t is, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= is * is) return;
    curandStateXORWOW_t s;
    curand_init(1, i, 0, &s);
    for (int k = 0; k < n; k++) out[(size_t)i * n + k] = curand_uniform(&s);
}
inline dim3 blocks_for(long is) { return dim3((unsigned)((is * is - 1) / 1024 + 1)); }
}  // namespace

extern "C" size_t ref_screen_state_bytes(void) { return sizeof(curandStateXORWOW_t); }

extern "C" int ref_screen_curand_init(void* states, long is, cudaStream_t st) {
    ref_ssao_ns::_curand_init<<<blocks_for(is), 1024, 0, st>>>((curandStateXORWOW_t*)states, (size_t)is);
    return (int)cudaGetLastError();
}

extern "C" int ref_screen_draws(float* out, long is, int n, cudaStream_t st) {
    ref_draws_kernel<<<blocks_for(is), 1024, 0, st>>>(out, (size_t)is, n);
    return (int)cudaGetLastError();
}

extern "C" int ref_ssao_kernel(float* occlusion, const float* depth, const float* normal_buffer, const int* face_ind_buffer,
                               void* states, long is, int sample_num, float sample_range_r, float width, cudaStream_t st) {
    ref_ssao_ns::SSAO_cuda<float32><<<blocks_for(is), 1024, 0, st>>>(occlusion, depth, normal_buffer, face_ind_buffer,
        (curandStateXORWOW_t*)states, (size_t)is, sample_num, sample_range_r, width);
    return (int)cudaGetLastError();
}

extern "C" int ref_ssdo_kernel(float* image, const float* color, const float* depth, const float* normal_buffer,
                               const int* face_ind_buffer, void* states, long is, int sample_num, float sample_range_r,
                               float width, cudaStream_t st) {
    ref_ssdo_ns::SSDO_cuda<float32><<<blocks_for(is), 1024, 0, st>>>(image, color, depth, normal_buffer, face_ind_buffer,
        (curandStateXORWOW_t*)states, (size_t)is, sample_num, sample_range_r, width);
    return (int)cudaGetLastError();
}

extern "C" int ref_ssao(float* occlusion, const float* depth, const float* normal_buffer, const int* face_ind_buffer,
                        long is, int sample_num, float sample_range_r, float width) {
    curandStateXORWOW_t* states;
    cudaMalloc(&states, (size_t)is * is * sizeof(curandStateXORWOW_t));
    ref_ssao_ns::_curand_init<<<blocks_for(is), 1024>>>(states, (size_t)is);
    cudaDeviceSynchronize();
    ref_ssao_ns::SSAO_cuda<float32><<<blocks_for(is), 1024>>>(occlusion, depth, normal_buffer, face_ind_buffer, states,
        (size_t)is, sample_num, sample_range_r, width);
    cudaFree(states);
    return (int)cudaGetLastError();
}

extern "C" int ref_ssdo(float* image, const float* color, const float* depth, const float* normal_buffer,
                        const int* face_ind_buffer, long is, int sample_num, float sample_range_r, float width) {
    curandStateXORWOW_t* states;
    cudaMalloc(&states, (size_t)is * is * sizeof(curandStateXORWOW_t));
    ref_ssdo_ns::_curand_init<<<blocks_for(is), 1024>>>(states, (size_t)is);
    cudaDeviceSynchronize();
    ref_ssdo_ns::SSDO_cuda<float32><<<blocks_for(is), 1024>>>(image, color, depth, normal_buffer, face_ind_buffer, states,
        (size_t)is, sample_num, sample_range_r, width);
    cudaFree(states);
    return (int)cudaGetLastError();
}

extern "C" int ref_fxaa(float* image, const float* texture_padded, long is, cudaStream_t st) {
    ref_fxaa_ns::FXAA_cuda<float32><<<blocks_for(is), 1024, 0, st>>>(image, texture_padded, (int)is);
    return (int)cudaGetLastError();
}
'''


class _Var(build_ref._Dummy):
    """A stand-in argument for the render2 ops, which convert their inputs before jt.code."""
    def float32(self):
        return self

    def int32(self):
        return self


class _Types:
    """build_ref._capture's `types`, whose stub jittor also has the zeros_like / ones_like the render2 ops call."""
    @staticmethod
    def ModuleType(name):
        m = types.ModuleType(name)
        m.zeros_like = m.ones_like = lambda x: x
        return m


def generate():
    os.makedirs(build_ref.OUT, exist_ok=True)
    parts = [PRE]
    with mock.patch.object(build_ref, "types", _Types):
        for fname, func, nargs, ns in OPS:
            hdr = build_ref._capture(os.path.join(build_ref.REFERENCE, SRC, fname), func, 0, extra=[_Var()] * nargs)
            hdr, n = PATCH[0].subn(PATCH[1], hdr)
            assert n > 0, "%s: nothing to patch" % fname
            parts.append("namespace %s {\n%s\n}  // namespace %s\n" % (ns, hdr, ns))
    text = "".join(parts) + LAUNCH
    p = os.path.join(build_ref.OUT, "ref_screen.cu")
    if not os.path.exists(p) or open(p).read() != text:
        open(p, "w").write(text)
    return p


def build(force=False, verbose=False):
    if not os.path.isdir(build_ref.REFERENCE):
        raise RuntimeError("reference checkout %s not present: use a prebuilt oracle/_ref" % build_ref.REFERENCE)
    p = generate()
    if not force and os.path.exists(LIB) and max(os.path.getmtime(p), os.path.getmtime(os.path.abspath(__file__))) <= os.path.getmtime(LIB):
        return LIB
    cmd = ["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
           "-w", "-Xcompiler", "-fPIC", "-shared", "-o", LIB, p]
    if verbose:
        print(" ".join(cmd))
    subprocess.run(cmd, check=True)
    return LIB


def lib():
    """The built library with its launchers bound, or None when it has not been built."""
    import ctypes as C
    if not os.path.exists(LIB):
        return None
    L = C.CDLL(LIB)
    P, I, F, Lg = C.c_void_p, C.c_int, C.c_float, C.c_long
    sigs = {"ref_screen_state_bytes": (C.c_size_t, []),
            "ref_screen_curand_init": (I, [P, Lg, P]),
            "ref_screen_draws": (I, [P, Lg, I, P]),
            "ref_ssao_kernel": (I, [P] * 5 + [Lg, I, F, F, P]),
            "ref_ssdo_kernel": (I, [P] * 6 + [Lg, I, F, F, P]),
            "ref_ssao": (I, [P] * 4 + [Lg, I, F, F]),
            "ref_ssdo": (I, [P] * 5 + [Lg, I, F, F]),
            "ref_fxaa": (I, [P, P, Lg, P])}
    for name, (res, args) in sigs.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    return L


def _stream(t):
    import torch
    return torch.cuda.current_stream(t.device).cuda_stream


def _padded(is_):
    """Pixels the reference's grid covers: its kernels test `i >= np` only after writing pixel i (and SSDO reads colour i
    there), so every buffer indexed by i gets this many pixels and the result is the first is * is."""
    return ((is_ * is_ - 1) // 1024 + 1) * 1024


def ssao(L, depth, face_ind_buffer, normal_buffer, width, sample_num, sample_range_r):
    """The reference SSAO_cuda op, allocation, init and sync included, on CUDA tensors -> occlusion [is, is]."""
    import torch
    d = depth.float().contiguous()
    n = d.shape[0]
    out = torch.zeros(_padded(n), dtype=torch.float32, device=d.device)
    rc = L.ref_ssao(out.data_ptr(), d.data_ptr(), normal_buffer.float().contiguous().data_ptr(),
                    face_ind_buffer.int().contiguous().data_ptr(), n, int(sample_num), float(sample_range_r), float(width))
    assert rc == 0, "reference SSAO launch failed: %d" % rc
    return out[:n * n].view(n, n)


def ssdo(L, color, depth, face_ind_buffer, normal_buffer, width, sample_num, sample_range_r):
    """The reference SSDO_cuda op on CUDA tensors -> image [is, is, 3]."""
    import torch
    n = color.shape[0]
    c = torch.zeros((_padded(n), 3), dtype=torch.float32, device=color.device)
    c[:n * n] = color.float().reshape(n * n, 3)
    out = torch.zeros_like(c)
    rc = L.ref_ssdo(out.data_ptr(), c.data_ptr(), depth.float().contiguous().data_ptr(),
                    normal_buffer.float().contiguous().data_ptr(), face_ind_buffer.int().contiguous().data_ptr(),
                    n, int(sample_num), float(sample_range_r), float(width))
    assert rc == 0, "reference SSDO launch failed: %d" % rc
    return out[:n * n].view(n, n, 3)


def fxaa(L, texture):
    """The reference FXAA_cuda op on a CUDA [is, is, 3] tensor, run on a copy padded with zero rows: tex_sample reads
    row `is` at the image's last row, and one pixel further at its last pixel, (is, is) -> image [is, is, 3]."""
    import torch
    t = texture.float()
    n = t.shape[0]
    padded = torch.zeros((n + 2, n, 3), dtype=torch.float32, device=t.device)
    padded[:n] = t
    out = torch.ones_like(t)
    rc = L.ref_fxaa(out.data_ptr(), padded.data_ptr(), n, _stream(t))
    assert rc == 0, "reference FXAA launch failed: %d" % rc
    return out


def draws(L, is_, n, device):
    """[is * is, n] uniform draws of each pixel's curand_init(1, i, 0) stream, in the order the kernels take them."""
    import torch
    out = torch.empty((is_ * is_, n), dtype=torch.float32, device=device)
    rc = L.ref_screen_draws(out.data_ptr(), is_, n, torch.cuda.current_stream(device).cuda_stream)
    assert rc == 0, "reference draws launch failed: %d" % rc
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
