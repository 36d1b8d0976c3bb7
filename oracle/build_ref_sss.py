"""Build oracle/_ref/libjrender_ref_sss.so from the reference's OWN subsurface-scattering blur kernels (TEST
INFRASTRUCTURE).

Same recipe as oracle/build_ref.py: the `cuda_header` of _blur_for_SSS in jrender/renderer/utils/gaussian_blur.py (read
in place in the reference checkout, build_ref.REFERENCE; never copied into this repo) is captured through build_ref's
stub `jittor`, two hand-written launchers restating its `cuda_src` (:167-203: 32 x 32 blocks, the y kernel for dim 0, the
x kernel for dim 1) are appended, and the result is compiled for sm_90a with nvcc defaults (fmad on, as a stock nvcc /
Jittor build would).

    python -m oracle.build_ref_sss

Outputs only into oracle/_ref/ (git-ignored; the library runs wherever the tree is copied to a GPU machine).  Used by
oracle/make_ref_sss_blur_golden.py, tests/test_sss_gpu.py and tools/time_sss.py.
"""
import os
import subprocess
import sys

from . import build_ref

LIB = os.path.join(build_ref.OUT, "libjrender_ref_sss.so")

LAUNCH_SSS = r'''
// ---- launchers: restate cuda_src of _blur_for_SSS (renderer/utils/gaussian_blur.py:167-203).  image [h, w, d],
// modulate_map [h, w], Gauss [tap_num] are device pointers; GaussWidth is the float the reference formats into its source.
// Asynchronous on `st`, like the op inside a Jittor graph.
extern "C" int ref_sss_blur_x(const float* image, const float* modulate_map, const float* gauss, float* image_blur,
                              int tap_num, float gauss_width, long h, long w, long d, cudaStream_t st) {
    const dim3 block(32, 32);
    const dim3 grid((unsigned)((w - 1) / block.x + 1), (unsigned)((h - 1) / block.y + 1));
    gaussain_blur_x_Kernel<float32><<<grid, block, 0, st>>>(image, modulate_map, gauss, image_blur, tap_num, gauss_width,
                                                            (size_t)h, (size_t)w, (size_t)d);
    return (int)cudaGetLastError();
}
extern "C" int ref_sss_blur_y(const float* image, const float* modulate_map, const float* gauss, float* image_blur,
                              int tap_num, float gauss_width, long h, long w, long d, cudaStream_t st) {
    const dim3 block(32, 32);
    const dim3 grid((unsigned)((w - 1) / block.x + 1), (unsigned)((h - 1) / block.y + 1));
    gaussain_blur_y_Kernel<float32><<<grid, block, 0, st>>>(image, modulate_map, gauss, image_blur, tap_num, gauss_width,
                                                            (size_t)h, (size_t)w, (size_t)d);
    return (int)cudaGetLastError();
}
'''


def generate():
    os.makedirs(build_ref.OUT, exist_ok=True)
    hdr = build_ref._capture(os.path.join(build_ref.REFERENCE, "jrender/renderer/utils/gaussian_blur.py"), "_blur_for_SSS", 7)
    text = build_ref.PREAMBLE + hdr + LAUNCH_SSS
    p = os.path.join(build_ref.OUT, "ref_sss_blur.cu")
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
    """The built library with ref_sss_blur_x / _y bound, or None when it has not been built."""
    import ctypes as C
    if not os.path.exists(LIB):
        return None
    L = C.CDLL(LIB)
    for name in ("ref_sss_blur_x", "ref_sss_blur_y"):
        fn = getattr(L, name)
        fn.restype = C.c_int
        fn.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_float, C.c_long, C.c_long, C.c_long, C.c_void_p]
    return L


def blur(L, image, mod, gauss, width, dim, stream=None):
    """One reference _blur_for_SSS on CUDA tensors: image [h, w] (d = 1) or [h, w, d], mod [h, w], gauss [tap_num]
    (device, float32); dim 1 = x kernel, 0 = y kernel.  Returns a new [h, w] tensor on the current stream."""
    import torch
    img = image.contiguous()
    h, w = img.shape[0], img.shape[1]
    d = img.shape[2] if img.dim() == 3 else 1
    out = torch.empty((h, w), dtype=torch.float32, device=img.device)   # the kernel writes every pixel
    st = torch.cuda.current_stream(img.device).cuda_stream if stream is None else stream
    fn = L.ref_sss_blur_x if dim == 1 else L.ref_sss_blur_y
    rc = fn(img.data_ptr(), mod.contiguous().data_ptr(), gauss.data_ptr(), out.data_ptr(), int(gauss.numel()), float(width),
            h, w, d, st)
    assert rc == 0, "reference blur launch failed: %d" % rc
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
