"""Build oracle/_ref/libjrender_ref_atlas.so from the reference's OWN texture-atlas kernel (TEST INFRASTRUCTURE).

Same recipe as oracle/build_ref.py, for the one export kernel: the `cuda_header` of
jrender/io/utils/create_texture_image.py (read in place in the reference checkout, build_ref.REFERENCE; never copied
into this repo) is
captured through build_ref's stub `jittor`, a hand-written launcher restating its `cuda_src` (:76-104) is appended, and
the result is compiled for sm_90a with nvcc defaults (fmad on, as a stock nvcc / Jittor build would).

    python -m oracle.build_ref_atlas

Outputs only into oracle/_ref/ (git-ignored; the library runs wherever the tree is copied to a GPU machine).  Used by
oracle/make_ref_atlas_golden.py to pin oracle/texture_atlas.py and the product kernel to the reference kernel.
"""
import os
import subprocess
import sys

from . import build_ref

LIB = os.path.join(build_ref.OUT, "libjrender_ref_atlas.so")

LAUNCH_ATLAS = r'''
// ---- launcher: restates cuda_src of create_texture_image (io/utils/create_texture_image.py:76-104).  The caller fills
// image with ones first (save_obj.py:11).  `image->size` is the image's size in BYTES, so the reference launches four
// times the threads it needs; the surplus ones find fn >= num_faces and return.
extern "C" int ref_create_texture_image(const float* faces, const float* textures, float* image, long num_faces,
                                        long textures_shape1, long image_shape0, long image_shape1) {
    const auto texture_res_in = int(sqrt((double)textures_shape1));
    const auto tile_width = int(sqrt((double)(num_faces - 1))) + 1;
    const auto texture_res_out = image_shape1 / tile_width;
    const int threads = 1024;
    const int image_size = (int)(image_shape0 * image_shape1 * 3 * sizeof(float));   // image->size
    const dim3 blocks((image_size / 3 - 1) / threads + 1);
    create_texture_image_cuda_kernel<float32><<<blocks, threads>>>(faces, textures, image, image_size, num_faces,
                                                                   texture_res_in, texture_res_out, tile_width, (float32)1e-05);
    cudaError_t e = cudaDeviceSynchronize();
    return (int)(e != cudaSuccess ? e : cudaGetLastError());
}
'''


def generate():
    os.makedirs(build_ref.OUT, exist_ok=True)
    hdr = build_ref._capture(os.path.join(build_ref.REFERENCE, "jrender/io/utils/create_texture_image.py"), "create_texture_image", 3,
                             extra=[1e-5])
    text = build_ref.PREAMBLE + hdr + LAUNCH_ATLAS
    p = os.path.join(build_ref.OUT, "ref_texture_atlas.cu")
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


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
