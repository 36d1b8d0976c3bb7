"""Build oracle/_ref/libjrender_ref_voxel.so from the reference's OWN voxelization kernels (TEST INFRASTRUCTURE).

Same recipe as oracle/build_ref_atlas.py: the four `cuda_header` strings of jrender/renderer/utils/cuda/voxelization.py
(read in place in the reference checkout, build_ref.REFERENCE; never copied into this repo) are captured through
build_ref's stub `jittor`, a hand-written launcher restating their `cuda_src` is appended, and the result is compiled for
sm_90a with nvcc defaults (fmad on, as a stock nvcc / Jittor build would).

The headers' `#if __CUDA_ARCH__ < 600` guard is also true in nvcc's host pass, where its atomicAdd(double*, double)
clashes with CUDA's own declaration; the generated file tests `defined(__CUDA_ARCH__)` as well.

    python -m oracle.build_ref_voxel

Outputs only into oracle/_ref/ (git-ignored; the library runs wherever the tree is copied to a GPU machine).  Used by
oracle/make_ref_voxel_golden.py.
"""
import os
import subprocess
import sys

from . import build_ref

LIB = os.path.join(build_ref.OUT, "libjrender_ref_voxel.so")

LAUNCH_VOXEL = r'''
// ---- launchers: restate the cuda_src of voxelize_sub1..4 (512 threads, one launch each).  Synchronous; the caller
// runs the host loop of voxelization.py:24-57 around them.
static int ref_sync() {
    cudaError_t e = cudaDeviceSynchronize();
    return (int)(e != cudaSuccess ? e : cudaGetLastError());
}
extern "C" int ref_voxelize_sub1(const float* faces, int* voxels, int batch_size, int num_faces, int voxel_size) {
    voxelize_sub1_kernel<float32><<<(batch_size * voxel_size * voxel_size - 1) / 512 + 1, 512>>>(faces, voxels, batch_size,
                                                                                             num_faces, voxel_size);
    return ref_sync();
}
extern "C" int ref_voxelize_sub2(const float* faces, int* voxels, int batch_size, int num_faces, int voxel_size) {
    voxelize_sub2_kernel<float32><<<(batch_size * num_faces - 1) / 512 + 1, 512>>>(faces, voxels, batch_size, num_faces,
                                                                                  voxel_size);
    return ref_sync();
}
extern "C" int ref_voxelize_sub3(int* voxels, int* visible, int batch_size, int voxel_size) {
    voxelize_sub3_kernel<float32><<<(batch_size * voxel_size * voxel_size * voxel_size - 1) / 512 + 1, 512>>>(
        voxels, visible, batch_size, voxel_size);
    return ref_sync();
}
extern "C" int ref_voxelize_sub4(int* voxels, int* visible, int batch_size, int voxel_size) {
    voxelize_sub4_kernel<float32><<<(batch_size * voxel_size * voxel_size * voxel_size - 1) / 512 + 1, 512>>>(
        voxels, visible, batch_size, voxel_size);
    return ref_sync();
}
'''

GUARD_FROM = "#if  __CUDA_ARCH__ < 600"
GUARD_TO = "#if defined(__CUDA_ARCH__) && __CUDA_ARCH__ < 600"


def generate():
    os.makedirs(build_ref.OUT, exist_ok=True)
    src = os.path.join(build_ref.REFERENCE, "jrender/renderer/utils/cuda/voxelization.py")
    hdrs = [build_ref._capture(src, "voxelize_sub1", 2), build_ref._capture(src, "voxelize_sub2", 2),
            build_ref._capture(src, "voxelize_sub3", 3), build_ref._capture(src, "voxelize_sub4", 3)]
    for h in hdrs:
        if GUARD_FROM not in h:
            raise RuntimeError("voxelization.py: the atomicAdd guard `%s` is not where expected" % GUARD_FROM)
    text = build_ref.PREAMBLE + "".join(h.replace(GUARD_FROM, GUARD_TO) for h in hdrs) + LAUNCH_VOXEL
    p = os.path.join(build_ref.OUT, "ref_voxelization.cu")
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
