"""Build oracle/_ref/libjrender_ref.so from the reference's OWN kernel sources (TEST INFRASTRUCTURE).

The reference keeps its CUDA C++ in Python string literals (`jt.code(cuda_header=..., cuda_src=...)`)
and needs Jittor to JIT them; Jittor is not installable here.  This recipe reads the `.py` files
where they lie under /root/reference (never copied into this repo), captures the `cuda_header`
strings through a stub `jittor` module, writes them -- plus a small hand-written launcher that
restates each op's `cuda_src` (memsets, grid/block sizes, argument order) -- to oracle/_ref/*.cu
and compiles them for sm_90a with nvcc defaults (fmad on, as a stock nvcc/Jittor build would).

    python -m oracle.build_ref

Outputs only into oracle/_ref/ (git-ignored, but shipped to the GPU box by gpurun).  Used to
(a) generate golden vectors from the real reference kernels on the GPU (oracle/make_ref_golden.py,
oracle/make_ref_parity_golden.py),
(b) cross-check the product kernels on the GPU, (c) time "the reference kernels on the same GPU".
"""
import os
import subprocess
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE = "/root/reference"
OUT = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT, "libjrender_ref.so")

PREAMBLE = "#include <cstdio>\n#include <cstdint>\ntypedef float float32;\n"


class _Dummy:
    def __init__(self, shape=(1,), dtype="float32"):
        self.shape, self.dtype = list(shape), dtype


def _capture(path, func, nargs, extra=()):
    """Import one reference .py with a stub jittor whose code() returns its kwargs."""
    stub = types.ModuleType("jittor")
    stub.code = lambda *a, **kw: kw
    stub.empty = lambda *a, **kw: _Dummy()
    saved = sys.modules.get("jittor")
    sys.modules["jittor"] = stub
    try:
        src = open(path).read()
        mod = types.ModuleType("ref_capture")
        exec(compile(src, path, "exec"), mod.__dict__)
        kw = getattr(mod, func)(*([_Dummy()] * nargs + list(extra)))
    finally:
        if saved is None:
            sys.modules.pop("jittor", None)
        else:
            sys.modules["jittor"] = saved
    return kw["cuda_header"]


LAUNCH_FWD = r'''
// ---- launcher: restates cuda_src of forward_soft_rasterize (cuda/soft_rasterize.py:459-521)
extern "C" int ref_softras_forward(const float* faces, const float* textures, float* faces_info,
        float* aggrs_info, float* soft_colors, int* faces_id_buffer, int batch_size, int num_faces,
        int texture_size, int image_size, int max_faces_id, float near, float far, float eps,
        float sigma_val, int func_id_dist, float dist_eps, float gamma_val, int func_id_rgb,
        int func_id_alpha, int texture_sample_type, int double_side, cudaStream_t st) {
    const size_t npix = (size_t)image_size * image_size;
    cudaMemsetAsync(faces_info, 0, sizeof(float) * 27 * (size_t)batch_size * num_faces, st);
    cudaMemsetAsync(aggrs_info, 0, sizeof(float) * 2 * npix * batch_size, st);
    cudaMemsetAsync(soft_colors, 0, sizeof(float) * 4 * npix * batch_size, st);
    cudaMemsetAsync(faces_id_buffer, -1, sizeof(int) * (size_t)max_faces_id * npix * batch_size, st);
    const int texture_res = int(sqrt((double)texture_size));
    const int threads = 512;
    const dim3 blocks_1((batch_size * num_faces - 1) / threads + 1);
    forward_soft_rasterize_inv_cuda_kernel<float32><<<blocks_1, threads, 0, st>>>(faces, faces_info, batch_size, num_faces, image_size);
    const dim3 blocks_2((batch_size * image_size * image_size - 1) / threads + 1);
    forward_soft_rasterize_cuda_kernel<float32><<<blocks_2, threads, 0, st>>>(faces, textures, faces_info, aggrs_info,
        soft_colors, faces_id_buffer, batch_size, num_faces, image_size, max_faces_id, texture_size, texture_res,
        near, far, eps, sigma_val, func_id_dist, dist_eps, gamma_val, func_id_rgb, func_id_alpha,
        texture_sample_type, double_side);
    return (int)cudaGetLastError();
}
'''

LAUNCH_BWD = r'''
// ---- launcher: restates cuda_src of backward_soft_rasterize (cuda/soft_rasterize.py:1363-1416)
// faces_id_buffer is [B,H,W,K] here (the host transposes first, soft_rasterize.py:108).
extern "C" int ref_softras_backward(const float* faces, const float* textures, const float* soft_colors,
        const float* faces_info, const float* aggrs_info, const int* faces_id_buffer_bhwk,
        float* grad_soft_colors, float* grad_faces, float* grad_textures, int batch_size, int num_faces,
        int texture_size, int image_size, int max_faces_id, float near, float far, float eps,
        float sigma_val, int func_id_dist, float dist_eps, float gamma_val, int func_id_rgb,
        int func_id_alpha, int texture_sample_type, int double_side, cudaStream_t st) {
    cudaMemsetAsync(grad_faces, 0, sizeof(float) * 9 * (size_t)batch_size * num_faces, st);
    cudaMemsetAsync(grad_textures, 0, sizeof(float) * 3 * (size_t)texture_size * batch_size * num_faces, st);
    const int texture_res = int(sqrt((double)texture_size));
    const int threads = 512;
    const dim3 blocks((batch_size * image_size * image_size - 1) / threads + 1);
    backward_soft_rasterize_cuda_kernel<float32><<<blocks, threads, 0, st>>>(faces, faces_id_buffer_bhwk, textures,
        soft_colors, faces_info, aggrs_info, grad_faces, grad_textures, grad_soft_colors, batch_size, num_faces,
        image_size, max_faces_id, texture_size, texture_res, near, far, eps, sigma_val, func_id_dist, dist_eps,
        gamma_val, func_id_rgb, func_id_alpha, texture_sample_type, (bool)double_side);
    return (int)cudaGetLastError();
}
'''

LAUNCH_C2F = r'''
// ---- launcher: restates cuda_src of forward_soft_rasterize_coarse_to_fine
// (cuda/soft_rasterize_coarse_to_fine.py:765-879), including its cudaMalloc / cudaMemset /
// cudaDeviceSynchronize / cudaFree calls, which are part of the reference op.
extern "C" int ref_softras_forward_c2f(const float* faces, const float* textures, float* faces_info,
        float* aggrs_info, float* soft_colors, int* faces_id_buffer, int batch_size, int num_faces,
        int texture_size, int image_size, int max_faces_id, float near, float far, float eps,
        float sigma_val, int func_id_dist, float dist_eps, float gamma_val, int func_id_rgb,
        int func_id_alpha, int texture_sample_type, int double_side, int bin_size, int max_elems_per_bin) {
    const size_t npix = (size_t)image_size * image_size;
    cudaMemsetAsync(faces_info, 0, sizeof(float) * 27 * (size_t)batch_size * num_faces);
    cudaMemsetAsync(aggrs_info, 0, sizeof(float) * 2 * npix * batch_size);
    cudaMemsetAsync(soft_colors, 0, sizeof(float) * 4 * npix * batch_size);
    cudaMemsetAsync(faces_id_buffer, -1, sizeof(int) * (size_t)max_faces_id * npix * batch_size);
    const int texture_res = int(sqrt((double)texture_size));
    const size_t threads_1 = 512;
    const size_t blocks_1 = ((batch_size * num_faces - 1) / threads_1 + 1);
    float* bboxes; bool* should_skip;
    cudaMalloc((void**)&bboxes, (size_t)batch_size * num_faces * 4 * sizeof(float));
    cudaMalloc((void**)&should_skip, (size_t)batch_size * num_faces * sizeof(bool));
    forward_soft_rasterize_inv_cuda_kernel<float32><<<blocks_1, threads_1>>>(faces, faces_info, batch_size, num_faces, image_size);
    TriangleBoundingBoxKernel<<<128, 256>>>(faces, batch_size * num_faces, 0.01, bboxes, should_skip);
    const int num_bins_edge = 1 + (image_size - 1) / bin_size;
    int* elems_per_bin; int* bin_elems;
    size_t size2 = (size_t)batch_size * num_bins_edge * num_bins_edge * sizeof(int);
    cudaMalloc((void**)&elems_per_bin, size2);
    cudaMemset(elems_per_bin, 0, size2);
    size_t size1 = (size_t)batch_size * num_bins_edge * num_bins_edge * max_elems_per_bin * sizeof(int);
    cudaMalloc((void**)&bin_elems, size1);
    cudaMemset(bin_elems, -1, size1);
    cudaDeviceSynchronize();
    const int chunk_size = 512;
    const int shared_size = num_bins_edge * num_bins_edge * chunk_size / 8;
    RasterizeCoarseCudaKernel<<<64, 512, shared_size>>>(bboxes, should_skip, batch_size, num_faces, image_size,
        bin_size, chunk_size, max_elems_per_bin, elems_per_bin, bin_elems);
    cudaDeviceSynchronize();
    cudaFree(bboxes);
    cudaFree(should_skip);
    const size_t threads_4 = 128;
    const size_t blocks_4 = (((size_t)batch_size * bin_size * bin_size * num_bins_edge * num_bins_edge - 1) / threads_4 + 1);
    forward_soft_rasterize_cuda_kernel<float32><<<blocks_4, threads_4>>>(faces, textures, faces_info, bin_elems,
        elems_per_bin, aggrs_info, soft_colors, faces_id_buffer, num_bins_edge, max_elems_per_bin, bin_size,
        batch_size, num_faces, image_size, max_faces_id, texture_size, texture_res, near, far, eps, sigma_val,
        func_id_dist, dist_eps, gamma_val, func_id_rgb, func_id_alpha, texture_sample_type, double_side);
    cudaError_t err = cudaGetLastError();
    cudaDeviceSynchronize();
    cudaFree(elems_per_bin);
    cudaFree(bin_elems);
    return (int)err;
}
'''


# ---------------------------------------------------------------- NMR (dr_type='n3mr')
# Launchers restating the cuda_src blocks of jrender/renderer/dr/n3mr/cuda/rasterize.py:
# :163-217 (K7: fills, thread mapping by power-of-two face count, lock buffer), :299-339 (K8),
# :614-647 (K9), :696-726 (K10), :790-823 (K11).  K7 takes image_size and the three return flags as
# template arguments (the reference bakes them into the JIT source), so a fixed set is instantiated.
LAUNCH_NMR_K7 = r'''
namespace {
__global__ void ref_fill_f32(float* p, size_t n, float v) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
template <int IS, int RGB, int A, int D>
void launch_k7(const float* faces, float* faces_inv, int32_t* fim, float* wm, float* dm, float* finv, int B, int nf,
               float near_, float far_, int nbits, int32_t* lock) {
    const int threads = 256;
    const dim3 blocks((B * (1 << nbits) - 1) / threads + 1);
    forward_face_index_map_cuda_kernel<float32, IS, RGB, A, D><<<blocks, threads>>>(faces, faces_inv, fim, wm, dm, finv, B, nf, near_, far_, nbits, lock);
}
template <int IS>
int dispatch_flags(int flags, const float* faces, float* faces_inv, int32_t* fim, float* wm, float* dm, float* finv, int B, int nf,
                   float near_, float far_, int nbits, int32_t* lock) {
    switch (flags) {
        case 0: launch_k7<IS, 0, 0, 0>(faces, faces_inv, fim, wm, dm, finv, B, nf, near_, far_, nbits, lock); break;
        case 1: launch_k7<IS, 1, 0, 0>(faces, faces_inv, fim, wm, dm, finv, B, nf, near_, far_, nbits, lock); break;
        case 2: launch_k7<IS, 0, 1, 0>(faces, faces_inv, fim, wm, dm, finv, B, nf, near_, far_, nbits, lock); break;
        case 3: launch_k7<IS, 1, 1, 0>(faces, faces_inv, fim, wm, dm, finv, B, nf, near_, far_, nbits, lock); break;
        case 4: launch_k7<IS, 0, 0, 1>(faces, faces_inv, fim, wm, dm, finv, B, nf, near_, far_, nbits, lock); break;
        case 5: launch_k7<IS, 1, 0, 1>(faces, faces_inv, fim, wm, dm, finv, B, nf, near_, far_, nbits, lock); break;
        case 6: launch_k7<IS, 0, 1, 1>(faces, faces_inv, fim, wm, dm, finv, B, nf, near_, far_, nbits, lock); break;
        default: launch_k7<IS, 1, 1, 1>(faces, faces_inv, fim, wm, dm, finv, B, nf, near_, far_, nbits, lock); break;
    }
    return 0;
}
}  // namespace

// face_inv_map_elems: number of floats in face_inv_map (B*is*is*9 when return_depth, else 1)
extern "C" int ref_nmr_forward_face_index_map(const float* faces, float* faces_inv, int32_t* face_index_map, float* weight_map,
                                              float* depth_map, float* face_inv_map, int32_t* lock, int B, int nf,
                                              int image_size, float near_, float far_, int return_rgb, int return_alpha,
                                              int return_depth, long face_inv_map_elems) {
    const size_t npix = (size_t)B * image_size * image_size;
    cudaMemset(face_index_map, 0xFF, npix * sizeof(int32_t));                      // thrust::fill(-1)
    cudaMemset(weight_map, 0, npix * 3 * sizeof(float));
    ref_fill_f32<<<(unsigned)((npix + 255) / 256), 256>>>(depth_map, npix, far_);    // thrust::fill(far)
    cudaMemset(face_inv_map, 0, (size_t)face_inv_map_elems * sizeof(float));
    cudaMemset(lock, 0, npix * sizeof(int32_t));
    int nbits = 0;
    while ((1 << nbits) < nf) nbits++;   // any n with 2^n >= num_faces maps threads to (batch, face) identically
    const int flags = (return_rgb ? 1 : 0) | (return_alpha ? 2 : 0) | (return_depth ? 4 : 0);
    switch (image_size) {
        case 32: dispatch_flags<32>(flags, faces, faces_inv, face_index_map, weight_map, depth_map, face_inv_map, B, nf, near_, far_, nbits, lock); break;
        case 48: dispatch_flags<48>(flags, faces, faces_inv, face_index_map, weight_map, depth_map, face_inv_map, B, nf, near_, far_, nbits, lock); break;
        case 64: dispatch_flags<64>(flags, faces, faces_inv, face_index_map, weight_map, depth_map, face_inv_map, B, nf, near_, far_, nbits, lock); break;
        case 256: dispatch_flags<256>(flags, faces, faces_inv, face_index_map, weight_map, depth_map, face_inv_map, B, nf, near_, far_, nbits, lock); break;
        case 512: dispatch_flags<512>(flags, faces, faces_inv, face_index_map, weight_map, depth_map, face_inv_map, B, nf, near_, far_, nbits, lock); break;
        case 1024: dispatch_flags<1024>(flags, faces, faces_inv, face_index_map, weight_map, depth_map, face_inv_map, B, nf, near_, far_, nbits, lock); break;
        default: return -1;  // image size not instantiated
    }
    cudaError_t e = cudaDeviceSynchronize();
    return (int)(e != cudaSuccess ? e : cudaGetLastError());
}
'''

LAUNCH_NMR_K8 = r'''
extern "C" int ref_nmr_forward_texture_sampling(const float* faces, const float* textures, const int32_t* face_index_map,
                                                const float* weight_map, const float* depth_map, float* rgb_map,
                                                int32_t* sampling_index_map, float* sampling_weight_map, int B, int nf,
                                                int image_size, int texture_size, float eps) {
    const size_t npix = (size_t)B * image_size * image_size;
    cudaMemset(rgb_map, 0, npix * 3 * sizeof(float));
    cudaMemset(sampling_index_map, 0, npix * 8 * sizeof(int32_t));
    cudaMemset(sampling_weight_map, 0, npix * 8 * sizeof(float));
    const int threads = 512;
    const dim3 blocks((unsigned)((npix - 1) / threads + 1));
    forward_texture_sampling_cuda_kernel<float32><<<blocks, threads>>>(faces, textures, face_index_map, weight_map, depth_map, rgb_map,
                                                                       sampling_index_map, sampling_weight_map, (size_t)B, nf,
                                                                       image_size, texture_size, eps);
    cudaError_t e = cudaDeviceSynchronize();
    return (int)(e != cudaSuccess ? e : cudaGetLastError());
}
'''

LAUNCH_NMR_K9 = r'''
extern "C" int ref_nmr_backward_pixel_map(const float* faces, int32_t* face_index_map, float* rgb_map, float* alpha_map,
                                          float* grad_rgb_map, float* grad_alpha_map, float* grad_faces, int B, int nf,
                                          int image_size, float eps, int return_rgb, int return_alpha) {
    cudaMemset(grad_faces, 0, (size_t)B * nf * 9 * sizeof(float));
    const int threads = 512;
    const dim3 blocks(((size_t)B * nf - 1) / threads + 1);
    backward_pixel_map_cuda_kernel<float32><<<blocks, threads>>>(faces, face_index_map, rgb_map, alpha_map, grad_rgb_map, grad_alpha_map,
                                                                 grad_faces, (size_t)B, (size_t)nf, image_size, eps, return_rgb, return_alpha);
    cudaError_t e = cudaDeviceSynchronize();
    return (int)(e != cudaSuccess ? e : cudaGetLastError());
}
'''

LAUNCH_NMR_K10 = r'''
extern "C" int ref_nmr_backward_textures(const int32_t* face_index_map, float* sampling_weight_map, int32_t* sampling_index_map,
                                         float* grad_rgb_map, float* grad_textures, int B, int nf, int image_size, int texture_size) {
    cudaMemset(grad_textures, 0, (size_t)B * nf * texture_size * texture_size * texture_size * 3 * sizeof(float));
    const int threads = 512;
    const dim3 blocks(((size_t)B * image_size * image_size - 1) / threads + 1);
    backward_textures_cuda_kernel<float32><<<blocks, threads>>>(face_index_map, sampling_weight_map, sampling_index_map, grad_rgb_map,
                                                                grad_textures, (size_t)B, (size_t)nf, image_size, (size_t)texture_size);
    cudaError_t e = cudaDeviceSynchronize();
    return (int)(e != cudaSuccess ? e : cudaGetLastError());
}
'''

LAUNCH_NMR_K11 = r'''
extern "C" int ref_nmr_backward_depth_map(const float* faces, const float* depth_map, const int32_t* face_index_map,
                                          const float* face_inv_map, const float* weight_map, float* grad_depth_map,
                                          float* grad_faces, int B, int nf, int image_size) {
    const int threads = 512;
    const dim3 blocks(((size_t)B * image_size * image_size - 1) / threads + 1);
    backward_depth_map_cuda_kernel<float32><<<blocks, threads>>>(faces, depth_map, face_index_map, face_inv_map, weight_map,
                                                                 grad_depth_map, grad_faces, (size_t)B, (size_t)nf, image_size);
    cudaError_t e = cudaDeviceSynchronize();
    return (int)(e != cudaSuccess ? e : cudaGetLastError());
}
'''


LAUNCH_BAKE = r'''
// ---- launcher: restates cuda_src of _load_textures_for_softras (io/utils/load_textures.py:71-98)
extern "C" int ref_bake_textures_softras(const float* image, const float* faces, const int32_t* is_update, float* textures,
                                         int nf, int texture_res, int image_height, int image_width) {
    const size_t texture_size = (size_t)nf * texture_res * texture_res * 3;   // textures->num
    const int threads = 1024;
    const dim3 blocks((unsigned)((texture_size / 3 - 1) / threads + 1));
    load_textures_cuda_kernel<float32><<<blocks, threads>>>(image, faces, is_update, textures, texture_size, (size_t)texture_res,
                                                            (size_t)image_height, (size_t)image_width);
    cudaError_t e = cudaDeviceSynchronize();
    return (int)(e != cudaSuccess ? e : cudaGetLastError());
}
'''


LAUNCH_BAKE_N3MR = r'''
// ---- launcher: restates cuda_src of _load_textures_for_n3mr (io/utils/load_textures.py:217-246); the wrapping mode and
// the sampling flavour are string-substituted into the header by the reference (:213-214), one translation unit each
extern "C" int ref_bake_textures_n3mr_@W@_@B@(const float* image, float* faces, const int32_t* is_update, float* textures,
                                              int nf, int texture_size, int image_height, int image_width) {
    const int textures_size = nf * texture_size * texture_size * texture_size * 3;   // textures->num
    const int threads = 1024;
    const dim3 blocks((textures_size / 3 - 1) / threads + 1);
    load_textures_cuda_kernel<float32><<<blocks, threads>>>(image, is_update, faces, textures, textures_size, texture_size,
                                                            image_height, image_width);
    cudaError_t e = cudaDeviceSynchronize();
    return (int)(e != cudaSuccess ? e : cudaGetLastError());
}
'''


def generate():
    os.makedirs(OUT, exist_ok=True)
    base = os.path.join(REFERENCE, "jrender/renderer/dr/softras/cuda")
    files = []
    hdr = _capture(os.path.join(base, "soft_rasterize.py"), "forward_soft_rasterize", 6, extra=[64, 1, 100, 1e-3, 1e-5, 2, 9.21, 1e-4, 1, 2, 0, 1])
    files.append(("ref_softras_fwd.cu", PREAMBLE + hdr + LAUNCH_FWD))
    hdr = _capture(os.path.join(base, "soft_rasterize.py"), "backward_soft_rasterize", 9, extra=[64, 1, 100, 1e-3, 1e-5, 2, 9.21, 1e-4, 1, 2, 0, 1])
    files.append(("ref_softras_bwd.cu", PREAMBLE + hdr + LAUNCH_BWD))
    hdr = _capture(os.path.join(base, "soft_rasterize_coarse_to_fine.py"), "forward_soft_rasterize_coarse_to_fine", 6,
                   extra=[64, 1, 100, 1e-3, 1e-5, 2, 9.21, 1e-4, 1, 2, 0, 1, 64, 100])
    files.append(("ref_softras_c2f.cu", PREAMBLE + hdr + LAUNCH_C2F))
    nmr = os.path.join(REFERENCE, "jrender/renderer/dr/n3mr/cuda/rasterize.py")
    hdr = _capture(nmr, "forward_face_index_map", 6, extra=[64, 0.1, 100.0, 1, 1, 1])
    files.append(("ref_nmr_k7.cu", PREAMBLE + hdr + LAUNCH_NMR_K7))
    hdr = _capture(nmr, "forward_texture_sampling", 8, extra=[64, 1e-3])
    files.append(("ref_nmr_k8.cu", PREAMBLE + hdr + LAUNCH_NMR_K8))
    hdr = _capture(nmr, "backward_pixel_map", 7, extra=[64, 1e-3, 1, 1])
    files.append(("ref_nmr_k9.cu", PREAMBLE + hdr + LAUNCH_NMR_K9))
    hdr = _capture(nmr, "backward_textures", 5, extra=[100])
    files.append(("ref_nmr_k10.cu", PREAMBLE + hdr + LAUNCH_NMR_K10))
    hdr = _capture(nmr, "backward_depth_map", 7, extra=[64])
    files.append(("ref_nmr_k11.cu", PREAMBLE + hdr + LAUNCH_NMR_K11))
    hdr = _capture(os.path.join(REFERENCE, "jrender/io/utils/load_textures.py"), "_load_textures_for_softras", 4)
    files.append(("ref_bake.cu", PREAMBLE + hdr + LAUNCH_BAKE))
    for wrap in range(4):
        for bil in range(2):
            hdr = _capture(os.path.join(REFERENCE, "jrender/io/utils/load_textures.py"), "_load_textures_for_n3mr", 4, extra=[wrap, bil])
            files.append(("ref_bake_n3mr_%d_%d.cu" % (wrap, bil),
                          PREAMBLE + hdr + LAUNCH_BAKE_N3MR.replace("@W@", str(wrap)).replace("@B@", str(bil))))
    paths = []
    for name, text in files:
        p = os.path.join(OUT, name)
        if not os.path.exists(p) or open(p).read() != text:
            open(p, "w").write(text)
        paths.append(p)
    return paths


def build(force=False, verbose=False):
    if not os.path.isdir(REFERENCE):
        raise RuntimeError("%s not present (GPU box?): use the prebuilt oracle/_ref" % REFERENCE)
    paths = generate()
    if not force and os.path.exists(LIB) and all(os.path.getmtime(p) <= os.path.getmtime(LIB) for p in paths + [os.path.abspath(__file__)]):
        return LIB
    cmd = ["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
           "-w", "-Xcompiler", "-fPIC", "-shared", "-o", LIB] + paths
    if verbose:
        print(" ".join(cmd))
    subprocess.run(cmd, check=True)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
