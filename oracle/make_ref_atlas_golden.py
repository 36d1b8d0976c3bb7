"""Golden vectors of the reference's OWN texture-atlas kernel, run on a GPU (TEST INFRASTRUCTURE).

    python -m oracle.make_ref_atlas_golden [--out DIR]     # writes DIR/ref_atlas_gpu_*.npz (default tests/golden)

Needs a CUDA device and oracle/_ref/libjrender_ref_atlas.so (python -m oracle.build_ref_atlas, which needs the
reference checkout; the built library can be copied with the tree to a GPU machine).  The kernel is create_texture_image_cuda_kernel (jrender/io/utils/create_texture_image.py),
fed the integer-row tile layout (oracle/texture_atlas.py:atlas_layout) and an image of ones, as save_obj.py:11 starts
from.  Each file holds the inputs, the reference's image, and the GPU and nvcc flags it was made with; the generator
prints how many pixels differ from the numpy oracle (the reference build contracts a*b+c).
"""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import build_ref_atlas, texture_atlas as oat  # noqa: E402

# (num_faces, R_in, R_out): one face, non-square face counts, R_in 1 / 4 / 5, R_out 2 / 4 / 16
CASES = ((1, 4, 16), (7, 5, 4), (23, 1, 2), (40, 4, 16), (13, 5, 16))


def main():
    import torch
    out_dir = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else os.path.join(ROOT, "tests", "golden")
    os.makedirs(out_dir, exist_ok=True)
    L = C.CDLL(build_ref_atlas.LIB)
    L.ref_create_texture_image.restype = C.c_int
    L.ref_create_texture_image.argtypes = [C.c_void_p] * 3 + [C.c_long] * 4
    dev = torch.device("cuda:0")
    for nf, R, R_out in CASES:
        rng = np.random.default_rng(100 * nf + 10 * R + R_out)
        tex = rng.random((nf, R * R, 3), dtype=np.float32)
        tri, tw, th = oat.atlas_layout(nf, R_out)
        H, W = th * R_out, tw * R_out
        t_tri, t_tex = torch.from_numpy(tri).to(dev), torch.from_numpy(tex).to(dev)
        img = torch.ones((H, W, 3), dtype=torch.float32, device=dev)
        rc = L.ref_create_texture_image(C.c_void_p(t_tri.data_ptr()), C.c_void_p(t_tex.data_ptr()), C.c_void_p(img.data_ptr()),
                                        nf, R * R, H, W)
        assert rc == 0, rc
        ref = img.cpu().numpy()
        cpu = oat.texture_atlas_softras(tri, tex, R_out, tw, H, W)
        name = "ref_atlas_gpu_nf%d_R%d_out%d" % (nf, R, R_out)
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), tile_vertices=tri, textures=tex, image=ref, texture_res_out=R_out,
                            tile_width=tw, provenance=json.dumps(dict(
                                gpu=torch.cuda.get_device_name(0), nvcc="12.9 -O3 -gencode arch=compute_90a,code=sm_90a (fmad default on)",
                                source="jrender/io/utils/create_texture_image.py:3-104 via oracle/build_ref_atlas.py")))
        diff = np.abs(ref - cpu).max(axis=-1) > 0
        print(json.dumps(dict(name=name, pixels=int(diff.size), pixels_differing_from_oracle=int(diff.sum()))), flush=True)


if __name__ == "__main__":
    main()
