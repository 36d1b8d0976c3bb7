"""Golden vectors of the reference's OWN voxelization kernels, run on a GPU (TEST INFRASTRUCTURE).

    python -m oracle.make_ref_voxel_golden [--out DIR]     # writes DIR/ref_voxel_gpu_*.npz (default tests/golden)

Needs a CUDA device and oracle/_ref/libjrender_ref_voxel.so (python -m oracle.build_ref_voxel, which needs the reference
checkout; the built library can be copied with the tree to a GPU machine).  The host side restates
jrender/renderer/utils/voxelization.py:5-57: sub1 on the three permuted copies of the faces, transposed back, sub2, the
OR, then sub3 and sub4 relaunched until visible.sum() stops changing, and 1 - visible.  Each file holds the faces in
voxel units, the OR'ed surface grid, the final grid bit-packed (np.packbits), and provenance; the generator prints how
many voxels differ from the numpy oracle (the reference build contracts a*b+c).
"""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import build_ref_voxel, voxelize as ov  # noqa: E402


def run_reference(L, faces, vs):
    """voxelization.py:41-57 after the scaling, on the reference kernels: returns (surface, final) int32 grids."""
    import torch
    dev = torch.device("cuda:0")
    B, nf = faces.shape[:2]
    grids = []
    for axis, perm in enumerate(ov.PERMS):                                   # voxelize_sub1, :5-16
        f = torch.from_numpy(np.ascontiguousarray(faces[:, :, :, list(perm)])).to(dev)
        vox = torch.zeros((B, vs, vs, vs), dtype=torch.int32, device=dev)
        assert L.ref_voxelize_sub1(C.c_void_p(f.data_ptr()), C.c_void_p(vox.data_ptr()), B, nf, vs) == 0
        grids.append(vox.permute(*((0, 3, 2, 1), (0, 1, 3, 2), (0, 1, 2, 3))[axis]))
    f = torch.from_numpy(np.ascontiguousarray(faces)).to(dev)
    vox = torch.zeros((B, vs, vs, vs), dtype=torch.int32, device=dev)       # voxelize_sub2, :18-22
    assert L.ref_voxelize_sub2(C.c_void_p(f.data_ptr()), C.c_void_p(vox.data_ptr()), B, nf, vs) == 0
    grids.append(vox)
    surf = ((grids[0] + grids[1] + grids[2] + grids[3]) > 0).int().contiguous()
    voxels = surf.clone()
    visible = torch.zeros_like(voxels)                                        # voxelize_sub3, :24-38
    assert L.ref_voxelize_sub3(C.c_void_p(voxels.data_ptr()), C.c_void_p(visible.data_ptr()), B, vs) == 0
    total = int(visible.sum())
    while True:
        assert L.ref_voxelize_sub4(C.c_void_p(voxels.data_ptr()), C.c_void_p(visible.data_ptr()), B, vs) == 0
        now = int(visible.sum())
        if now == total:
            break
        total = now
    return surf.cpu().numpy(), (1 - visible).cpu().numpy()


def load_lib():
    L = C.CDLL(build_ref_voxel.LIB)
    for name in ("ref_voxelize_sub1", "ref_voxelize_sub2"):
        getattr(L, name).restype = C.c_int
        getattr(L, name).argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    for name in ("ref_voxelize_sub3", "ref_voxelize_sub4"):
        getattr(L, name).restype = C.c_int
        getattr(L, name).argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    return L


def main():
    import torch
    out_dir = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else os.path.join(ROOT, "tests", "golden")
    os.makedirs(out_dir, exist_ok=True)
    L = load_lib()
    for name, faces, vs in ov.golden_cases():
        surf, final = run_reference(L, faces, vs)
        np.savez_compressed(os.path.join(out_dir, "ref_voxel_gpu_%s.npz" % name), faces=faces, voxel_size=vs, surface=surf,
                            final_packed=np.packbits(final.astype(np.uint8).ravel()), provenance=json.dumps(dict(
                                gpu=torch.cuda.get_device_name(0),
                                nvcc="12.9 -O3 -gencode arch=compute_90a,code=sm_90a (fmad default on)",
                                source="jrender/renderer/utils/cuda/voxelization.py via oracle/build_ref_voxel.py, "
                                       "host loop of jrender/renderer/utils/voxelization.py:5-57")))
        cpu = ov.surface(faces, vs)
        print(json.dumps(dict(name=name, voxels=int(surf.size), surface_voxels=int(surf.sum()),
                              surface_differing_from_oracle=int((surf != cpu).sum()), filled=int(final.sum()))), flush=True)


if __name__ == "__main__":
    main()
