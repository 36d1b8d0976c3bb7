"""Time voxelization() on the GPU: the surface and fill kernels separately (CUDA events, after warm-up) and, when
oracle/_ref/libjrender_ref_voxel.so exists, the reference kernels with their own host loop and its synchronisations.

    python tools/bench_voxel.py [--reps N]

Meshes: the 39 200-face UV sphere at radius 0.45 and the spot cow, both through Mesh.voxelize's mapping; vs in
{32, 64, 128, 256}, B in {1, 4}.  Prints one JSON line per case with the card's name and power limit read in this run.
"""
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import voxelize as ov  # noqa: E402

# the module, not the function jrender_b200.voxelization that the package exports under the same name
jv = importlib.import_module("jrender_b200.voxelization")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def timed(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / reps


def main():
    assert torch.cuda.is_available(), "bench_voxel needs a CUDA device"
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 20
    name, power = card()
    dev = torch.device("cuda:0")
    ref = None
    from oracle import build_ref_voxel
    if os.path.exists(build_ref_voxel.LIB):
        from oracle import make_ref_voxel_golden as mrg
        ref = mrg.load_lib()
    meshes = {"sphere39200": ov.sphere_faces(39200, radius=0.45), "spot": ov.spot_faces()}
    for mesh, fv in meshes.items():
        for vs in (32, 64, 128, 256):
            for B in (1, 4):
                faces = torch.from_numpy(np.repeat(ov.mesh_voxelize_faces(fv, vs) * np.float32(vs), B, axis=0)).to(dev)
                surf = jv.voxelize_surface(faces, vs)
                grid = surf.clone()
                jv.voxelize_fill(grid)                                            # warm-up
                t_surface = timed(lambda: jv.voxelize_surface(faces, vs), reps)
                t_fill = timed(lambda: jv.voxelize_fill(grid.copy_(surf)), reps) - timed(lambda: grid.copy_(surf), reps)
                jv.voxelize_fill(grid.copy_(surf))                                # the timed copies left grid unfilled
                row = dict(mesh=mesh, nf=int(faces.shape[1]), vs=vs, B=B, surface_ms=round(t_surface, 4),
                           fill_ms=round(t_fill, 4), total_ms=round(t_surface + t_fill, 4), filled=int(grid.sum()),
                           gpu=name, power_limit=power)
                if ref is not None and vs <= 128:
                    fc = faces.cpu().numpy()
                    mrg.run_reference(ref, fc, vs)                                # warm-up
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    _, final = mrg.run_reference(ref, fc, vs)
                    torch.cuda.synchronize()
                    row["reference_ms"] = round(1e3 * (time.perf_counter() - t0), 3)
                    row["reference_equal"] = bool(np.array_equal(final, grid.cpu().numpy()))
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
