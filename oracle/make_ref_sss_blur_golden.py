"""Golden vectors of the reference's OWN subsurface-scattering blur kernels (TEST INFRASTRUCTURE).

Runs gaussain_blur_x_Kernel / gaussain_blur_y_Kernel (jrender/renderer/utils/gaussian_blur.py:33-164, built by
oracle/build_ref_sss.py into oracle/_ref) once on a GPU, on small generated single-channel maps, and writes
tests/golden/ref_sss_gpu_blur_<h>x<w>.npz.  tests/test_sss_cpu.py holds oracle/sss.py to them.

    python -m oracle.make_ref_sss_blur_golden [OUT_DIR]       (on a GPU machine, after build(); default tests/golden)

The maps cover: zero and <= 1e-6 regions (1e-6 itself, which is below the double 1e-6 once stored as float32), negative
values; modulation values of exactly 0 and 1 and up to 1.4 (a blurred stretch map can pass 1 where a tap extrapolates);
taps that run off both edges (the widest level, v = 300, reaches 3 * sqrt(300) * 1.4 = 73 px); all three variances, both
directions, a modulation map independent of the image and the stretch chain's "blur a map by itself"; a square 64 x 64
map for both kernels, a 48 x 80 map for the x kernel and an 80 x 48 map for the y kernel (whose rows are clamped against
the width, inside an h > w map).
"""
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle import build_ref_sss  # noqa: E402
from oracle import sss as osss  # noqa: E402

OUT_DIR = os.path.join(ROOT, "tests", "golden")
SHAPES = {(64, 64): (0, 1), (48, 80): (1,), (80, 48): (0,)}


def maps(h, w, seed):
    """(image, mod) float32 [h, w] with the special values listed in the module docstring."""
    rng = np.random.default_rng(seed)
    img = rng.uniform(0.05, 1.0, (h, w)).astype(np.float32)
    img[h // 4:h // 2, w // 3:w // 2] = 0                                   # a background hole
    img[:, :3] = np.where(rng.random((h, 3)) < 0.5, 0, img[:, :3])          # holes on the edges
    special = np.float32([1e-6, 5e-7, 1e-7, 0.0, -0.25, 2e-6])
    pick = rng.random((h, w)) < 0.12
    img[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
    mod = rng.uniform(0, 1.4, (h, w)).astype(np.float32)
    mod[rng.random((h, w)) < 0.15] = 0
    mod[rng.random((h, w)) < 0.15] = 1
    return img, mod


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True)
        return q.stdout.strip()
    except OSError:
        return "unknown"


def main(out_dir=OUT_DIR):
    import torch
    L = build_ref_sss.lib()
    assert L is not None, "oracle/_ref/libjrender_ref_sss.so is not built (python -m oracle.build_ref_sss)"
    dev = torch.device("cuda:0")
    for (h, w), dims in SHAPES.items():
        res = {}
        for dim in dims:
            for v in osss.levels():
                g, width = osss.taps(v)
                for variant in ("rand", "self"):
                    img, mod = maps(h, w, seed=h * 1000 + w + 7 * v + dim + (0 if variant == "rand" else 1))
                    if variant == "self":    # the stretch chain: a [0, 1] map blurred with itself as the modulation
                        img = np.clip(np.where(img < 0, 0, img) * np.float32(1.3), 0, 1).astype(np.float32)
                        mod = img
                    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)
                    out = build_ref_sss.blur(L, t(img), t(mod), t(g), width, dim)
                    torch.cuda.synchronize()
                    key = "d%d_v%d_%s" % (dim, v, variant)
                    res[key + "_image"], res[key + "_mod"] = img, mod
                    res[key + "_out"] = out.cpu().numpy()
                    res[key + "_taps"], res[key + "_width"] = g, np.float32(width)
        res["provenance"] = np.frombuffer((
            "jrender/renderer/utils/gaussian_blur.py gaussain_blur_{x,y}_Kernel via oracle/build_ref_sss.py "
            "(nvcc -O3 sm_90a, fmad on), 32x32 blocks; GPU: %s" % card()).encode(), np.uint8)
        os.makedirs(out_dir, exist_ok=True)
        path = os.path.join(out_dir, "ref_sss_gpu_blur_%dx%d.npz" % (h, w))
        np.savez_compressed(path, **res)
        print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT_DIR)
