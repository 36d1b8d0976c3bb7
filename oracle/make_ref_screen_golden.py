"""Golden vectors of the reference's render2 screen-space kernels (SSAO_cuda, SSDO_cuda, FXAA_cuda), run from
oracle/_ref/libjrender_ref_screen.so (oracle/build_ref_screen.py) on a GPU, on small G-buffers of spot standing on a
ground plane (examples/render_ssao.py's gbuffers) and on FXAA inputs with hard edges, noise and non-finite pixels.

    python -m oracle.make_ref_screen_golden [OUT_DIR]       (on a GPU machine, after build(); default tests/golden)

Writes tests/golden/ref_screen_<name>.npz, each with the inputs, the reference outputs and, for SSAO / SSDO, every
pixel's uniform draws (curand_init(1, i, 0), three per sample) so that oracle/screen_space.py can replay them on the
CPU.  tests/test_screen_space_cpu.py holds the numpy restatement to them; tests/test_screen_space_gpu.py holds the
kernels to them where oracle/_ref is absent.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import build_ref_screen  # noqa: E402

# (name, image size, samples, sample radius)
SCENES = (("spot32", 32, 64, 0.3), ("spot48", 48, 24, 0.15), ("spot64", 64, 16, 0.15))   # draws stay under 0.8 MB


def spot_scene(size):
    from examples.render_ssao import gbuffers, ground_plane, shade
    from examples.render_gbuffers import load_spot
    v, f = ground_plane(*load_spot(torch.device("cuda")))
    depth, face_ind, normal, width = gbuffers(v, f, size)
    return depth, face_ind, normal, width, shade(face_ind, normal)


def fxaa_inputs(rng, color):
    """[name -> [is, is, 3]] FXAA inputs: a hard-edged render, uniform noise, a constant, and noise with NaN / +-inf."""
    n = color.shape[0]
    noise = rng.uniform(0, 1, (n, n, 3)).astype(np.float32)
    bad = noise.copy()
    idx = rng.choice(n * n * 3, size=40, replace=False)
    bad.reshape(-1)[idx[:14]] = np.nan
    bad.reshape(-1)[idx[14:27]] = np.inf
    bad.reshape(-1)[idx[27:]] = -np.inf
    return {"render": color, "noise": noise, "const": np.full((n, n, 3), 0.37, np.float32), "nonfinite": bad}


def main(out_dir):
    L = build_ref_screen.lib()
    assert L is not None, "oracle/_ref/libjrender_ref_screen.so is not built (python -m oracle.build_ref_screen)"
    rng = np.random.default_rng(7)
    for name, size, samples, radius in SCENES:
        depth, face_ind, normal, width, color = spot_scene(size)
        draws = build_ref_screen.draws(L, size, 3 * samples, depth.device)
        ao = build_ref_screen.ssao(L, depth, face_ind, normal, width, samples, radius)
        do = build_ref_screen.ssdo(L, color, depth, face_ind, normal, width, samples, radius)
        data = dict(depth=depth, face_ind=face_ind, normal=normal, color=color, draws=draws, ssao=ao, ssdo=do)
        data = {k: v.cpu().numpy() for k, v in data.items()}
        data.update(width=np.float32(width), sample_num=np.int32(samples), sample_range_r=np.float32(radius))
        for k, img in fxaa_inputs(rng, data["color"]).items():
            data["fxaa_in_" + k] = img
            data["fxaa_out_" + k] = build_ref_screen.fxaa(L, torch.from_numpy(img).cuda()).cpu().numpy()
        data["source"] = np.array("jrender/render2/utils/cuda/{SSAO,SSDO,FXAA}_cuda.py via oracle/build_ref_screen.py, "
                                  "on %s" % torch.cuda.get_device_name())
        path = os.path.join(out_dir, "ref_screen_%s.npz" % name)
        np.savez_compressed(path, **data)
        print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
