"""Time one iteration of the demo 5 (metallic) and demo 6 (roughness) fitting loops on the spot cow at 256^2 -- render,
loss, backward, Adam step -- with the fused surface lighting (Lighting.fused = True) against the op-by-op PyTorch mirror
(False).  The two arms alternate in this one process after a warm-up; each window is timed with CUDA events.

    python tools/time_material_fit.py [--iters 20] [--rounds 5]

Prints one JSON line per (demo, arm): median and min ms per iteration over the rounds, the library's launch count per
iteration (b200r_launch_count: kernels of this project, not PyTorch's), and the card's name and power limit read in
this run.  The cow comes from tests/golden (spot_triangulated.obj.xz + spot_texture.png).
"""
import json
import lzma
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from examples import demo5_optim_metallic_textures as demo5  # noqa: E402
from examples import demo6_optim_roughness_textures as demo6  # noqa: E402
from jrender_b200 import _lib  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def unpack_spot(d):
    golden = os.path.join(ROOT, "tests", "golden")
    with lzma.open(os.path.join(golden, "spot_triangulated.obj.xz"), "rb") as f, \
            open(os.path.join(d, "spot_triangulated.obj"), "wb") as o:
        o.write(f.read())
    with open(os.path.join(d, "spot_triangulated.mtl"), "w") as o:
        o.write("newmtl material_1\nmap_Kd spot_texture.png\n")
    shutil.copyfile(os.path.join(golden, "spot_texture.png"), os.path.join(d, "spot_texture.png"))
    return os.path.join(d, "spot_triangulated.obj")


def main():
    assert torch.cuda.is_available(), "time_material_fit needs a CUDA device"
    iters = int(sys.argv[sys.argv.index("--iters") + 1]) if "--iters" in sys.argv else 20
    rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 5
    name, power = card()
    dev = torch.device("cuda:0")
    L = _lib.lib()
    with tempfile.TemporaryDirectory() as d:
        obj = unpack_spot(d)
        for demo, mod, param in (("demo5", demo5, "metallic_textures"), ("demo6", demo6, "roughness_textures")):
            model = mod.Model(obj, None, dev)
            p = getattr(model, param)
            opt = torch.optim.Adam([p], lr=0.1, betas=(0.5, 0.999))
            p0 = p.detach().clone()

            def step():
                opt.zero_grad(set_to_none=True)
                loss = model()
                loss.backward()
                opt.step()

            arms = {True: [], False: []}
            launches = {}
            for fused in (True, False):   # warm-up, and the library launches of one iteration
                model.renderer.lighting.fused = fused
                for _ in range(3):
                    step()
                torch.cuda.synchronize()
                n0 = L.b200r_launch_count()
                step()
                torch.cuda.synchronize()
                launches[fused] = L.b200r_launch_count() - n0
            for _ in range(rounds):
                for fused in (True, False):
                    model.renderer.lighting.fused = fused
                    with torch.no_grad():   # every window fits from the same start
                        p.copy_(p0)
                    opt.state.clear()
                    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    start.record()
                    for _ in range(iters):
                        step()
                    end.record()
                    end.synchronize()
                    arms[fused].append(start.elapsed_time(end) / iters)
            for fused in (True, False):
                print(json.dumps(dict(demo=demo, lighting="fused" if fused else "op-by-op", image_size=256,
                                      nf=int(model.faces.shape[1]), iters_per_window=iters, rounds=rounds,
                                      ms_per_iter_median=round(float(np.median(arms[fused])), 4),
                                      ms_per_iter_min=round(float(np.min(arms[fused])), 4),
                                      library_launches_per_iter=int(launches[fused]), gpu=name, power_limit=power)), flush=True)
            print(json.dumps(dict(demo=demo, speedup_median=round(float(np.median(arms[False]) / np.median(arms[True])), 3))), flush=True)


if __name__ == "__main__":
    main()
