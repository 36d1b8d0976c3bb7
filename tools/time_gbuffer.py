"""Time the normal and depth G-buffers (Lighting(Gbuffer=...)): the fused kernels (Lighting.fused = True) against the
op-by-op PyTorch mirror (False), forward plus backward to the vertices (and the normal textures on the normal-map path).
The arms alternate round by round in this one process after a warm-up; every window is timed with CUDA events.

    python tools/time_gbuffer.py [--iters 20] [--rounds 5]

Sizes: spot (5 856 faces, T = 25, B = 1) in both modes; a normal-mapped sphere cut to the head's 66 282 faces with
T = 225 texels (tools/time_normal_lighting.py's scene) in normal mode; a 39 200-face sphere at B = 4 in depth mode.
Prints one JSON line per measurement with the card's name and power limit read in this run.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import jrender_b200 as jr  # noqa: E402
from jrender_b200 import workloads as wl  # noqa: E402
from examples.render_gbuffers import load_spot  # noqa: E402
from tools.time_normal_lighting import card, scene as head_scene  # noqa: E402


def cases(dev):
    rng = np.random.default_rng(1)
    sv, sf = load_spot(dev)
    yield "spot_5856_T25", "normal", dict(v=sv[None], f=sf[None], tex=torch.rand((1, sf.shape[0], 25, 3), device=dev))
    yield "spot_5856_T25", "depth", dict(v=sv[None], f=sf[None], tex=torch.rand((1, sf.shape[0], 25, 3), device=dev))
    h = head_scene(dev)
    yield "head_66282_T225_normal_map", "normal", dict(v=h["v"], f=h["f"], tex=h["tex"], nt=h["nt"], tbn=h["tbn"])
    v, f = wl.sphere_by_faces(39200)
    v = torch.from_numpy(v).to(dev)[None].repeat(4, 1, 1) + torch.from_numpy(
        rng.normal(0, 0.01, (4,) + v.shape).astype(np.float32)).to(dev)
    f = torch.from_numpy(f).to(dev)[None].repeat(4, 1, 1)
    yield "sphere_39200_B4", "depth", dict(v=v, f=f, tex=torch.rand((4, f.shape[1], 1, 3), device=dev))


def step(sc, mode, fused, eyes):
    v = sc["v"].detach().requires_grad_(True)
    nt = sc["nt"].detach().requires_grad_(True) if "nt" in sc else None
    tr = jr.Transform(camera_mode='look_at')
    tr.set_eyes(eyes)
    light = jr.Lighting(Gbuffer=mode, transform=tr)
    light.fused = fused
    mesh = jr.Mesh(v, sc["f"], textures=sc["tex"], normal_textures=nt, TBN=sc.get("tbn"),
                   texture_res=int(round(sc["tex"].shape[2] ** 0.5)))
    out = light(mesh, eyes).textures
    out.sum().backward()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda")
    gpu = card()
    for name, mode, sc in cases(dev):
        B = sc["v"].shape[0]
        eyes = torch.tensor([wl.get_points_from_angles(2.732, 30.0, 40.0 + 90 * b) for b in range(B)], device=dev)
        for fused in (True, False):
            for _ in range(3):
                step(sc, mode, fused, eyes)
        torch.cuda.synchronize()
        ms = {True: [], False: []}
        for _ in range(a.rounds):
            for fused in (True, False):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    step(sc, mode, fused, eyes)
                e1.record()
                torch.cuda.synchronize()
                ms[fused].append(e0.elapsed_time(e1) / a.iters)
        f_ms, m_ms = float(np.median(ms[True])), float(np.median(ms[False]))
        print(json.dumps(dict(case=name, mode=mode, fused_ms=round(f_ms, 4), mirror_ms=round(m_ms, 4),
                              speedup=round(m_ms / f_ms, 2), fused_spread_ms=[round(min(ms[True]), 4), round(max(ms[True]), 4)],
                              mirror_spread_ms=[round(min(ms[False]), 4), round(max(ms[False]), 4)],
                              what="forward + backward per step, median of %d rounds x %d steps" % (a.rounds, a.iters),
                              gpu=gpu)), flush=True)


if __name__ == "__main__":
    main()
