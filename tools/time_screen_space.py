"""Time SSAO_cuda (256 samples), SSDO_cuda (1024 samples) and FXAA_cuda at 1024^2 against the reference's own kernels
(oracle/_ref, built by oracle/build_ref_screen.py), on spot's G-buffers on a ground plane (examples/render_ssao.py).

    python tools/time_screen_space.py [--iters 10] [--rounds 3] [--size 1024]

For SSAO and SSDO the reference is timed twice: the whole op as it runs (cudaMalloc of 48 B of curand state per pixel,
the init kernel, cudaDeviceSynchronize, the kernel, cudaFree), and its kernel alone on states initialised once
beforehand (the kernel advances them, so later windows draw other numbers; the work per sample is the same).  Product
and reference alternate round by round after a warm-up; each window is timed with CUDA events around `iters` calls.
Prints one JSON line per measurement, with the card's name and power limit read in this run.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from jrender_b200.render2 import FXAA_cuda, SSAO_cuda, SSDO_cuda  # noqa: E402
from examples.render_gbuffers import load_spot  # noqa: E402
from examples.render_ssao import gbuffers, ground_plane, shade  # noqa: E402
from oracle import build_ref_screen  # noqa: E402
from tools.time_normal_lighting import card  # noqa: E402

SAMPLES = {"ssao": 256, "ssdo": 1024}
RADIUS = 0.15


def window(fn, iters):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def arms(L, S, depth, face_ind, normal, width, color):
    """{(pass, arm): callable}."""
    st = torch.cuda.current_stream().cuda_stream
    npad = build_ref_screen._padded(S)
    states = torch.empty(npad * L.ref_screen_state_bytes(), dtype=torch.uint8, device=depth.device)
    assert L.ref_screen_curand_init(states.data_ptr(), S, st) == 0
    occ = torch.empty(npad, device=depth.device)
    img = torch.empty((npad, 3), device=depth.device)
    cpad = torch.zeros((npad, 3), device=depth.device)
    cpad[:S * S] = color.reshape(-1, 3)
    p = [t.data_ptr() for t in (depth, normal, face_ind)]
    tex = torch.zeros((S + 2, S, 3), device=depth.device)   # build_ref_screen.fxaa's zero padding, made once
    tex[:S] = color
    fx = torch.empty_like(color)
    n_ao, n_do = SAMPLES["ssao"], SAMPLES["ssdo"]
    return {
        ("ssao", "product"): lambda: SSAO_cuda(depth, face_ind, normal, width, n_ao, RADIUS),
        ("ssao", "reference_op"): lambda: build_ref_screen.ssao(L, depth, face_ind, normal, width, n_ao, RADIUS),
        ("ssao", "reference_kernel"): lambda: L.ref_ssao_kernel(occ.data_ptr(), *p, states.data_ptr(), S, n_ao, RADIUS,
                                                                width, st),
        ("ssdo", "product"): lambda: SSDO_cuda(color, depth, face_ind, normal, width, n_do, RADIUS),
        ("ssdo", "reference_op"): lambda: build_ref_screen.ssdo(L, color, depth, face_ind, normal, width, n_do, RADIUS),
        ("ssdo", "reference_kernel"): lambda: L.ref_ssdo_kernel(img.data_ptr(), cpad.data_ptr(), *p, states.data_ptr(), S,
                                                                n_do, RADIUS, width, st),
        ("fxaa", "product"): lambda: FXAA_cuda(color),
        ("fxaa", "reference_kernel"): lambda: L.ref_fxaa(fx.data_ptr(), tex.data_ptr(), S, st),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--size', type=int, default=1024)
    a = ap.parse_args()
    L = build_ref_screen.lib()
    if L is None:
        sys.exit("oracle/_ref/libjrender_ref_screen.so is not built (python -m oracle.build_ref_screen)")
    dev = torch.device("cuda")
    gpu = card()
    depth, face_ind, normal, width = gbuffers(*ground_plane(*load_spot(dev)), a.size)
    color = shade(face_ind, normal).contiguous()
    normal = normal.contiguous()
    fns = arms(L, a.size, depth, face_ind, normal, width, color)
    for fn in fns.values():   # warm-up: module loads, allocator
        fn()
    times = {k: [] for k in fns}
    for _ in range(a.rounds):
        for k, fn in fns.items():
            times[k].append(window(fn, a.iters))
    covered = int((face_ind >= 0).sum())
    for (p, arm), ts in times.items():
        print(json.dumps({"pass": p, "arm": arm, "size": a.size, "samples": SAMPLES.get(p), "covered_pixels": covered,
                          "ms_min": round(min(ts), 4), "ms_median": round(sorted(ts)[len(ts) // 2], 4),
                          "ms_all": [round(t, 4) for t in ts], "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
