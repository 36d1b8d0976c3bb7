"""Time the normal-mapped surface lighting at the reference head's size (66 282 faces, texture_res 15 so T = 225 texels
per face, B = 1): the fused kernels (Lighting.fused = True) against the op-by-op PyTorch mirror (False), forward plus
backward to the vertices, textures, normal textures, metallic and roughness.  The arms alternate round by round in this
one process after a warm-up; every window is timed with CUDA events.

    python tools/time_normal_lighting.py [--iters 20] [--rounds 5]

Also times the forward kernel alone (b200r_normal_mapped_lighting_forward through _lib.call) and reports its achieved
bytes/s against the H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth.  The bytes are computed from the shapes: per
texel, textures, normal textures and output (3 floats each) and metallic and roughness (1 float each), plus the TBN,
faces and vertices once.  Prints one JSON line per measurement with the card's name and power limit read in this run.
The geometry is synthetic (a jittered UV sphere, random UVs and tangent-space normals); the kernel's work does not
depend on the values.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import jrender_b200 as jr  # noqa: E402
from jrender_b200 import _lib  # noqa: E402
from jrender_b200 import io as jio  # noqa: E402
from jrender_b200 import workloads as wl  # noqa: E402

HBM3_BYTES_PER_S = 3.35e12


def card():
    """'<name>, <power limit>' of device 0 from nvidia-smi (a read-only query)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True)
        if q.stdout.strip():
            return q.stdout.strip()
    except OSError:
        pass
    return torch.cuda.get_device_name(0) + ", power limit not readable"


def scene(dev, segments=194, rings=172, R=15, seed=0):
    """A jittered UV sphere of 2 * 194 * 171 = 66 348 faces, cut to the head's 66 282."""
    rng = np.random.default_rng(seed)
    v, f = wl.uv_sphere(segments, rings, jitter=0.002)
    f = f[:66282]
    nf, T = f.shape[0], R * R
    tbn = jio.create_TBN(rng.uniform(0, 1, (nf, 3, 2)).astype(np.float32), v[f])
    tbn = np.where(np.isfinite(tbn), tbn, 0).astype(np.float32)
    nt = rng.normal(0, 0.3, (1, nf, T, 3)).astype(np.float32)
    nt[..., 2] += 1
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(dev)
    return dict(v=t(v[None]), f=torch.from_numpy(f[None]).to(dev), tbn=t(tbn[None]), nt=t(nt),
                tex=t(rng.uniform(0, 1, (1, nf, T, 3))), met=t(rng.uniform(0, 1, (1, nf, T, 1))),
                rou=t(rng.uniform(0.2, 1, (1, nf, T, 1))), eye=torch.tensor([[0.3, 0.5, -2.0]], device=dev))


def step(s, light, params):
    m = jr.Mesh(params[0], s["f"], textures=params[1], normal_textures=params[2], TBN=s["tbn"], metallic_textures=params[3],
                roughness_textures=params[4])
    out = light(m, s["eye"]).textures
    out.backward(torch.ones_like(out))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--rounds", type=int, default=5)
    a = p.parse_args()
    dev = torch.device("cuda")
    s = scene(dev)
    who = card()
    light = jr.Lighting(intensity_ambient=0.45, intensity_directionals=1.0, directions=[0.65, -0.2, -1.0])
    params = [s[k].clone().requires_grad_(True) for k in ("v", "tex", "nt", "met", "rou")]
    nf, T = s["tex"].shape[1], s["tex"].shape[2]
    times = {True: [], False: []}
    for fused in (True, False):   # warm-up
        light.fused = fused
        step(s, light, params)
    torch.cuda.synchronize()
    for _ in range(a.rounds):
        for fused in (True, False):
            light.fused = fused
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                step(s, light, params)
            e1.record()
            torch.cuda.synchronize()
            times[fused].append(e0.elapsed_time(e1) / a.iters)
    for fused in (True, False):
        print(json.dumps(dict(what="normal-mapped lighting forward + backward", arm="fused" if fused else "op-by-op",
                              faces=nf, texels_per_face=T, batch=1, ms_median=float(np.median(times[fused])),
                              ms_min=float(np.min(times[fused])), rounds=a.rounds, iters=a.iters, card=who)))

    # the forward kernel alone
    out = torch.empty_like(s["tex"])
    d = light.directionals[0]
    from jrender_b200.lighting import _normalized_direction
    args = (1, 1, 1, 1, 1, nf, T, 1, nf, s["v"].shape[1], nf, T, 0.45, _lib._f3(light.ambient.light_color), 1.0,
            _lib._f3(d.light_color), _lib._f3(_normalized_direction(d.light_direction)), 1)
    call = lambda: _lib.call("b200r_normal_mapped_lighting_forward", dev, s["v"], s["f"].int(), s["tex"], s["nt"], s["tbn"],
                             s["met"], s["rou"], s["eye"], out, *args)
    call()
    torch.cuda.synchronize()
    ks = []
    for _ in range(a.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            call()
        e1.record()
        torch.cuda.synchronize()
        ks.append(e0.elapsed_time(e1) / a.iters)
    texels = nf * T
    nbytes = texels * 4 * (3 + 3 + 3 + 1 + 1) + nf * 4 * (9 + 3) + s["v"].numel() * 4
    ms = float(np.median(ks))
    print(json.dumps(dict(what="b200r_normal_mapped_lighting_forward kernel", faces=nf, texels_per_face=T, bytes=nbytes,
                          ms_median=ms, ms_min=float(np.min(ks)), achieved_TB_per_s=nbytes / (ms * 1e-3) / 1e12,
                          share_of_3_35_TB_per_s=nbytes / (ms * 1e-3) / HBM3_BYTES_PER_S, card=who)))


if __name__ == "__main__":
    main()
