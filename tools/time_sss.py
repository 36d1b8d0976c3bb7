"""Time one subsurface-scattering frame (Lighting with a with_SSS mesh) at the reference head's size: 66 282 faces,
texture_res 15 (T = 225 texels per face), B = 1, demo 1.5's lights.  The head is used when tools/stage_assets.py has
staged it (normal-map branch); otherwise a jittered UV sphere of the same face count with planar UVs stands in
(face-normal branch), and the output says which.

    python tools/time_sss.py [--iters 10] [--rounds 5]

Reports, one JSON line each, with the card's name and power limit read in this run:
- the whole frame (CUDA events around Lighting(mesh, eye), no grad), median over rounds;
- its split by the library's per-kernel profiler: the three texture-space SoftRas forwards, b200r_sss_stretch and
  b200r_sss_blur_pyramid (7 launches), the bake; the rest of the frame is PyTorch work: the op-by-op lighting terms,
  sqrt(textures * diffuse), the UV coordinates, allocations;
- the op-by-op lighting terms alone (events), and their share of the frame;
- the stretch + blur pyramid alone (events), against the reference's own blur kernels (oracle/_ref, built by
  oracle/build_ref_sss.py) in their 36-launch sequence on the same maps (3 channels x 3 levels x 4 blurs; the
  reference's elementwise passes are not counted), when that library is present.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import jrender_b200 as jr  # noqa: E402
from jrender_b200 import _lib, lighting  # noqa: E402
from jrender_b200 import workloads as wl  # noqa: E402
from tools.time_normal_lighting import card  # noqa: E402

HEAD = os.path.join(ROOT, "baseline", "_ref", "assets", "data", "head", "head.obj")
LIGHT = dict(intensity_ambient=0.45, color_ambient=[1, 1, 1], intensity_directionals=1.0,
             color_directionals=[1.0, 1.0, 1.0], directions=[0.65, -0.2, -1])   # demo1.5-SSS.py:27-29
SOFTRAS_IDS = (0, 20, 1, 4, 2)   # face setup, chunk rectangles, coarse binning, tile order, forward
K_SSS, K_BAKE = 25, 16


def scene(dev, R=15, seed=0):
    """(mesh, name): the staged head, else a UV sphere cut to the head's 66 282 faces with planar UVs."""
    if os.path.exists(HEAD):
        m = jr.Mesh.from_obj(HEAD, load_texture=True, texture_res=R, texture_type='surface', dr_type='softras',
                             normalization=True, with_SSS=True).to(dev)
        return m, "head (normal-map branch)"
    rng = np.random.default_rng(seed)
    v, f = wl.uv_sphere(194, 172, jitter=0.002)
    f = f[:66282]
    uv = np.clip((v[:, :2] / 1.1 + 1) / 2, 0, 1).astype(np.float32)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(dev)
    m = jr.Mesh(t(v[None]), torch.from_numpy(f[None]).to(dev), textures=t(rng.uniform(0, 1, (1, f.shape[0], R * R, 3))),
                texture_res=R, with_SSS=True, face_texcoords=t(uv[f][None]))
    return m, "generated UV sphere, 66 282 faces (face-normal branch)"


def timed(fn, iters, rounds):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / iters)
    return float(np.median(ms)), float(np.min(ms))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=10)
    p.add_argument("--rounds", type=int, default=5)
    a = p.parse_args()
    dev = torch.device("cuda")
    who = card()
    mesh, name = scene(dev)
    textures = mesh.textures
    eye = torch.tensor([[1.1, 0.5, -1.5]], device=dev)
    light = jr.Lighting(**LIGHT)
    nf, T = textures.shape[1], textures.shape[2]
    base = dict(mesh=name, faces=nf, texels_per_face=T, map=lighting.SSS_IMAGE_SIZE, card=who)

    def frame():
        mesh.textures = textures
        with torch.no_grad():
            return light(mesh, eye).textures

    def terms():
        """The op-by-op diffuse / specular light of Lighting, without SSS."""
        with torch.no_grad():
            return light._light_terms(mesh, eye)

    ms, mn = timed(frame, a.iters, a.rounds)
    print(json.dumps(dict(what="SSS frame (Lighting with with_SSS)", ms_median=ms, ms_min=mn, rounds=a.rounds,
                          iters=a.iters, **base)))

    L = _lib.lib()
    torch.cuda.synchronize()
    L.b200r_profile_reset()
    L.b200r_profile_enable(1)
    try:
        for _ in range(a.iters):
            frame()
        torch.cuda.synchronize()
    finally:
        L.b200r_profile_enable(0)

    def prof(k):
        t, n = C.c_double(0), C.c_longlong(0)
        assert L.b200r_profile_read(k, C.byref(t), C.byref(n)) == 0
        return t.value / a.iters, n.value // a.iters
    raster = sum(prof(k)[0] for k in SOFTRAS_IDS)
    sss_ms, sss_n = prof(K_SSS)
    bake_ms, bake_n = prof(K_BAKE)
    terms_ms, _ = timed(terms, a.iters, a.rounds)
    print(json.dumps(dict(what="SSS frame split (kernel time per frame, profiler)", texture_space_raster_ms=raster,
                          stretch_and_blur_ms=sss_ms, stretch_and_blur_launches=sss_n, bake_ms=bake_ms,
                          bake_launches=bake_n, rest_of_frame_ms=ms - raster - sss_ms - bake_ms,
                          lighting_terms_ms=terms_ms, lighting_terms_share=terms_ms / ms, **base)))

    # the stretch + pyramid alone, and the reference's blur sequence, on this frame's maps
    d, s = terms()
    if mesh.normal_textures is None:
        d, s = d[:, :, None, :], s[:, :, None, :]
    with torch.no_grad():
        world_map, irr_map, spec_map = lighting._sss_maps(d, s, mesh)
    S = lighting.SSS_IMAGE_SIZE
    su, sv = torch.empty((S, S), device=dev), torch.empty((S, S), device=dev)
    variances = [25, 75, 300]
    taps, widths = zip(*[lighting._sss_taps(v) for v in variances])
    ctaps = (C.c_float * 21)(*[t for lv in taps for t in lv])
    cwidths = (C.c_float * 3)(*widths)
    cweights = (C.c_float * 9)(*[w for ch in lighting.SSS_WEIGHTS for w in ch])
    nbytes = L.b200r_sss_workspace_bytes(S, S)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    out = torch.empty((S, S, 3), device=dev)

    def product():
        _lib.call("b200r_sss_stretch", dev, world_map, su, sv, S, S)
        _lib.call("b200r_sss_blur_pyramid", dev, su, sv, irr_map, spec_map, out, ws, nbytes, ctaps, cwidths, cweights,
                  3, S, S)
    pm, pmin = timed(product, a.iters, a.rounds)
    print(json.dumps(dict(what="b200r_sss_stretch + b200r_sss_blur_pyramid (7 launches)", ms_median=pm, ms_min=pmin,
                          **base)))
    from oracle import build_ref_sss
    RL = build_ref_sss.lib()
    if RL is None:
        print(json.dumps(dict(what="reference blur sequence", skipped="oracle/_ref/libjrender_ref_sss.so not built")))
        return
    irr_c = [irr_map[0, j].contiguous() for j in range(3)]
    gw = [(torch.tensor(t, dtype=torch.float32, device=dev), np.float32(w)) for t, w in zip(taps, widths)]

    def reference():
        for j in range(3):   # lighting.py:133-143: per channel, the stretch chains recomputed
            su_c, sv_c, x = su, sv, irr_c[j]
            for g, w in gw:
                su_c = build_ref_sss.blur(RL, su_c, su_c, g, w, 1)
                x = build_ref_sss.blur(RL, x, su_c, g, w, 1)
                sv_c = build_ref_sss.blur(RL, sv_c, sv_c, g, w, 0)
                x = build_ref_sss.blur(RL, x, sv_c, g, w, 0)
    rm, rmin = timed(reference, a.iters, a.rounds)
    print(json.dumps(dict(what="reference blur kernels, 36 launches", ms_median=rm, ms_min=rmin,
                          product_stretch_and_pyramid_ms=pm, speedup=rm / pm, **base)))


if __name__ == "__main__":
    main()
