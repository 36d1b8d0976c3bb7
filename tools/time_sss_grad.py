"""Time one differentiable subsurface-scattering frame (Lighting.sss_grad = True) at the reference head's size, forward
and backward, with the textures and the vertices requiring grad, on tools/time_sss.py's scene (the staged head, else a
UV sphere of the head's 66 282 faces).

    python tools/time_sss_grad.py [--iters 5] [--rounds 5]

Prints JSON lines:
- the frame, forward + backward, and the forward alone with grad (CUDA events, medians over alternating rounds);
- the backward's split by the library's per-kernel profiler: the pyramid backward (its recomputed forward passes and
  its transposed passes) with the stretch backward, the bake backward (the SSS and bake profiler ids, less the
  forward's own launches: the backwards share the forwards' profiler ids), the three texture-space SoftRas backwards;
  the rest of the backward is the op-by-op lighting backward in PyTorch;
- b200r_sss_blur_pyramid_backward alone at 2048^2, against torch autograd of the mirror (oracle/sss_grad.py) run in
  float32 on the same maps.
Each line records the card and its power limit.
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
from tools.time_sss import LIGHT, scene  # noqa: E402

K_SSS, K_BAKE, K_SOFTRAS_BWD, K_SOFTRAS_BWD_FINALIZE = 25, 16, 3, 9


def events(fns, iters, rounds):
    """Median ms per call of each fn, rounds alternating between them."""
    for fn in fns:
        fn()
    torch.cuda.synchronize()
    ms = [[] for _ in fns]
    for _ in range(rounds):
        for i, fn in enumerate(fns):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms[i].append(e0.elapsed_time(e1) / iters)
    return [float(np.median(m)) for m in ms]


def prof(run, ids):
    L = _lib.lib()
    torch.cuda.synchronize()
    L.b200r_profile_reset()
    L.b200r_profile_enable(1)
    try:
        run()
        torch.cuda.synchronize()
    finally:
        L.b200r_profile_enable(0)
    out = {}
    for k in ids:
        t, n = C.c_double(0), C.c_longlong(0)
        assert L.b200r_profile_read(k, C.byref(t), C.byref(n)) == 0
        out[k] = (t.value, n.value)
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=5)
    p.add_argument("--rounds", type=int, default=5)
    a = p.parse_args()
    dev = torch.device("cuda")
    who = card()
    mesh, name = scene(dev)
    tex0, v0 = mesh.textures.detach().clamp(0.05, 1), mesh.vertices.detach()
    light = jr.Lighting(**LIGHT)
    light.sss_grad = True
    eyes = torch.tensor([[1.1, 0.5, -1.5]], device=dev)
    weight = torch.rand_like(tex0)
    base = dict(mesh=name, faces=int(mesh.faces.shape[1]), texels_per_face=int(tex0.shape[2]),
                map=lighting.SSS_IMAGE_SIZE, card=who)

    def frame(backward=True):
        tx, v = tex0.clone().requires_grad_(True), v0.clone().requires_grad_(True)
        m = jr.Mesh(v, mesh.faces, textures=tx, texture_res=mesh.texture_res, normal_textures=mesh.normal_textures,
                    TBN=mesh.TBN, with_SSS=True, face_texcoords=mesh.face_texcoords)
        out = (light(m, eyes).textures * weight).sum()
        if backward:
            out.backward()
    both, fwd = events([frame, lambda: frame(False)], a.iters, a.rounds)
    print(json.dumps(dict(base, what="SSS frame with sss_grad, textures and vertices requiring grad",
                          forward_and_backward_ms=both, forward_ms=fwd, backward_ms=both - fwd)))
    st = prof(frame, (K_SSS, K_BAKE, K_SOFTRAS_BWD, K_SOFTRAS_BWD_FINALIZE))
    fst = prof(lambda: frame(False), (K_SSS, K_BAKE))   # the forward's own SSS and bake launches, taken off
    pyr_ms, pyr_n = st[K_SSS][0] - fst[K_SSS][0], st[K_SSS][1] - fst[K_SSS][1]
    bake_ms = st[K_BAKE][0] - fst[K_BAKE][0]
    ras_ms = st[K_SOFTRAS_BWD][0] + st[K_SOFTRAS_BWD_FINALIZE][0]
    print(json.dumps(dict(base, what="backward split (kernel time per frame, profiler)",
                          pyramid_and_stretch_backward_ms=pyr_ms, pyramid_and_stretch_launches=pyr_n, bake_backward_ms=bake_ms,
                          softras_backwards_ms=ras_ms, softras_backward_launches=st[K_SOFTRAS_BWD][1],
                          op_by_op_lighting_and_rest_ms=both - fwd - pyr_ms - bake_ms - ras_ms)))

    # the pyramid backward alone, against autograd of the float32 mirror on the same maps
    from oracle import sss_grad as sg
    S = lighting.SSS_IMAGE_SIZE
    world, irr, _ = wl.sss_maps(S, 11)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(dev)
    su_t, sv_t, irr_t = torch.empty((S, S), device=dev), torch.empty((S, S), device=dev), t(np.transpose(irr, (2, 0, 1)))
    _lib.call("b200r_sss_stretch", dev, t(np.transpose(world, (2, 0, 1))), su_t, sv_t, S, S)
    su, sv = su_t.cpu().numpy(), sv_t.cpu().numpy()
    taps, widths, weights, L = lighting._sss_levels()
    g = torch.randn((S, S, 3), device=dev)
    nbytes = _lib.lib().b200r_sss_backward_workspace_bytes(S, S, L)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    gi, gs = torch.empty_like(irr_t), torch.empty_like(irr_t)
    gu, gv = torch.empty_like(su_t), torch.empty_like(sv_t)

    def kernel(stretch_grads=True):
        _lib.call("b200r_sss_blur_pyramid_backward", dev, su_t, sv_t, irr_t, g, gi, gs, gu if stretch_grads else None,
                  gv if stretch_grads else None, ws, nbytes, taps, widths, weights, L, S, S)
    levels = sg.walk(su, sv, irr)
    args = [t(x).requires_grad_(True) for x in (su, sv, irr, np.zeros_like(irr))]

    def mirror():
        for x in args:
            x.grad = None
        sg.pyramid(*args, levels).backward(g)
    k_ms, k0_ms, m_ms = events([kernel, lambda: kernel(False), mirror], 1, a.rounds)
    print(json.dumps(dict(base, what="b200r_sss_blur_pyramid_backward at 2048^2 (12 launches, incl. its recomputed forward)",
                          kernel_ms=k_ms, kernel_without_stretch_grads_ms=k0_ms, torch_autograd_float32_mirror_ms=m_ms,
                          workspace_bytes=int(nbytes))))


if __name__ == "__main__":
    main()
