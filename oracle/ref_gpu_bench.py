#!/usr/bin/env python
"""Times the reference's OWN CUDA kernels (oracle/_ref/libjrender_ref.so, compiled from the kernel strings under
/root/reference by oracle/build_ref.py) on this GPU, on the same inputs bench.py uses.  BASELINE INFRASTRUCTURE, never
product code: bench.py runs this file as a subprocess AFTER its own timed regions and copies the numbers into the
`reference_gpu` object of its JSON line ("beat THAT kernel", BASELINE.md section 2).

SoftRas legs (host semantics of jrender/renderer/dr/softras/soft_rasterize.py:34-133):
  naive   K1 + K2                       (bin_size = 0)
  c2f     K1 + K3 + K4 + K5             (bin_size = 64, max_elems_per_bin = nf / 5; the launcher keeps the reference's
                                         cudaMalloc / cudaMemset / cudaDeviceSynchronize calls, so it is wall-clock timed)
  bwd     [B,K,H,W] -> [B,H,W,K] id transpose (:108) + K6
NMR legs (jrender/renderer/dr/n3mr/n3mr.py:29-123): K7 + K8 forward, K9 + K10 backward, rgb mode.
Prints one JSON object; {"unavailable": "..."} when oracle/_ref was not built.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def med(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def softras(args):
    import numpy as np
    import torch
    from oracle import ref_gpu
    from oracle import softras as osr
    from jrender_b200 import workloads as wl
    dev = torch.device("cuda", 0)
    B, nf, H = args.batch, args.faces, args.image_size
    fv_h, tex_h = wl.make_scene(nf, batch=B)
    fv, tex = torch.from_numpy(fv_h).to(dev), torch.from_numpy(tex_h).to(dev)
    grad = torch.from_numpy(np.random.default_rng(2).uniform(-1, 1, (B, 4, H, H)).astype(np.float32)).to(dev)
    P = osr.Params(image_size=H)

    def wall(fn, n):
        ts = []
        for _ in range(n):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        return r, ts
    out = {"batch": B, "faces": nf, "image_size": H}
    if not args.skip_naive:
        ref_gpu.forward_t(fv, tex, P)
        fwd, ts = wall(lambda: ref_gpu.forward_t(fv, tex, P), args.naive_reps)
        out["naive_fwd_ms"] = med(ts)
    _, _ = wall(lambda: ref_gpu.forward_t(fv, tex, P, c2f_bin_size=64), 1)
    fwd_c2f, ts = wall(lambda: ref_gpu.forward_t(fv, tex, P, c2f_bin_size=64), args.reps)
    out["c2f_fwd_ms"] = med(ts)
    out["c2f_fwd_ms_min_max"] = [min(ts), max(ts)]
    src = fwd if not args.skip_naive else fwd_c2f

    def bwd():
        ids = src["faces_id_buffer"].permute(0, 2, 3, 1).contiguous()     # soft_rasterize.py:108
        return ref_gpu.backward_t(fv, tex, src, grad, P, ids_bhwk=ids)
    bwd()
    _, ts = wall(bwd, args.reps)
    out["bwd_ms"] = med(ts)
    out["step_ms_c2f"] = out["c2f_fwd_ms"] + out["bwd_ms"]
    out["frames_per_s_c2f"] = B * 1e3 / out["step_ms_c2f"]
    if "naive_fwd_ms" in out:
        out["step_ms_naive"] = out["naive_fwd_ms"] + out["bwd_ms"]
        out["frames_per_s_naive"] = B * 1e3 / out["step_ms_naive"]
    out["what"] = ("reference kernel strings compiled with nvcc -O3 for sm_90a, launched with the reference's grids "
                   "(512 threads, 1 thread / pixel); wall clock around synchronised calls, median of %d" % args.reps)
    return out


def nmr(args):
    import numpy as np
    import torch
    from oracle import ref_gpu
    from jrender_b200 import workloads as wl
    B, nf, H, ts_ = args.batch, args.faces, args.image_size, 2
    v, f = wl.sphere_by_faces(nf)
    eyes = np.asarray([wl.get_points_from_angles(2.732, 30.0, 360.0 * b / B) for b in range(B)], np.float32)
    fv = wl.face_vertices(wl.perspective(wl.look_at(np.repeat(v[None], B, 0), eyes), 30.0), f)
    faces = np.ascontiguousarray(np.concatenate([fv, fv[:, :, ::-1]], 1))
    tex = np.random.default_rng(1).random((B, faces.shape[1], ts_, ts_, ts_, 3), dtype=np.float32)
    g = np.random.default_rng(0).uniform(-1, 1, (B, H, H, 3)).astype(np.float32)
    L = ref_gpu._nmr_lib()
    import ctypes as C
    dev = torch.device("cuda", 0)
    fc, tx, gr = (torch.from_numpy(a).to(dev) for a in (faces, tex, g))
    p = lambda t: C.c_void_p(t.data_ptr())                                           # noqa: E731
    one = torch.zeros(1, dtype=torch.float32, device=dev)
    nf2 = faces.shape[1]
    fim = torch.empty((B, H, H), dtype=torch.int32, device=dev)
    wm = torch.empty((B, H, H, 3), dtype=torch.float32, device=dev)
    dm = torch.empty((B, H, H), dtype=torch.float32, device=dev)
    lock = torch.empty((B, H, H), dtype=torch.int32, device=dev)
    finv_faces = torch.zeros_like(fc)
    rgb = torch.empty((B, H, H, 3), dtype=torch.float32, device=dev)
    sim = torch.empty((B, H, H, 8), dtype=torch.int32, device=dev)
    swm = torch.empty((B, H, H, 8), dtype=torch.float32, device=dev)
    gf = torch.empty((B, nf2, 3, 3), dtype=torch.float32, device=dev)
    gt = torch.empty_like(tx)

    def fwd():
        rc = L.ref_nmr_forward_face_index_map(p(fc), p(finv_faces), p(fim), p(wm), p(dm), p(one), p(lock), B, nf2, H, 0.1, 100.0, 1, 0, 0, 1)
        rc |= L.ref_nmr_forward_texture_sampling(p(fc), p(tx), p(fim), p(wm), p(dm), p(rgb), p(sim), p(swm), B, nf2, H, ts_, 1e-3)
        if rc:
            raise RuntimeError("reference NMR forward failed: %d" % rc)

    def bwd():
        rc = L.ref_nmr_backward_pixel_map(p(fc), p(fim), p(rgb), p(one), p(gr), p(one), p(gf), B, nf2, H, 1e-3, 1, 0)
        rc |= L.ref_nmr_backward_textures(p(fim), p(swm), p(sim), p(gr), p(gt), B, nf2, H, ts_)
        if rc:
            raise RuntimeError("reference NMR backward failed: %d" % rc)

    def wall(fn, n):
        ts = []
        for _ in range(n):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        return ts
    fwd(); bwd()
    tf, tb = med(wall(fwd, args.reps)), med(wall(bwd, args.reps))
    return {"batch": B, "faces": nf2, "image_size": H, "texture_size": ts_, "fwd_ms": tf, "bwd_ms": tb, "step_ms": tf + tb,
            "frames_per_s": B * 1e3 / (tf + tb),
            "what": "reference K7+K8 / K9+K10 compiled with nvcc -O3 for sm_90a, reference launch shapes, rgb mode, "
                    "no background mix / flip (host ops); wall clock around synchronised calls, median of %d" % args.reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kind", default="softras", choices=["softras", "nmr"])
    ap.add_argument("--faces", type=int, default=39200)
    ap.add_argument("--image-size", type=int, default=1024)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--naive-reps", type=int, default=2)
    ap.add_argument("--skip-naive", action="store_true")
    args = ap.parse_args()
    try:
        from oracle import ref_gpu
        if not ref_gpu.available():
            print(json.dumps({"unavailable": "oracle/_ref/libjrender_ref.so not built (needs /root/reference at build time)"}))
            return
        print(json.dumps(softras(args) if args.kind == "softras" else nmr(args)), flush=True)
    except Exception as e:  # a baseline leg must never take the bench line down
        print(json.dumps({"unavailable": "%s: %s" % (type(e).__name__, e)}), flush=True)


if __name__ == "__main__":
    main()
