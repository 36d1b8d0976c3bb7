"""Times NeRF volume rendering on the GPU: the fused kernels of jrender_b200.vol against the op-by-op PyTorch mirror of
the reference (oracle/volume.py), alternating in one process.

    python tools/time_nerf_step.py [--rounds 7] [--window 50] [--json out.json]

Per ray count (1024 = demo 7's N_rand, 8192 = its render chunk, 160 000) one step is: coarse compositing of 64 samples,
the fine resampling of 128 more, fine compositing of 192, and the backward of both colour maps (the network is left
out: raw is a leaf tensor).  Then one whole demo-7 training iteration (D=8, W=256 coarse and fine networks, 1024 rays,
Adam).  Each figure is the median over rounds of CUDA-event time per step over a window of steps; the two variants
alternate round by round.  The card's name and power limit are read in the same run and printed with the numbers.
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
from jrender_b200 import vol  # noqa: E402
from oracle import volume as ov  # noqa: E402

FUSED = (vol._composite, vol._resample)
MIRROR = (lambda raw, z, d, noise, white: ov.integrator_mirror(raw, z, d, noise, white),
          lambda z, w, n, u: ov.fine_stage_mirror(z, w, n, u))


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


def use(impl):
    vol._composite, vol._resample = impl


def volume_step(N, dev, S=64, Ni=128, C=5):
    g = torch.Generator(device=dev).manual_seed(N)
    d = torch.randn(N, 3, device=dev, generator=g)
    z = torch.sort(2. + 4. * torch.rand(N, S, device=dev, generator=g), -1)[0]
    raw0 = (2. * torch.randn(N, S, C, device=dev, generator=g)).requires_grad_(True)
    raw1 = (2. * torch.randn(N, S + Ni, C, device=dev, generator=g)).requires_grad_(True)

    def step():
        rgb0, _, _, w, _ = vol._composite(raw0, z, d, None, True)
        _, zf = vol._resample(z, w, Ni, None)
        rgb, _, _, _, _ = vol._composite(raw1, zf, d, None, True)
        (rgb.sum() + rgb0.sum()).backward()
    return step


def demo_step(dev):
    from examples import demo7_nerf as demo
    a = demo.parser().parse_args([])
    train_kw, _, _, opt = demo.create_nerf(a, dev)
    train_kw.update(near=a.near, far=a.far)
    g = torch.Generator(device=dev).manual_seed(0)
    o = torch.tensor([0., 0., 2.732], device=dev).expand(a.N_rand, 3)
    rd = torch.randn(a.N_rand, 3, device=dev, generator=g) * .15 + torch.tensor([0., 0., -1.], device=dev)
    target = torch.rand(a.N_rand, 3, device=dev, generator=g)

    def step():
        rgb, _, _, ex = vol.render(a.size, a.size, 55., chunk=a.chunk, rays=torch.stack([o, rd]), retraw=True,
                                   **train_kw)
        loss = demo.img2mse(rgb, target) + demo.img2mse(ex['rgb0'], target)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    return step


def window_ms(step, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        step()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def compare(make, rounds, window, warmup=3):
    steps = {}
    for name, impl in (("fused", FUSED), ("op_by_op", MIRROR)):
        use(impl)
        steps[name] = make()
        for _ in range(warmup):
            steps[name]()
    times = {k: [] for k in steps}
    for _ in range(rounds):
        for name, impl in (("fused", FUSED), ("op_by_op", MIRROR)):
            use(impl)
            times[name].append(window_ms(steps[name], window))
    use(FUSED)
    out = {k: float(np.median(v)) for k, v in times.items()}
    out["speedup"] = out["op_by_op"] / out["fused"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--window", type=int, default=50)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_nerf_step.py measures on a CUDA device; none found")
    dev = torch.device("cuda:0")
    res = dict(card=card(), rounds=args.rounds, window=args.window, unit="ms per step (median over rounds)")
    for N in (1024, 8192, 160000):
        res["volume_%d_x_64+128" % N] = compare(lambda: volume_step(N, dev), args.rounds, args.window)
        torch.cuda.empty_cache()
    res["demo7_iteration_1024_rays"] = compare(lambda: demo_step(dev), args.rounds, args.window)
    print(json.dumps(res, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
