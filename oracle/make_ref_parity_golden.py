"""Golden samples of the reference's OWN kernels at full workload size (TEST INFRASTRUCTURE).

    python -m oracle.make_ref_parity_golden --out DIR     # on a GPU, with oracle/_ref/libjrender_ref.so built

tests/test_softras_gpu.py::test_against_reference_kernels_on_gpu and
tests/test_nmr_gpu.py::test_c4_against_reference_kernels_on_gpu compare the product with the reference kernels at
sizes the CPU oracle would take minutes for.  The full outputs are tens of MB, so each case stores a fixed, seeded
sample of them: the per-pixel outputs at 2048 pixels and the gradients of 2048 faces, drawn uniformly (every 4th of
8192 seeded pixel draws, every 2nd of 4096 seeded face draws; float16 gradients: its 5e-4 relative rounding is far below the relative-L1 tolerances the tests apply to them).  The inputs
are not stored -- they are the seeded scenes of jrender_b200.workloads -- but their float64 sums are, so a test
notices when a scene generator changes.

Besides DIR/parity_*.npz (copied to tests/golden/), DIR/report.json gives, per case, the test's statistics
of the product against the reference over the full outputs and over the stored sample.
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jrender_b200 import workloads as wl  # noqa: E402
from oracle import ref_gpu, softras as osr  # noqa: E402

SOFTRAS_CASES = [(3280, 512), (39200, 512), (39200, 1024)]   # (faces, image size) of test_against_reference_kernels_on_gpu


def sample_indices(n, k, seed):
    return np.sort(np.random.default_rng(seed).choice(n, size=min(k, n), replace=False)).astype(np.int32)


def pixel_sample(npix):
    return sample_indices(npix, 8192, 100)[::4]


def face_sample(nf):
    return sample_indices(nf, 4096, 101)[::2]


def softras_inputs(nfaces, H):
    fv, tex = wl.make_scene(nfaces, batch=1)
    g = np.random.default_rng(2).uniform(-1, 1, (1, 4, H, H)).astype(np.float32)
    return fv, tex, g


def nmr_inputs():
    faces, tex = wl.nmr_scene(39200, batch=1, ts=2, fill_back=True, seed=1)
    g = np.random.default_rng(0).uniform(-1, 1, (1, 1024, 1024, 3)).astype(np.float32)
    ga = np.random.default_rng(1).uniform(-1, 1, (1, 1024, 1024)).astype(np.float32)
    return faces, tex, g, ga


def checksums(*arrays):
    return np.array([float(np.asarray(a, np.float64).sum()) for a in arrays], np.float64)


def softras_sample(out, pix, fidx):
    """[B=1] outputs -> the stored sample: ids sorted per pixel (-1 last), RGBA, gradients of the sampled faces."""
    K = out["faces_id_buffer"].shape[1]
    ids = out["faces_id_buffer"][0].reshape(K, -1)[:, pix].T.astype(np.int64)
    ids[ids < 0] = np.iinfo(np.int32).max
    ids.sort(axis=1)
    ids[ids == np.iinfo(np.int32).max] = -1
    return dict(ids=ids.astype(np.int32), soft_colors=out["soft_colors"][0].reshape(4, -1)[:, pix].T.copy(),
                grad_faces=out["grad_faces"][0][fidx], grad_textures=out["grad_textures"][0][fidx])


def softras_stats(ref, got):
    same = (ref["ids"] == got["ids"]).all(1).mean()
    d = np.abs(ref["soft_colors"] - got["soft_colors"]).max(1)
    r = dict(same=float(same), colour_frac_over_2e3=float((d > 2e-3).mean()), colour_mean=float(d.mean()))
    for k in ("grad_faces", "grad_textures"):
        a, b = ref[k].astype(np.float64), got[k].astype(np.float64)
        m = np.isfinite(a) & np.isfinite(b)
        r[k + "_rel_l1"] = float(np.abs(a[m] - b[m]).sum() / np.abs(a[m]).sum())
    return r


def nmr_sample(out, pix, fidx):
    return dict(face_index_map=out["face_index_map"][0].reshape(-1)[pix].astype(np.int32),
                depth_map=out["depth_map"][0].reshape(-1)[pix].astype(np.float32),
                rgb_map=out["rgb_map"][0].reshape(-1, 3)[pix].astype(np.float32),
                grad_faces=out["grad_faces"][0][fidx], grad_textures=out["grad_textures"][0][fidx])


def nmr_stats(ref, got):
    same = ref["face_index_map"] == got["face_index_map"]
    dd = np.abs(ref["depth_map"] - got["depth_map"])[same]
    dc = np.abs(ref["rgb_map"] - got["rgb_map"])[same]
    r = dict(same=float(same.mean()), depth_frac_over_1e4=float((dd > 1e-4).mean()), depth_max=float(dd.max()),
             rgb_frac_over_2e3=float((dc > 2e-3).mean()), rgb_max=float(dc.max()))
    for k in ("grad_faces", "grad_textures"):
        a, b = ref[k].astype(np.float64), got[k].astype(np.float64)
        m = np.isfinite(a) & np.isfinite(b)
        r[k + "_rel_l1"] = float(np.abs(a[m] - b[m]).sum() / np.abs(a[m]).sum())
    return r


def _provenance(source):
    import torch
    return json.dumps(dict(gpu=torch.cuda.get_device_name(0), nvcc="-O3 -gencode arch=compute_90a,code=sm_90a (fmad default on)",
                           source=source))


def _f16(d):
    return {k: (v.astype(np.float16) if k.startswith("grad_") else v) for k, v in d.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    from tests.util import run_cuda, run_nmr_cuda
    os.makedirs(args.out, exist_ok=True)
    report = []
    for nf, H in SOFTRAS_CASES:
        fv, tex, g = softras_inputs(nf, H)
        P = osr.Params(image_size=H)
        ref = ref_gpu.run(fv, tex, P, grad=g)
        got = run_cuda(fv, tex, P, grad=g, want_faces_info=False)
        pix, fidx = pixel_sample(H * H), face_sample(nf)
        rs, gs = softras_sample(ref, pix, fidx), softras_sample(got, pix, fidx)
        allpix, allf = np.arange(H * H), np.arange(nf)
        full = softras_stats(softras_sample(ref, allpix, allf), softras_sample(got, allpix, allf))
        np.savez_compressed(os.path.join(args.out, "parity_softras_%d_%d.npz" % (nf, H)), pixels=pix, faces=fidx,
                            input_sums=checksums(fv, tex, g), params=json.dumps(dict(P)), **_f16(rs),
                            provenance=_provenance("jrender/renderer/dr/softras/cuda/soft_rasterize.py kernels via oracle/build_ref.py"))
        np.savez_compressed(os.path.join(args.out, "product_softras_%d_%d.npz" % (nf, H)), **_f16(gs))
        r = dict(case="softras_%d_%d" % (nf, H), full=full, sample=softras_stats(_f16(rs), _f16(gs)))
        report.append(r)
        print(json.dumps(r), flush=True)
    faces, tex, g, ga = nmr_inputs()
    ref = ref_gpu.nmr_run(faces, tex, 1024, 0.1, 100.0, 1e-3, (0, 0, 0), (True, True, False), grads=(g, ga, None))
    got = run_nmr_cuda(faces, tex, 1024, flags=(True, True, False), grads=(g, ga, None))
    pix, fidx = pixel_sample(1024 * 1024), face_sample(faces.shape[1])
    rs, gs = nmr_sample(ref, pix, fidx), nmr_sample(got, pix, fidx)
    full = nmr_stats(nmr_sample(ref, np.arange(1024 * 1024), np.arange(faces.shape[1])),
                     nmr_sample(got, np.arange(1024 * 1024), np.arange(faces.shape[1])))
    np.savez_compressed(os.path.join(args.out, "parity_nmr_39200_1024.npz"), pixels=pix, faces=fidx,
                        input_sums=checksums(faces, tex, g, ga), **_f16(rs),
                        provenance=_provenance("jrender/renderer/dr/n3mr/cuda/rasterize.py kernels via oracle/build_ref.py"))
    np.savez_compressed(os.path.join(args.out, "product_nmr_39200_1024.npz"), **_f16(gs))
    r = dict(case="nmr_39200_1024", full=full, sample=nmr_stats(_f16(rs), _f16(gs)))
    report.append(r)
    print(json.dumps(r), flush=True)
    json.dump(report, open(os.path.join(args.out, "report.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
