"""Shared helpers of the parity tests: run the CUDA path / the oracle on the same inputs."""
import numpy as np

from oracle import softras as osr


def run_oracle(fv, tex, params, grad=None, rows=None):
    out = osr.forward(fv, tex, params, rows=rows)
    if grad is not None:
        out["grad_faces"], out["grad_textures"] = osr.backward(fv, tex, out, grad, params, accumulate_double=True, rows=rows)
    return out


def run_cuda(fv, tex, params, grad=None, device="cuda:0", want_faces_info=True):
    """Through the public torch API -> ctypes -> C ABI -> sm_90a kernels."""
    import torch
    from jrender_b200 import SoftRasterizeFunction
    dev = torch.device(device)
    fvt = torch.from_numpy(np.ascontiguousarray(fv)).to(dev).requires_grad_(grad is not None)
    txt = torch.from_numpy(np.ascontiguousarray(tex)).to(dev).requires_grad_(grad is not None)
    fn = SoftRasterizeFunction(
        image_size=params["image_size"], near=params["near"], far=params["far"], fill_back=params["fill_back"],
        eps=params["eps"], sigma_val=params["sigma_val"], dist_func=params["dist_func"], dist_eps=params["dist_eps"],
        gamma_val=params["gamma_val"], aggr_func_rgb=params["aggr_func_rgb"], aggr_func_alpha=params["aggr_func_alpha"],
        texture_type=params["texture_type"], max_faces_per_pixel_for_grad=params["max_faces_per_pixel_for_grad"])
    fn.return_faces_info = want_faces_info
    soft_colors, aggrs_info, ids = fn.raw(fvt, txt)
    from jrender_b200.softras import pad_face_ids
    ids = pad_face_ids(ids)   # the library terminates the per-pixel lists with one -1; the reference pads all K slots
    out = dict(soft_colors=soft_colors.detach().cpu().numpy(), aggrs_info=aggrs_info.cpu().numpy(),
               faces_id_buffer=ids.cpu().numpy())
    if want_faces_info:
        out["faces_info"] = fn.save_vars[3].cpu().numpy()
    if grad is not None:
        soft_colors.backward(torch.from_numpy(np.ascontiguousarray(grad)).to(dev))
        out["grad_faces"] = fvt.grad.cpu().numpy()
        out["grad_textures"] = txt.grad.cpu().numpy()
    torch.cuda.synchronize()
    return out


def backward_bound_ratio(got, fv, tex, params, grad, exact_tail=False, row_stride=1):
    """Holds the SoftRas gradients of `got` (run_cuda) to the oracle's K6 sums, entry by entry.  The oracle's backward
    runs on the kernel's own forward outputs, so both sides sum the same pairs' terms: NaN / inf must sit where the
    oracle's do, and every finite entry meets |got - g64| <= osr.backward_bound.  exact_tail: the kernel's
    softras_exact_tail (the bound for 0 also holds under 1).  -> {tensor: worst |got - g64| / bound}."""
    fwd = dict(soft_colors=got["soft_colors"], aggrs_info=got["aggrs_info"], faces_id_buffer=got["faces_id_buffer"])
    fwd["faces_info"] = got["faces_info"] if "faces_info" in got else osr.forward(fv, tex, params, rows=(0, 0))["faces_info"]
    stats = osr.backward(fv, tex, fwd, grad, params, stats=True, exact_tail=exact_tail, row_stride=row_stride)
    worst = {}
    for k, st in zip(("grad_faces", "grad_textures"), stats):
        a, ref = got[k].astype(np.float64), st["g64"]
        assert np.array_equal(np.isnan(a), np.isnan(ref)), "%s NaN pattern differs" % k
        assert np.array_equal(np.isposinf(a), np.isposinf(ref)) and np.array_equal(np.isneginf(a), np.isneginf(ref)), k
        m = np.isfinite(ref)
        err, bound = np.abs(a[m] - ref[m]), osr.backward_bound(st)[m]
        bad = ~(err <= bound)
        if bad.any():
            i = np.flatnonzero(m.ravel())[np.flatnonzero(bad)]
            j = int(i[np.argmax(err[bad] / np.maximum(bound[bad], 1e-300))])
            idx = np.unravel_index(j, a.shape)
            raise AssertionError("%s: %d entries outside the bound; worst at %s: got %r, oracle %r, bound %r (A %r, N %d, "
                                 "E %r)" % (k, bad.sum(), idx, a[idx], ref[idx], osr.backward_bound(st)[idx],
                                            st["A"][idx], st["N"][idx], st["E"][idx]))
        worst[k] = float((err / np.maximum(bound, 1e-300)).max(initial=0.0))
    return worst


def sorted_ids(ids):
    """[B,K,H,W] -> per-pixel ascending id sets with -1 (empty) moved last."""
    a = ids.astype(np.int64).copy()
    a[a < 0] = np.iinfo(np.int32).max
    a.sort(axis=1)
    return a


def rel_err(a, b):
    """max |a-b| / max(|b|, tiny): scale-relative error of a whole tensor."""
    denom = max(float(np.abs(b).max()), 1e-30)
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max()) / denom


def nmr_scene(num_faces=280, batch=1, ts=2, fill_back=True, seed=1):
    from jrender_b200 import workloads as wl
    return wl.nmr_scene(num_faces, batch=batch, ts=ts, fill_back=fill_back, seed=seed)


def run_nmr_cuda(faces, textures, image_size, near=0.1, far=100.0, eps=1e-3, background_color=(0, 0, 0),
                 flags=(True, True, True), grads=None, device="cuda:0"):
    """Through jrender_b200.n3mr.RasterizeFunction -> ctypes -> C ABI.  grads = (g_rgb, g_alpha, g_depth)."""
    import torch
    from jrender_b200.n3mr import RasterizeFunction
    dev = torch.device(device)
    fc = torch.from_numpy(np.ascontiguousarray(faces)).to(dev).requires_grad_(grads is not None)
    tx = torch.from_numpy(np.ascontiguousarray(textures)).to(dev).requires_grad_(grads is not None) if flags[0] else None
    fn = RasterizeFunction(image_size, near, far, eps, background_color, *flags)
    rgb, alpha, depth = fn(fc, tx)
    sv = fn.save_vars
    out = dict(face_index_map=sv[2].cpu().numpy(), weight_map=sv[3].cpu().numpy(), depth_map=sv[4].cpu().numpy())
    if flags[0]:
        out.update(rgb_map=rgb.detach().cpu().numpy(), sampling_index_map=sv[8].cpu().numpy(), sampling_weight_map=sv[9].cpu().numpy())
    if flags[1]:
        out["alpha_map"] = alpha.detach().cpu().numpy()
    if flags[2]:
        out["face_inv_map"] = sv[7].cpu().numpy()
    if grads is not None:
        outs, gs = [], []
        for o, g, f in zip((rgb, alpha, depth), grads, flags):
            if f:
                outs.append(o)
                gs.append(torch.from_numpy(np.ascontiguousarray(g)).to(dev))
        torch.autograd.backward(outs, gs)
        out["grad_faces"] = fc.grad.cpu().numpy()
        if flags[0]:
            out["grad_textures"] = tx.grad.cpu().numpy()
    torch.cuda.synchronize()
    return out
