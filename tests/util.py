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


def same_nonfinite(a, b, what):
    """NaN, +inf and -inf in the same places of a and b; returns the mask of b's finite entries."""
    assert np.array_equal(np.isnan(a), np.isnan(b)), "%s NaN pattern differs" % what
    assert np.array_equal(np.isposinf(a), np.isposinf(b)) and np.array_equal(np.isneginf(a), np.isneginf(b)), what
    return np.isfinite(b)


def hold_to_bound(a, ref, bound, what, live=None):
    """Every finite entry of a within its bound of ref, bit-equal where the bound is 0, NaN / inf where ref has them.
    live ([B,H,W] site bits, None): named in the failure message.  -> (worst |a - ref| / bound, entries with bound > 0)."""
    m = same_nonfinite(a, ref, what)
    eq0 = (bound == 0) & m
    a32, r32 = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(ref, np.float32)
    diff0 = eq0 & (a32.view(np.uint32) != r32.view(np.uint32))
    err = np.where(m, np.abs(a.astype(np.float64) - ref.astype(np.float64)), 0.0)
    bad = diff0 | (m & ~(err <= bound))
    if bad.any():
        ratio = np.where(bad, err / np.where(bound > 0, bound, 1e-300), 0.0)
        idx = np.unravel_index(int(np.argmax(np.where(diff0, np.inf, ratio))), a.shape)
        sites = "" if live is None else " live sites %s" % osr.site_names(live[(idx[0],) + tuple(idx[-2:])])
        raise AssertionError("%s: %d entries outside the forward bound; worst at %s: got %r, oracle %r, bound %r%s" % (
            what, int(bad.sum()), idx, float(a[idx]), float(ref[idx]), float(bound[idx]), sites))
    pos = m & (bound > 0)
    return float((err[pos] / bound[pos]).max(initial=0.0)), int(pos.sum())


def forward_bound_ratio(got, fv, tex, params, exact_tail=False, row_stride=1, ref=None, nan=False):
    """Holds the SoftRas forward's float outputs of `got` (run_cuda) to the oracle, entry by entry: soft_colors and the
    softmax sum (aggrs_info[:, 0]) within osr.forward_bound's per-entry bound (bit-equal where it is 0: no rounding
    site live), softmax_max and the hard-mode aggregates bit-exact.  nan=False: no NaN in any of these outputs;
    nan=True (inputs on which the reference's own arithmetic yields NaN): NaN / inf where the oracle's are.
    exact_tail: the kernel's softras_exact_tail; each setting has its own bound, since the two tails round
    differently.  row_stride: compare rows 0, row_stride, ... only.  ref: osr.forward_bound's result for these inputs,
    if already computed.
    -> dict(colors=(worst err / bound, entries with a non-zero bound), sum=(...), ref=the oracle's outputs)."""
    H = int(params["image_size"])
    # the forward takes the fp32 tails in euclidean mode only; the other distances always run the exact tails
    # (softras_fwd.cu b200r_launch_forward)
    exact_tail = exact_tail or params["dist_func"] != "euclidean"
    if ref is None:
        ref = osr.forward_bound(fv, tex, params, exact_tail=exact_tail, row_stride=row_stride)
    rows = np.arange(0, H, row_stride)
    sc, ag = got["soft_colors"][:, :, rows], got["aggrs_info"][:, :, rows]
    if not nan:
        assert not np.isnan(sc).any(), "NaN in soft_colors"
        assert not np.isnan(ag).any(), "NaN in aggrs_info"
    live = ref["live"][:, rows]
    res = dict(ref=ref)
    res["colors"] = hold_to_bound(sc, ref["soft_colors"][:, :, rows], ref["bound_colors"][:, :, rows], "soft_colors", live)
    if params["aggr_func_rgb"] == "softmax":
        marg = ref["marginal"][:, rows]
        same = (ag[:, 1] == ref["aggrs_info"][:, 1, rows]) | (np.isnan(ag[:, 1]) & np.isnan(ref["aggrs_info"][:, 1, rows]))
        assert same.all(), "softmax_max not bit-exact (%d entries, %d of them at pixels with a marginal decision)" % (
            (~same).sum(), (~same & (marg != 0)).sum())
        res["sum"] = hold_to_bound(ag[:, 0], ref["aggrs_info"][:, 0, rows], ref["bound_sum"][:, rows], "softmax_sum", live)
    else:
        assert np.array_equal(ag, ref["aggrs_info"][:, :, rows], equal_nan=True), "hard-mode aggrs_info not bit-exact"
    return res


def pooled_bound(ref_sc, bound):
    """2x2 mean pooling of the oracle's soft_colors in the order of the forward's anti-aliasing epilogue and avg_pool2d
    (window row-major, sum / 4), and the bound on the pooled kernel output: each input anywhere in [ref - bound,
    ref + bound] (ends rounded outwards to float), the same float adds evaluated on the ends.  -> (pooled, bound)."""
    def pool(s):
        return (((s[:, :, 0::2, 0::2] + s[:, :, 0::2, 1::2]) + s[:, :, 1::2, 0::2]) + s[:, :, 1::2, 1::2]) / np.float32(4)
    r64 = ref_sc.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        lo64, hi64 = r64 - bound, r64 + bound
        lo, hi = lo64.astype(np.float32), hi64.astype(np.float32)
        lo = np.where(lo > lo64, np.nextafter(lo, np.float32(-np.inf)), lo)
        hi = np.where(hi < hi64, np.nextafter(hi, np.float32(np.inf)), hi)
        lo, hi = np.where(bound == 0, ref_sc, lo), np.where(bound == 0, ref_sc, hi)
        p, plo, phi = pool(ref_sc), pool(lo), pool(hi)
        b = np.maximum(phi.astype(np.float64) - p, p.astype(np.float64) - plo)
    b = np.where(np.isnan(b), np.inf, b)
    b[(plo == p) & (phi == p)] = 0.0
    return p, b


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
