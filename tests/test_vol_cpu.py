"""NeRF volume rendering on the CPU: the oracles of oracle/volume.py against the reference's own jrender_vol
(tests/golden/ref_host_vol.npz, made by oracle/make_ref_host_vol_golden.py), jrender_b200.vol's host plumbing (rays,
sampling, batching, reshapes) with the two kernel calls swapped for the numpy oracle, and the C ABI's declarations."""
import json
import os
import re

import numpy as np
import pytest
import torch

from jrender_b200 import _lib
from jrender_b200 import vol
from oracle import volume as ov
from tests.conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_host_vol.npz")
G = np.load(GOLDEN)
META = json.loads(bytes(G["meta_json"]).decode())


def case_names(kind):
    return [n for n, m in META.items() if m["kind"] == kind]


def inp(name, k):
    return G["%s_in_%s" % (name, k)]


def out(name, k):
    return G["%s_out_%s" % (name, k)]


def recorded_draws(name):
    """The reference's random draws of a case, in draw order, with their kinds."""
    return [(kind, G["%s_draw%d" % (name, i)]) for i, kind in enumerate(META[name]["draws"])]


class Replay:
    """Stand-in for vol._random that hands out a golden case's recorded draws in order, checking kind and shape."""

    def __init__(self, name, device):
        self.draws = recorded_draws(name)
        self.device = device
        self.i = 0

    def __call__(self, shape, device, normal=False):
        kind, x = self.draws[self.i]
        self.i += 1
        assert kind == ("normal" if normal else "uniform") and tuple(x.shape) == tuple(shape), (kind, x.shape, shape)
        return torch.from_numpy(x).to(device)

    def done(self):
        return self.i == len(self.draws)


def close(got, ref, rel=1e-5):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    err = np.abs(got - ref)
    tol = rel * np.maximum(np.abs(ref), np.abs(ref).max() if ref.size else 0.)
    assert np.all(err <= tol + 1e-30), (err.max(), np.abs(ref).max())


@pytest.mark.parametrize("name", [n for n in case_names("integrator") if n != "int_s1"])
def test_oracle_composite_reproduces_reference_integrator(name):
    m = META[name]
    noise = None
    if m["draws"]:
        noise = G[name + "_draw0"] * np.float32(m["args"]["raw_noise_std"])
    got = ov.composite(inp(name, "raw"), inp(name, "z_vals"), inp(name, "rays_d"), noise, m["args"]["white_bkgd"])
    for k in ("rgb_map", "disp_map", "acc_map", "weights", "depth_map"):
        close(got[k], out(name, k))
    if name == "int_plain":   # the all-empty ray and the opaque sample the golden was built with
        assert out(name, "acc_map")[0] == 0 and out(name, "disp_map")[0] == np.float32(1e10)
        assert got["disp_map"][0] == np.float32(1e10)
        w = out(name, "weights")[1]
        S = w.shape[0]
        assert np.all(w[S // 2 + 1:] < 1e-9) and w[S // 2] > 0


def test_reference_integrator_degenerates_at_one_sample():
    """With S = 1 the reference's `dists[..., :1]` is empty, so its weights are [N, 0] and every map is zero; here the
    single sample takes the 1e10 * |d| interval of every ray's last sample instead (DESIGN.md section 9)."""
    name = "int_s1"
    assert out(name, "weights").shape == (4, 0)
    assert np.all(out(name, "acc_map") == 0)
    got = ov.composite(inp(name, "raw"), inp(name, "z_vals"), inp(name, "rays_d"))
    sigma = inp(name, "raw")[:, 0, 3]
    assert np.array_equal(got["acc_map"], (sigma > 0).astype(np.float32))


@pytest.mark.parametrize("name", case_names("sample_pdf"))
def test_oracle_resample_reproduces_reference_sample_pdf(name):
    m = META[name]
    u = G[name + "_draw0"] if m["draws"] else None
    bins = inp(name, "bins")
    got, none = ov.resample(inp(name, "weights"), m["args"]["N_samples"], u, bins=bins)
    assert none is None
    # the cdf is summed in another order, so a sample may sit on the other side of a bin edge: the inverse cdf is
    # continuous there, so the value still agrees
    assert np.abs(got - out(name, "samples")).max() <= 1e-6 * (bins.max() - bins.min())


@pytest.mark.parametrize("name", case_names("integrator")[:3] + case_names("sample_pdf"))
def test_torch_mirror_reproduces_reference(name):
    m = META[name]
    t = lambda a: torch.from_numpy(np.asarray(a))
    if m["kind"] == "integrator":
        noise = t(G[name + "_draw0"] * np.float32(m["args"]["raw_noise_std"])) if m["draws"] else None
        got = ov.integrator_mirror(t(inp(name, "raw")), t(inp(name, "z_vals")), t(inp(name, "rays_d")), noise,
                                   m["args"]["white_bkgd"])
        for k, g in zip(("rgb_map", "disp_map", "acc_map", "weights", "depth_map"), got):
            close(g.numpy(), out(name, k))
    else:
        u = t(G[name + "_draw0"]) if m["draws"] else None
        got = ov.sample_pdf_mirror(t(inp(name, "bins")), t(inp(name, "weights")), m["args"]["N_samples"],
                                   m["args"]["det"], u)
        # torch's cumsum order differs from both; (u - cdf0) / denom magnifies that by 1 / denom
        bins = inp(name, "bins")
        assert np.abs(got.numpy() - out(name, "samples")).max() <= 4e-6 * (bins.max() - bins.min())


@pytest.mark.parametrize("name", case_names("sample"))
def test_sample_reproduces_reference(name, monkeypatch):
    a = META[name]["args"]
    monkeypatch.setattr(vol, "_random", Replay(name, "cpu"))
    z = vol.sample(a["N_rays"], a["N_samples"], a["lindisp"], a["perturb"], torch.from_numpy(inp(name, "near")),
                   torch.from_numpy(inp(name, "far")))
    close(z.numpy(), out(name, "z_vals"), rel=1e-6)


@pytest.mark.parametrize("name", case_names("pinhole") + case_names("ndc"))
def test_rays_reproduce_reference(name):
    a = META[name]["args"]
    t = lambda k: torch.from_numpy(inp(name, k))
    if META[name]["kind"] == "pinhole":
        intr = t("intrinsic") if name + "_in_intrinsic" in G else None
        o, d = vol.pinhole_get_rays(a["H"], a["W"], a["focal"], t("c2w"), intr)
    else:
        o, d = vol.ndc_rays(a["H"], a["W"], a["focal"], a["near"], t("rays_o"), t("rays_d"))
    close(o.numpy(), out(name, "rays_o"), rel=1e-6)
    close(d.numpy(), out(name, "rays_d"), rel=1e-6)


def cpu_kernels(monkeypatch):
    """Swap vol's two kernel calls for the numpy oracle, so the host plumbing runs on the CPU."""
    def composite(raw, z, d, noise, white):
        r = ov.composite(raw.detach().numpy(), z.numpy(), d.numpy(), None if noise is None else noise.numpy(), white)
        return tuple(torch.from_numpy(r[k]) for k in ("rgb_map", "disp_map", "acc_map", "weights", "depth_map"))

    def resample(z, w, n, u):
        s, zf = ov.resample(w.numpy(), n, None if u is None else u.numpy(), z_vals=z.numpy())
        return torch.from_numpy(s), torch.from_numpy(zf)
    monkeypatch.setattr(vol, "_composite", composite)
    monkeypatch.setattr(vol, "_resample", resample)


def render_case(name, device):
    """vol.render on a golden render case with the analytic field; returns (outputs dict, replay)."""
    a = META[name]["args"]
    ch = a["channels"]
    replay = Replay(name, device)
    query = lambda pts, viewdirs, fn: ov.field_torch(pts, viewdirs, ch)
    kw = {k: a[k] for k in ("chunk", "ndc", "near", "far", "use_viewdirs", "N_samples", "N_importance", "perturb",
                            "raw_noise_std", "white_bkgd", "lindisp", "retraw")}
    if name + "_in_c2w" in G:
        geo = dict(c2w=torch.from_numpy(inp(name, "c2w")).to(device))
    else:
        r = torch.from_numpy(inp(name, "rays")).to(device)
        geo = dict(rays=(r[0], r[1]))
    return (lambda: vol.render(a["H"], a["W"], a["focal"], network_fn=None, network_query_fn=query, network_fine=None,
                               **geo, **kw)), replay


def check_render(name, rgb, disp, acc, extras, rel):
    got = dict(extras, rgb_map=rgb, disp_map=disp, acc_map=acc)
    assert sorted(got) == sorted(META[name]["outputs"])
    for k in got:
        if k != "raw":
            close(got[k].detach().cpu().numpy(), out(name, k), rel=rel)
    # raw is the network at the fine samples.  Where a bin's pdf mass is just above the 1e-5 floor, the inverse cdf
    # moves a sample by (bin width / mass) per unit of cdf, i.e. up to ~1e4 x an ulp of the cdf, and with det the last
    # u = 1 meets the cdf's end, which rounds either side of 1; the cdf's summation order is not the reference's, so a
    # few such samples land elsewhere.  Their weights are near zero (the maps above agree), so they are bounded, not
    # matched.
    g, r = got["raw"].detach().cpu().numpy(), out(name, "raw")
    err = np.abs(g - r)
    scale = np.abs(r).max()
    assert g.shape == r.shape and np.mean(err > rel * scale) <= 0.02 and err.max() <= 0.05 * scale, (err.max(), scale)


@pytest.mark.parametrize("name", case_names("render"))
def test_render_plumbing_reproduces_reference_on_cpu(name, monkeypatch):
    cpu_kernels(monkeypatch)
    run, replay = render_case(name, "cpu")
    monkeypatch.setattr(vol, "_random", replay)
    rgb, disp, acc, extras = run()
    assert replay.done()
    check_render(name, rgb, disp, acc, extras, rel=2e-5)


def test_render_shapes_follow_the_rays(monkeypatch):
    """Image rendering returns [H, W, ...] maps; a ray batch of any leading shape returns that shape."""
    cpu_kernels(monkeypatch)
    query = lambda pts, viewdirs, fn: ov.field_torch(pts, viewdirs, 4)
    c2w = torch.tensor([[1., 0., 0., 0.], [0., 1., 0., 0.], [0., 0., -1., 1.6]])
    rgb, disp, acc, ex = vol.render(3, 4, 4., chunk=5, c2w=c2w, ndc=False, near=.6, far=2.6, network_fn=None,
                                    network_query_fn=query, N_samples=8, N_importance=4, retraw=True)
    assert rgb.shape == (3, 4, 3) and disp.shape == (3, 4) and acc.shape == (3, 4)
    assert ex["raw"].shape == (3, 4, 12, 4) and ex["rgb0"].shape == (3, 4, 3) and ex["acc0"].shape == (3, 4)
    o = torch.zeros(2, 5, 3)
    d = torch.tensor([0., 0., 1.]).expand(2, 5, 3)
    o[..., 2] = -2
    rgb, disp, acc, ex = vol.render(8, 8, 4., rays=(o, d), ndc=False, near=1., far=3., network_fn=None,
                                    network_query_fn=query, N_samples=6)
    assert rgb.shape == (2, 5, 3) and disp.shape == (2, 5) and ex == {}


def test_kernel_entry_points_reject_cpu_tensors():
    z = torch.linspace(2, 6, 8).expand(3, 8)
    with pytest.raises(_lib.B200RasterError, match="no CPU fallback"):
        vol.integrator(torch.zeros(3, 8, 4), z, torch.ones(3, 3))
    with pytest.raises(_lib.B200RasterError, match="no CPU fallback"):
        vol.sample_pdf(z, torch.ones(3, 7), 4, det=True)


def test_header_declares_the_volume_entry_points_and_profiler_ids():
    src = open(os.path.join(ROOT, "include", "b200raster.h")).read()
    sigs = _lib.parse_header(src)
    assert len(sigs["b200r_vol_composite_forward"][1]) == 14
    assert len(sigs["b200r_vol_composite_backward"][1]) == 17
    assert len(sigs["b200r_vol_resample"][1]) == 10
    enum = re.search(r"enum \{ (B200R_K_\w+ = 0,[^}]*)\}", src).group(1)
    ids = dict((k, int(v)) for k, v in re.findall(r"(B200R_K_\w+) = (\d+)", enum))
    assert list(ids.values()) == list(range(len(ids)))
    assert (ids["B200R_K_DEBUG"], ids["B200R_K_VOL_COMPOSITE_FWD"], ids["B200R_K_VOL_COMPOSITE_BWD"],
            ids["B200R_K_VOL_RESAMPLE"]) == (21, 22, 23, 24)
    assert enum.rstrip().endswith("B200R_K_COUNT")
    assert int(re.search(r"#define B200R_VOL_MAX_SAMPLES (\d+)", src).group(1)) >= 1024
    cu = open(os.path.join(ROOT, "jrender_b200", "csrc", "vol_api.cu")).read()
    for k in ("B200R_K_VOL_COMPOSITE_FWD", "B200R_K_VOL_COMPOSITE_BWD", "B200R_K_VOL_RESAMPLE"):
        assert cu.count(k) == 1, k   # each kernel launches under exactly one id


def test_vol_names_stay_out_of_the_top_level_namespace():
    import jrender_b200 as jr
    for k in ("render", "render_rays", "integrator", "sample_pdf", "pinhole_get_rays", "ndc_rays", "batchify_rays"):
        assert not hasattr(jr, k), k
