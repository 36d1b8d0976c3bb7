"""The render2 image passes that read G-buffers (jrender/render2/utils/cuda): screen-space ambient occlusion, screen-space
directional occlusion, FXAA and the small image filter `Render` composes them with.

Same names, signatures and layouts as the reference.  Images are square, [is, is, C] HWC with row 0 at the top:
    depth          [is, is]     view-space z of the nearest face, e.g. aggrs_info[0, 0] of a hard SoftRas raster
    face_ind_buffer [is, is]    face id of that face, -1 on the background (aggrs_info[0, 1])
    normal_buffer  [is, is, 3]  view-space normals
    width          tan(viewing_angle): x, y = NDC * width * z

SSAO_cuda, SSDO_cuda and FXAA_cuda run one sm_90a kernel each (csrc/screen_space_api.cu) on the current stream: they
allocate only their output, never synchronise, and can be captured in a CUDA graph.  Their results are the reference
kernels' bit for bit.  No gradient flows through them: like the reference's jt.code ops, which have no grad source,
they return tensors that do not require grad.  Inputs are converted the way the reference converts them (float32,
int32); they must be CUDA tensors.
"""
import torch

from . import _lib


def _square(name, t, channels):
    """The image size of t, a square [is, is] (channels None) or [is, is, channels] tensor; ValueError otherwise."""
    if not isinstance(t, torch.Tensor):
        raise ValueError("%s must be a torch.Tensor, got %s" % (name, type(t).__name__))
    want = 2 if channels is None else 3
    if t.dim() != want or t.shape[0] != t.shape[1] or t.shape[0] < 1 or (channels is not None and t.shape[2] != channels):
        shape = "[is, is]" if channels is None else "[is, is, %d]" % channels
        raise ValueError("%s must be a square %s image, got %s" % (name, shape, tuple(t.shape)))
    return t.shape[0]


def _check(**buffers):
    """Every (tensor, channels) in `buffers` square, all of one size and on one CUDA device; returns the size."""
    sizes = {name: _square(name, t, c) for name, (t, c) in buffers.items()}
    if len(set(sizes.values())) > 1:
        raise ValueError("the buffers must match in size, got %s"
                         % ", ".join("%s %s" % (n, tuple(buffers[n][0].shape)) for n in sizes))
    for name, (t, _) in buffers.items():
        if not t.is_cuda:
            raise ValueError("%s must be a CUDA tensor (there is no CPU path), got device %s" % (name, t.device))
    if len({t.device for t, _ in buffers.values()}) > 1:
        raise ValueError("the buffers must be on one device, got %s" % ", ".join(str(t.device) for t, _ in buffers.values()))
    return next(iter(sizes.values()))


def _gbuffer(depth, face_ind_buffer, normal_buffer, sample_num, **more):
    is_ = _check(depth=(depth, None), face_ind_buffer=(face_ind_buffer, None), normal_buffer=(normal_buffer, 3), **more)
    if int(sample_num) < 0:
        raise ValueError("sample_num must be >= 0, got %r" % (sample_num,))
    return (is_, depth.detach().float().contiguous(), face_ind_buffer.detach().int().contiguous(),
            normal_buffer.detach().float().contiguous())


def SSAO_cuda(depth, face_ind_buffer, normal_buffer, width, sample_num, sample_range_r):
    """Screen-space ambient occlusion (SSAO_cuda.py:3-212) -> occlusion [is, is], float32.

    For each covered pixel, the share of `sample_num` points, drawn in the half ball of radius `sample_range_r` on the normal's side of the
    pixel's view-space point, that lie behind the depth buffer where they project; 0 on the background.  Pixel i draws
    from curand's XORWOW stream curand_init(1, i, 0), as the reference does.  No gradient."""
    is_, d, f, n = _gbuffer(depth, face_ind_buffer, normal_buffer, sample_num)
    out = torch.empty((is_, is_), dtype=torch.float32, device=d.device)
    _lib.call("b200r_ssao", d.device, d, f, n, out, is_, int(sample_num), float(sample_range_r), float(width))
    return out


def SSDO_cuda(color, depth, face_ind_buffer, normal_buffer, width, sample_num, sample_range_r):
    """Screen-space directional occlusion with one bounce of indirect light (SSDO_cuda.py:3-247) -> [is, is, 3].

    The same samples as SSAO_cuda: each covered pixel's colour times the share of samples no more than 0.01 in front of
    the depth buffer, plus 0.2 * cos * cos * (area per sample) / distance^2 times the colour of the other samples'
    pixels.  The background keeps its colour.  No gradient."""
    is_, d, f, n = _gbuffer(depth, face_ind_buffer, normal_buffer, sample_num, color=(color, 3))
    c = color.detach().float().contiguous()
    out = torch.empty((is_, is_, 3), dtype=torch.float32, device=d.device)
    _lib.call("b200r_ssdo", d.device, c, d, f, n, out, is_, int(sample_num), float(sample_range_r), float(width))
    return out


def FXAA_cuda(texture):
    """FXAA of a [is, is, 3] image (FXAA_cuda.py:3-262), as the reference computes it -> [is, is, 3].

    The reference's edge search never moves (its `uv1 -= offset` calls a free operator that returns a new value), so
    the edge offset is always 0 and each pixel is either kept (a luma range below max(0.0312, 0.125 * max luma)) or
    resampled bilinearly at the sub-pixel offset, up to 0.75 pixel across the edge.  That behaviour is kept; it is not
    textbook FXAA.  No gradient."""
    is_ = _check(texture=(texture, 3))
    t = texture.detach().float().contiguous()
    out = torch.empty_like(t)
    _lib.call("b200r_fxaa", t.device, t, out, is_)
    return out


def conv_for_image(x, w, overflow=0):
    """The k x k image filter of conv.py:5-21: x [H, W] or [H, W, d], w [kh, kw] ->
    y[i, j] = sum_ab w[a, b] * x[i + a - 1, j + b - 1], with `overflow` outside the image.  The anchor is the
    reference's: centred for 3 x 3, shifted towards the bottom right for larger filters (Render.SSAO's 5 x 5, the
    shadow PCF's 7 x 7).  Differentiable with respect to x and w; not a hot path, so it is PyTorch ops."""
    flat = x.dim() == 2
    if flat:
        x = x.unsqueeze(2)
    if x.dim() != 3 or w.dim() != 2:
        raise ValueError("conv_for_image takes x [H, W] or [H, W, d] and w [kh, kw], got %s and %s"
                         % (tuple(x.shape), tuple(w.shape)))
    kh, kw = w.shape
    H, W, _ = x.shape
    # rows i + a - 1 for a < kh: pad 1 above and kh - 2 below (at least 0; a 1-row filter reads row i - 1)
    top, left = 1, 1
    bottom, right = max(kh - 2, 0), max(kw - 2, 0)
    xp = torch.nn.functional.pad(x.permute(2, 0, 1), (left, right, top, bottom), value=float(overflow))
    y = 0
    for a in range(kh):
        for b in range(kw):
            y = y + w[a, b] * xp[:, a:a + H, b:b + W]
    y = y.permute(1, 2, 0)
    return y.squeeze(2) if flat else y
