"""Lighting: the surface-mode path (the renderer's default) runs as ONE fused kernel forward and one backward
(csrc/lighting_api.cu, SURVEY.md section 8f rank 1); everything else is the op-by-op PyTorch mirror below.

Mirrors jrender/renderer/lighting/{ambient_lighting,directional_lighting,lighting}.py for the
paths the rasterizer demos use: ambient + directional light in 'surface' and 'vertex' modes,
including the Cook-Torrance specular branch the reference takes by default
(Mesh.with_specular defaults to True, structures/mesh.py:74).  Normal-mapped meshes (mesh.normal_textures, one normal
per texel from surface_ResNormals) take the surface branch's normal-map path: one fused kernel forward and one backward
(b200r_normal_mapped_lighting_*), or the op-by-op directional_lighting_texels.  Meshes with with_SSS and SoftRas
surface textures take the texture-space subsurface scattering of lighting.py:86-156 (SSS below) on both surface
branches.  The Gbuffer debug modes are not mirrored.
"""
import ctypes as C
import math

import torch
from torch import nn
import torch.nn.functional as F

from . import _lib
from ._lib import _f3
from .transform import _t


def ambient_lighting(light, light_intensity=0.5, light_color=(1, 1, 1)):
    """ambient_lighting.py:4-9."""
    light_color = _t(light_color, light)
    if light_color.dim() == 1:
        light_color = light_color[None, :]
    return light + light_intensity * light_color[:, None, :]


def GGX(N, H, roughness):
    a = roughness * roughness
    a2 = a * a
    NdotH = F.relu(torch.sum(N * H, dim=2))
    NdotH2 = (NdotH * NdotH)[:, :, None]
    denom = (NdotH2 * (a2 - 1.0) + 1.0)
    denom = 3.1415 * denom * denom
    return a2 / denom


def SchlickGGX(NdotV, roughness):
    r = roughness + 1.0
    k = (r * r) / 8.0
    NdotV = NdotV[:, :, None]
    return NdotV / (NdotV * (1.0 - k) + k)


def GeometrySmith(N, V, L, roughness):
    NdotV = F.relu(torch.sum(N * V, dim=2))
    NdotL = F.relu(torch.sum(N * L, dim=2))
    return SchlickGGX(NdotL, roughness) * SchlickGGX(NdotV, roughness)


def fresnelSchlick(cosTheta, F0):
    return F0 + (1.0 - F0) * torch.pow(1.0 - cosTheta, 5)[:, :, None]


def directional_lighting(diffuseLight, specularLight, normals, light_intensity=0.5, light_color=(1, 1, 1),
                         light_direction=(0, 1, 0), positions=None, eye=None, with_specular=False,
                         metallic_textures=None, roughness_textures=None):
    """directional_lighting.py:54-145 for 3-D normals ([B, n, 3])."""
    light_color = _t(light_color, normals)
    light_direction = F.normalize(_t(light_direction, normals), dim=0, eps=1e-12)
    if light_color.dim() == 1:
        light_color = light_color[None, :]
    if light_direction.dim() == 1:
        light_direction = light_direction[None, :]
    cosine = F.relu(torch.sum(normals * light_direction, dim=2))

    if with_specular and metallic_textures is not None and roughness_textures is not None:
        if metallic_textures.dim() == 4:
            total = metallic_textures.shape[2] * 1.0
            metallic_textures = torch.sum(metallic_textures, dim=2) / total
            roughness_textures = torch.sum(roughness_textures, dim=2) / total
        elif metallic_textures.dim() == 6:
            total = metallic_textures.shape[2] * metallic_textures.shape[3] * metallic_textures.shape[4] * 1.0
            metallic_textures = metallic_textures.sum(dim=(2, 3, 4)) / total
            roughness_textures = roughness_textures.sum(dim=(2, 3, 4)) / total

    if with_specular and eye is not None and positions is not None and metallic_textures is not None \
            and roughness_textures is not None:
        eye = _t(eye, normals)
        if eye.dim() == 1:
            eye = eye[None, :]
        if eye.dim() == 2:
            eye = eye[:, None, :]
        N = normals
        V = F.normalize(eye - positions, dim=2, eps=1e-12)
        L = light_direction
        H = F.normalize(V + L, dim=2, eps=1e-12)
        metallic = metallic_textures
        roughness = roughness_textures
        F0 = _t((0.4, 0.4, 0.4), normals)[None, None, :] * (1 - metallic) + _t((1.0, 1.0, 1.0), normals)[None, None, :] * metallic
        radiance = light_intensity * (light_color[:, None, :] * cosine[:, :, None])
        NDF = GGX(N, H, roughness)
        G = GeometrySmith(N, V, L, roughness)
        Fr = fresnelSchlick(F.relu(torch.sum(H * V, dim=2)), F0)
        KD = (1.0 - Fr) * (1.0 - metallic)
        diffuseLight = diffuseLight + KD * radiance
        numerator = NDF * G * Fr
        denominator = (4.0 * F.relu(torch.sum(N * V, dim=2)) * F.relu(torch.sum(N * L, dim=2)))[:, :, None]
        specular = numerator / torch.clamp(denominator, min=0.01)
        specularLight = specularLight + specular * radiance
    else:
        diffuseLight = diffuseLight + light_intensity * (light_color[:, None, :] * cosine[:, :, None])
    return [diffuseLight, specularLight]


def directional_lighting_texels(diffuseLight, specularLight, normals, light_intensity=0.5, light_color=(1, 1, 1),
                                light_direction=(0, 1, 0), positions=None, eye=None, with_specular=False,
                                metallic_textures=None, roughness_textures=None):
    """directional_lighting.py:54-135 for 4-D normals ([B, nf, T, 3], one per texel): reductions over dim 3, positions
    [B, nf, 3] unsqueezed to [B, nf, 1, 3], and the per-texel metallic / roughness [B, nf, T, 1] used as they are."""
    light_color = _t(light_color, normals)
    light_direction = F.normalize(_t(light_direction, normals), dim=0, eps=1e-12)
    if light_color.dim() == 1:
        light_color = light_color[None, :]
    if light_direction.dim() == 1:
        light_direction = light_direction[None, :]
    cosine = F.relu(torch.sum(normals * light_direction, dim=3))
    positions = positions.unsqueeze(2)
    if with_specular and eye is not None and positions is not None and metallic_textures is not None \
            and roughness_textures is not None:
        eye = _t(eye, normals)
        if eye.dim() == 1:
            eye = eye[None, :]
        if eye.dim() == 2:
            eye = eye[:, None, None, :]
        N, L = normals, light_direction
        V = F.normalize(eye - positions, dim=3, eps=1e-12)
        H = F.normalize(V + L, dim=3, eps=1e-12)
        metallic, roughness = metallic_textures, roughness_textures
        F0 = _t((0.4, 0.4, 0.4), normals)[None, None, None, :] * (1 - metallic) + \
            _t((1.0, 1.0, 1.0), normals)[None, None, None, :] * metallic
        radiance = light_intensity * (light_color[:, None, None, :] * cosine[..., None])
        a = roughness * roughness
        a2 = a * a
        NdotH = F.relu(torch.sum(N * H, dim=3))
        denom = (NdotH * NdotH)[..., None] * (a2 - 1.0) + 1.0
        NDF = a2 / (3.1415 * denom * denom)                                              # GGX
        r = roughness + 1.0
        k = (r * r) / 8.0
        NdotV = F.relu(torch.sum(N * V, dim=3))[..., None]
        NdotL = F.relu(torch.sum(N * L, dim=3))[..., None]
        G = (NdotL / (NdotL * (1.0 - k) + k)) * (NdotV / (NdotV * (1.0 - k) + k))        # GeometrySmith
        Fr = F0 + (1.0 - F0) * torch.pow(1.0 - F.relu(torch.sum(H * V, dim=3)), 5)[..., None]
        KD = (1.0 - Fr) * (1.0 - metallic)
        diffuseLight = diffuseLight + KD * radiance
        denominator = (4.0 * F.relu(torch.sum(N * V, dim=3)) * F.relu(torch.sum(N * L, dim=3)))[..., None]
        specularLight = specularLight + (NDF * G * Fr) / torch.clamp(denominator, min=0.01) * radiance
    else:
        diffuseLight = diffuseLight + light_intensity * (light_color[:, None, None, :] * cosine[..., None])
    return [diffuseLight, specularLight]


class _FusedNormalMappedLighting(torch.autograd.Function):
    """clamp(textures * diffuse + specular, 0, 1) with one normal per texel, normalize(n_t . TBN):
    b200r_normal_mapped_lighting_*.  Differentiable w.r.t. vertices (through the face centroid), textures, normal
    textures and the per-texel metallic / roughness; not w.r.t. the TBN."""

    @staticmethod
    def forward(ctx, vertices, textures, normal_textures, metallic, roughness, faces, tbn, eye, params):
        v, tx, nt = vertices.contiguous(), textures.contiguous(), normal_textures.contiguous()
        B, nf, T = tx.shape[0], tx.shape[1], tx.shape[2]
        out = torch.empty_like(tx)
        amb_i, amb_c, dir_i, dir_c, direction, with_spec = params
        args = (B, v.shape[0], faces.shape[0], 0 if eye is None else eye.shape[0], nt.shape[0], nt.shape[1], nt.shape[2],
                tbn.shape[0], tbn.shape[1], v.shape[1], nf, T, float(amb_i), _f3(amb_c), float(dir_i), _f3(dir_c),
                _f3(direction), int(bool(with_spec)))
        _lib.call("b200r_normal_mapped_lighting_forward", v.device, v, faces, tx, nt, tbn, metallic, roughness, eye, out, *args)
        ctx.save_for_backward(v, tx, nt, metallic, roughness, faces, tbn, eye)
        ctx.args = args
        return out

    @staticmethod
    def backward(ctx, grad_out):
        v, tx, nt, metallic, roughness, faces, tbn, eye = ctx.saved_tensors
        need = ctx.needs_input_grad
        gv = torch.empty_like(v) if need[0] else None
        gt = torch.empty_like(tx) if need[1] else None
        gn = torch.empty_like(nt) if need[2] else None
        gm = torch.empty_like(metallic) if need[3] else None
        gr = torch.empty_like(roughness) if need[4] else None
        _lib.call("b200r_normal_mapped_lighting_backward", v.device, v, faces, tx, nt, tbn, metallic, roughness, eye,
                  grad_out.contiguous(), gt, gn, gv, gm, gr, *ctx.args)
        return gv, gt, gn, gm, gr, None, None, None, None


class _FusedSurfaceLighting(torch.autograd.Function):
    """clamp(textures * diffuse + specular, 0, 1) with diffuse / specular from the face normals: b200r_surface_lighting_*.
    Differentiable w.r.t. vertices, textures, and metallic / roughness (through each face's mean material value)."""

    @staticmethod
    def forward(ctx, vertices, textures, faces, metallic, roughness, eye, params):
        v = vertices.contiguous()
        tx = textures.contiguous()
        B, nf = tx.shape[0], tx.shape[1]
        T = tx[0, 0].numel() // 3
        Tm = 0 if metallic is None else metallic[0, 0].numel()
        out = torch.empty_like(tx)
        amb_i, amb_c, dir_i, dir_c, direction, with_spec = params
        args = (B, v.shape[0], faces.shape[0], 0 if eye is None else eye.shape[0], v.shape[1], nf, T, Tm,
                float(amb_i), _f3(amb_c), float(dir_i), _f3(dir_c), _f3(direction), int(bool(with_spec)))
        _lib.call("b200r_surface_lighting_forward", v.device, v, faces, tx, metallic, roughness, eye, out, *args)
        ctx.save_for_backward(v, tx, faces, metallic, roughness, eye)
        ctx.args = args
        return out

    @staticmethod
    def backward(ctx, grad_out):
        v, tx, faces, metallic, roughness, eye = ctx.saved_tensors
        g = grad_out.contiguous()
        gt = torch.empty_like(tx)
        gv = torch.empty_like(v) if ctx.needs_input_grad[0] else None
        gm = torch.empty_like(metallic) if ctx.needs_input_grad[3] else None
        gr = torch.empty_like(roughness) if ctx.needs_input_grad[4] else None
        _lib.call("b200r_surface_lighting_backward", v.device, v, faces, tx, metallic, roughness, eye, g, gt, gv, gm, gr, *ctx.args)
        return gv, (gt if ctx.needs_input_grad[1] else None), None, gm, gr, None, None


def _normalized_direction(d):
    """F.normalize(light_direction, dim=0, eps=1e-12) on the host, in float32 like the mirror."""
    t = torch.tensor([float(x) for x in (d.detach().cpu().tolist() if isinstance(d, torch.Tensor) else d)], dtype=torch.float32)
    return F.normalize(t, dim=0, eps=1e-12).tolist()


SSS_IMAGE_SIZE = 2048                                             # lighting.py:90
SSS_TAP_NUM = 7                                                   # :117
SSS_GAUSSIAN_BASIS = (0, 25, 100, 400)                            # :113: levels of variance 25, 75 and 300
SSS_WEIGHTS = ((0.7, 0.2, 0.1), (0.1, 0.2, 0.7), (0.1, 0.2, 0.7))  # :123-126, [channel][level]


def _sss_taps(v, tap_num=SSS_TAP_NUM):
    """gaussian_blur.py:7-13: the tap weights Gauss[i] = sqrt(v) N(v; -sqrt(v)(3 - i)) in Python doubles, and GaussWidth
    = sqrt(v); both are stored as float32 by the caller."""
    width = math.sqrt(v)
    g1 = lambda r: math.exp(-r ** 2 / (2 * v)) / math.sqrt(2 * math.pi * v)
    return [width * g1(-width * ((tap_num - 1) / 2 - i)) for i in range(tap_num)], width


def _sss_maps(diffuseLight, specular, mesh):
    """lighting.py:88-106: the world-coordinate, irradiance and specular maps of SSS, each the [1, 4, S, S] output of
    one texture-space SoftRas forward (the face UVs as positions); the kernels read their first three planes as the
    reference's [S, S, 3] maps."""
    from .softras import SoftRasterizeFunction
    dev = mesh.textures.device
    irradiance = torch.sqrt(mesh.textures * diffuseLight)
    rasterize = SoftRasterizeFunction(image_size=SSS_IMAGE_SIZE, background_color=[0, 0, 0], near=1, far=100, fill_back=True,
                                      eps=1e-5, sigma_val=1e-5, dist_func='barycentric', dist_eps=1e-5,
                                      gamma_val=1e-4, aggr_func_rgb='hard', aggr_func_alpha='prod',
                                      texture_type='surface')
    # [1, nf, 3, 3] as three texels per face in the reference (:97); its SoftRas samples a surface texture of T texels
    # at resolution int(sqrt(T)) = 1, i.e. texel 0 (soft_rasterize.py:157-166), so every pixel of a face takes vertex 0's
    # position and the map is flat over each face.  Passing that texel alone rasterizes the same map.
    worldcoord_textures = ((mesh.face_vertices + 1) / 2 * 255.)[:, :, :1]
    coords = (mesh.face_texcoords.to(dev, torch.float32) - 0.5) * 2
    coords = torch.cat([coords, torch.full(tuple(coords.shape[:3]) + (1,), 1.5, dtype=torch.float32, device=dev)], dim=3)
    world_map = rasterize(coords, worldcoord_textures)
    irradiance_map = rasterize(coords, irradiance)
    specular_map = rasterize(coords, specular)
    return world_map, irradiance_map, specular_map


def _sss_levels():
    """The host arrays of the blur pyramid: (taps [L][7], tap widths [L], weights [3][L], L) as ctypes float arrays."""
    variances = [SSS_GAUSSIAN_BASIS[i + 1] - SSS_GAUSSIAN_BASIS[i] for i in range(len(SSS_GAUSSIAN_BASIS) - 1)]
    L = len(variances)
    taps, widths = zip(*[_sss_taps(v) for v in variances])
    return ((C.c_float * (L * SSS_TAP_NUM))(*[t for level in taps for t in level]), (C.c_float * L)(*widths),
            (C.c_float * (3 * L))(*[w for channel in SSS_WEIGHTS for w in channel]), L)


def _map_grad(like):
    """A gradient for a [1, 4, S, S] SoftRas map whose first three planes a kernel overwrites: the alpha plane is 0."""
    g = torch.empty_like(like)
    g[:, 3].zero_()
    return g


class _SSSStretch(torch.autograd.Function):
    """b200r_sss_stretch / _backward: the world-coordinate map [1, 4, S, S] -> the clamped stretch maps (u, v) [S, S]."""

    @staticmethod
    def forward(ctx, world_map):
        S = world_map.shape[-1]
        su = torch.empty((S, S), dtype=torch.float32, device=world_map.device)
        sv = torch.empty_like(su)
        _lib.call("b200r_sss_stretch", world_map.device, world_map, su, sv, S, S)
        ctx.save_for_backward(world_map)
        return su, sv

    @staticmethod
    def backward(ctx, gu, gv):
        world_map, = ctx.saved_tensors
        S = world_map.shape[-1]
        gw = _map_grad(world_map)
        _lib.call("b200r_sss_stretch_backward", world_map.device, world_map, gu.contiguous(), gv.contiguous(), gw, S, S)
        return gw


class _SSSPyramid(torch.autograd.Function):
    """b200r_sss_blur_pyramid / _backward: (stretch u, v [S, S], irradiance and specular maps [1, 4, S, S]) -> the
    composed map [S, S, 3], rows flipped."""

    @staticmethod
    def forward(ctx, stretch_u, stretch_v, irradiance_map, specular_map):
        dev, S = stretch_u.device, stretch_u.shape[-1]
        taps, widths, weights, L = _sss_levels()
        nbytes = _lib.lib().b200r_sss_workspace_bytes(S, S)
        workspace = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        final_map = torch.empty((S, S, 3), dtype=torch.float32, device=dev)
        _lib.call("b200r_sss_blur_pyramid", dev, stretch_u, stretch_v, irradiance_map, specular_map, final_map, workspace,
                  nbytes, taps, widths, weights, L, S, S)
        ctx.save_for_backward(stretch_u, stretch_v, irradiance_map)
        return final_map

    @staticmethod
    def backward(ctx, g):
        su, sv, irr = ctx.saved_tensors
        dev, S = su.device, su.shape[-1]
        taps, widths, weights, L = _sss_levels()
        stretch = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        gsu = torch.empty_like(su) if stretch else None
        gsv = torch.empty_like(sv) if stretch else None
        girr, gspec = _map_grad(irr), _map_grad(irr)
        nbytes = _lib.lib().b200r_sss_backward_workspace_bytes(S, S, L)
        workspace = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        _lib.call("b200r_sss_blur_pyramid_backward", dev, su, sv, irr, g.contiguous(), girr, gspec, gsu, gsv, workspace,
                  nbytes, taps, widths, weights, L, S, S)
        return gsu, gsv, girr, gspec


class _SSSBake(torch.autograd.Function):
    """b200r_bake_textures_softras / _backward on the composed map [S, S, 3]: every face's R*R texels, [nf, R*R, 3]."""

    @staticmethod
    def forward(ctx, final_map, faces_uv, R):
        dev, nf = final_map.device, faces_uv.shape[0]
        upd = torch.ones((nf,), dtype=torch.int32, device=dev)
        out = torch.ones((nf, R * R, 3), dtype=torch.float32, device=dev)
        _lib.call("b200r_bake_textures_softras", dev, final_map, faces_uv, upd, out, nf, R, final_map.shape[0],
                  final_map.shape[1])
        ctx.save_for_backward(faces_uv, upd)
        ctx.R, ctx.shape = R, final_map.shape
        return out

    @staticmethod
    def backward(ctx, g):
        faces_uv, upd = ctx.saved_tensors
        gmap = torch.empty(ctx.shape, dtype=torch.float32, device=g.device)
        _lib.call("b200r_bake_textures_softras_backward", g.device, g.contiguous(), faces_uv, upd, gmap, faces_uv.shape[0],
                  ctx.R, ctx.shape[0], ctx.shape[1])
        return gmap, None, None


def SSS(diffuseLight, specular, mesh, grad=False):
    """Texture-space subsurface scattering, lighting.py:86-156: the mesh's textures [1, nf, R*R, 3] lit by diffuseLight
    and specular ([1, nf, 1, 3] per face, or [1, nf, R*R, 3] per texel), returned as new textures [1, nf, R*R, 3]
    (unclamped; Lighting clamps them).

    sqrt(textures * diffuse), the world coordinates (face_vertices + 1) / 2 * 255 and the specular light are rasterized
    into the 2048^2 texture space (the face UVs as positions) by the SoftRas forward; b200r_sss_stretch turns the world
    coordinate map into the clamped stretch maps; b200r_sss_blur_pyramid blurs the irradiance over three levels, modulated
    by the stretch, and composes `sum_k w_k blur_k * irradiance + specular`; the bake samples that map back into textures.

    With grad=False (the default), as in the reference, gradients stop here: the result does not require grad.  With
    grad=True and grad mode on, the result carries a graph to textures, diffuseLight, specular and the mesh's
    face_vertices (through the world-coordinate and stretch maps), through the backward kernels of each stage and the
    SoftRas backward of the three texture-space rasterizations; the values are the same bits either way.  The gradient
    of sqrt(textures * diffuse) is infinite where the product is 0, as torch's own: keep fitted textures away from 0.
    Nothing flows to face_texcoords, which must not require grad then (ValueError).

    The batch must be 1, the mesh must carry face_texcoords, and its textures must hold texture_res^2 texels per face
    (ValueError otherwise)."""
    from . import io
    tx = mesh.textures
    if tx.dim() != 4 or tx.shape[0] != 1:
        raise ValueError("SSS: needs a batch of one mesh with SoftRas surface textures [1, nf, T, 3], got %s"
                         % (tuple(tx.shape),))
    ftc = mesh.face_texcoords
    if ftc is None:
        raise ValueError("SSS: the mesh has no face_texcoords (load it with Mesh.from_obj(..., load_texture=True))")
    nf, T, R = tx.shape[1], tx.shape[2], int(mesh.texture_res)
    if T != R * R:
        raise ValueError("SSS: %d texels per face, texture_res %d needs %d" % (T, R, R * R))
    if tuple(ftc.shape) != (1, nf, 3, 2):
        raise ValueError("SSS: face_texcoords %s do not match %d faces" % (tuple(ftc.shape), nf))
    dev = tx.device
    S = SSS_IMAGE_SIZE
    if grad and torch.is_grad_enabled():
        if ftc.requires_grad:
            raise ValueError("SSS: face_texcoords require grad, but no gradient flows to them")
        if any(t.requires_grad for t in (diffuseLight, specular, tx, mesh.face_vertices)):
            world_map, irradiance_map, specular_map = _sss_maps(diffuseLight, specular, mesh)
            stretch_u, stretch_v = _SSSStretch.apply(world_map)
            final_map = _SSSPyramid.apply(stretch_u, stretch_v, irradiance_map, specular_map)
            return _SSSBake.apply(final_map, ftc[0].to(dev, torch.float32).contiguous(), R)[None]
    with torch.no_grad():
        world_map, irradiance_map, specular_map = _sss_maps(diffuseLight, specular, mesh)
        stretch_u = torch.empty((S, S), dtype=torch.float32, device=dev)
        stretch_v = torch.empty_like(stretch_u)
        _lib.call("b200r_sss_stretch", dev, world_map, stretch_u, stretch_v, S, S)
        taps, widths, weights, L = _sss_levels()
        nbytes = _lib.lib().b200r_sss_workspace_bytes(S, S)
        workspace = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        final_map = torch.empty((S, S, 3), dtype=torch.float32, device=dev)
        _lib.call("b200r_sss_blur_pyramid", dev, stretch_u, stretch_v, irradiance_map, specular_map, final_map, workspace,
                  nbytes, taps, widths, weights, L, S, S)
        final = io.bake_textures_for_softras(final_map, ftc[0], torch.ones((nf, R * R, 3), dtype=torch.float32, device=dev),
                                             torch.ones((nf,), dtype=torch.int32, device=dev), device=dev)
    return final[None]


class AmbientLighting(nn.Module):
    def __init__(self, light_intensity=0.5, light_color=(1, 1, 1)):
        super(AmbientLighting, self).__init__()
        self.light_intensity = light_intensity
        self.light_color = light_color

    def forward(self, light):
        return ambient_lighting(light, self.light_intensity, self.light_color)

    execute = forward


class DirectionalLighting(nn.Module):
    def __init__(self, light_intensity=0.5, light_color=(1, 1, 1), light_direction=(0, 1, 0)):
        super(DirectionalLighting, self).__init__()
        self.light_intensity = light_intensity
        self.light_color = light_color
        self.light_direction = light_direction

    def forward(self, diffuseLight, specularLight, normals, positions=None, eye=None, with_specular=False,
                metallic_textures=None, roughness_textures=None):
        return directional_lighting(diffuseLight, specularLight, normals, self.light_intensity, self.light_color,
                                    self.light_direction, positions, eye, with_specular, metallic_textures,
                                    roughness_textures)

    execute = forward


class Lighting(nn.Module):
    """lighting.py:159-223."""

    def __init__(self, light_mode='surface',
                 intensity_ambient=0.5, color_ambient=[1, 1, 1],
                 intensity_directionals=0.5, color_directionals=[1, 1, 1],
                 directions=[0, 1, 0], Gbuffer='None', transform=None):
        super(Lighting, self).__init__()
        if light_mode not in ['surface', 'vertex']:
            raise ValueError('Lighting mode only support surface and vertex')
        if Gbuffer not in ('None', None, 'albedo'):
            raise NotImplementedError("Gbuffer=%r (render2 debug outputs) is outside this repo's scope" % (Gbuffer,))
        self.Gbuffer = Gbuffer
        self.transform = transform
        self.light_mode = light_mode
        self.ambient = AmbientLighting(intensity_ambient, color_ambient)
        self.directionals = nn.ModuleList([DirectionalLighting(intensity_directionals, color_directionals, directions)])

    fused = True   # CUDA float32 surface-mode inputs take the one-launch kernel (b200r_surface_lighting_forward)
    sss_grad = False   # with_SSS meshes: differentiate SSS (SSS(..., grad=True)); off, its result carries no graph

    def _fusable(self, mesh, eyes):
        tx, v = mesh.textures, mesh.vertices
        if not (self.fused and len(self.directionals) == 1 and tx.is_cuda and v.is_cuda and tx.device == v.device):
            return False
        if tx.dtype != torch.float32 or v.dtype != torch.float32 or tx.dim() not in (4, 6) or tx.shape[-1] != 3:
            return False
        if mesh.faces.device != v.device or mesh.faces.dim() != 3 or mesh.faces.shape[1] != tx.shape[1]:
            return False
        d = self.directionals[0]
        for c in (self.ambient.light_color, d.light_color, d.light_direction):
            n = c.numel() if isinstance(c, torch.Tensor) else len(c)
            if n != 3:   # per-batch light colours / directions: op-by-op path
                return False
        for t in (mesh.metallic_textures, mesh.roughness_textures):
            if t is not None and (t.device != v.device or t.dtype != torch.float32
                                  or t.shape[:2] != tx.shape[:2] or t.shape[-1] != 1):
                return False
        if isinstance(eyes, torch.Tensor) and eyes.requires_grad:
            return False
        return True

    def _fused_surface(self, mesh, eyes):
        v = mesh.vertices
        d = self.directionals[0]
        eye = None
        spec = bool(mesh.with_specular) and eyes is not None and mesh.metallic_textures is not None and mesh.roughness_textures is not None
        if spec:
            eye = _t(eyes, v).reshape(-1, 3).contiguous()
            if eye.shape[0] not in (1, mesh.textures.shape[0]):
                return None
        faces = mesh.faces if mesh.faces.dtype == torch.int32 else mesh.faces.int()
        params = (self.ambient.light_intensity, self.ambient.light_color, d.light_intensity, d.light_color,
                  _normalized_direction(d.light_direction), spec)
        return _FusedSurfaceLighting.apply(v, mesh.textures, faces.contiguous(),
                                           mesh.metallic_textures.contiguous() if spec else None,
                                           mesh.roughness_textures.contiguous() if spec else None, eye, params)

    def _check_normal_map(self, mesh):
        tx, nt, tbn = mesh.textures, mesh.normal_textures, mesh.TBN
        if tx.dim() != 4:
            raise ValueError("Lighting: a normal map needs SoftRas surface textures [B, nf, T, 3], got %s"
                             % (tuple(tx.shape),))
        if nt.dim() != 4 or tuple(nt.shape[1:]) != tuple(tx.shape[1:]) or tbn is None or tbn.dim() != 4 \
                or tuple(tbn.shape[1:]) != (tx.shape[1], 3, 3):
            raise ValueError("Lighting: normal_textures %s / TBN %s do not match textures %s"
                             % (tuple(nt.shape), None if tbn is None else tuple(tbn.shape), tuple(tx.shape)))

    def _fused_normal_mapped(self, mesh, eyes):
        """The normal-map branch in one launch, or None where it must run op by op: anything _fusable rejects, an eye or
        TBN that requires grad, or tensors the kernel does not take (dtype, device, batch, material texel count)."""
        if not self._fusable(mesh, eyes):
            return None
        v, tx, nt, tbn = mesh.vertices, mesh.textures, mesh.normal_textures, mesh.TBN
        B, nf, T = tx.shape[:3]
        for x in (nt, tbn):
            if x.dtype != torch.float32 or x.device != v.device or x.shape[0] not in (1, B):
                return None
        if tbn.requires_grad:
            return None
        d = self.directionals[0]
        spec = bool(mesh.with_specular) and eyes is not None and mesh.metallic_textures is not None \
            and mesh.roughness_textures is not None
        eye = met = rou = None
        if spec:
            eye = _t(eyes, v).reshape(-1, 3).contiguous()
            if eye.shape[0] not in (1, B):
                return None
            if mesh.metallic_textures.shape[2] not in (1, T) or mesh.roughness_textures.shape[2] not in (1, T):
                return None
            met = mesh.metallic_textures.expand(B, nf, T, 1).contiguous()   # a per-face value broadcasts over the texels
            rou = mesh.roughness_textures.expand(B, nf, T, 1).contiguous()
        faces = mesh.faces if mesh.faces.dtype == torch.int32 else mesh.faces.int()
        params = (self.ambient.light_intensity, self.ambient.light_color, d.light_intensity, d.light_color,
                  _normalized_direction(d.light_direction), spec)
        return _FusedNormalMappedLighting.apply(v, tx, nt, met, rou, faces.contiguous(), tbn.contiguous(), eye, params)

    def _normal_mapped(self, mesh, eyes):
        """lighting.py:186-192 and 200-201: the surface branch with mesh.normal_textures."""
        self._check_normal_map(mesh)
        lit = self._fused_normal_mapped(mesh, eyes)
        if lit is None:
            diffuseLight = torch.zeros(mesh.textures.shape, dtype=mesh.textures.dtype, device=mesh.vertices.device)
            specularLight = torch.zeros_like(diffuseLight)
            diffuseLight = self.ambient(diffuseLight)
            for d in self.directionals:
                diffuseLight, specularLight = directional_lighting_texels(
                    diffuseLight, specularLight, mesh.surface_ResNormals, d.light_intensity, d.light_color,
                    d.light_direction, torch.sum(mesh.face_vertices, dim=2) / 3.0, eyes, mesh.with_specular,
                    mesh.metallic_textures, mesh.roughness_textures)
            lit = torch.clamp(mesh.textures * diffuseLight + torch.ones_like(mesh.textures) * specularLight, 0.0, 1.0)
        mesh.textures = lit
        return mesh

    def _subsurface(self, mesh, eyes):
        """lighting.py:182-201 with mesh.with_SSS and 4-D textures: the op-by-op diffuse and specular light of either
        surface branch (per face, or per texel with a normal map), then clamp(SSS(diffuse, specular, mesh), 0, 1)."""
        if mesh.normal_textures is not None:
            self._check_normal_map(mesh)
            diffuseLight = torch.zeros(mesh.textures.shape, dtype=mesh.textures.dtype, device=mesh.vertices.device)
            specularLight = torch.zeros_like(diffuseLight)
            diffuseLight = self.ambient(diffuseLight)
            for d in self.directionals:
                diffuseLight, specularLight = directional_lighting_texels(
                    diffuseLight, specularLight, mesh.surface_ResNormals, d.light_intensity, d.light_color,
                    d.light_direction, torch.sum(mesh.face_vertices, dim=2) / 3.0, eyes, mesh.with_specular,
                    mesh.metallic_textures, mesh.roughness_textures)
        else:
            diffuseLight = torch.zeros(mesh.faces.shape, dtype=torch.float32, device=mesh.vertices.device)
            specularLight = torch.zeros_like(diffuseLight)
            diffuseLight = self.ambient(diffuseLight)
            for directional in self.directionals:
                diffuseLight, specularLight = directional(
                    diffuseLight, specularLight, mesh.surface_normals, torch.sum(mesh.face_vertices, dim=2) / 3.0, eyes,
                    mesh.with_specular, mesh.metallic_textures, mesh.roughness_textures)
            diffuseLight = diffuseLight[:, :, None, :]
            specularLight = specularLight[:, :, None, :]
        mesh.textures = torch.clamp(SSS(diffuseLight, specularLight, mesh, grad=self.sss_grad), 0.0, 1.0)
        return mesh

    def forward(self, mesh, eyes=None):
        if self.Gbuffer == "albedo":
            return mesh
        if self.light_mode == 'surface' and mesh.with_SSS and mesh.textures.dim() == 4:
            return self._subsurface(mesh, eyes)
        if self.light_mode == 'surface' and mesh.normal_textures is not None:
            return self._normal_mapped(mesh, eyes)
        if self.light_mode == 'surface' and self._fusable(mesh, eyes):
            lit = self._fused_surface(mesh, eyes)
            if lit is not None:
                mesh.textures = lit
                return mesh
        if self.light_mode == 'surface':
            diffuseLight = torch.zeros(mesh.faces.shape, dtype=torch.float32, device=mesh.vertices.device)
            specularLight = torch.zeros_like(diffuseLight)
            diffuseLight = self.ambient(diffuseLight)
            for directional in self.directionals:
                diffuseLight, specularLight = directional(
                    diffuseLight, specularLight, mesh.surface_normals, torch.sum(mesh.face_vertices, dim=2) / 3.0, eyes,
                    mesh.with_specular, mesh.metallic_textures, mesh.roughness_textures)
            diffuseLight = diffuseLight[:, :, None, :]
            specularLight = specularLight[:, :, None, :]
            if mesh.textures.dim() == 4:
                mesh.textures = torch.clamp(mesh.textures * diffuseLight + torch.ones_like(mesh.textures) * specularLight, 0.0, 1.0)
            elif mesh.textures.dim() == 6:
                mesh.textures = torch.clamp(mesh.textures * diffuseLight[:, :, :, None, None, :] +
                                            torch.ones_like(mesh.textures) * specularLight[:, :, :, None, None, :], 0.0, 1.0)
        elif self.light_mode == 'vertex':
            diffuseLight = torch.zeros(mesh.vertices.shape, dtype=torch.float32, device=mesh.vertices.device)
            specularLight = torch.zeros_like(diffuseLight)
            diffuseLight = self.ambient(diffuseLight)
            for directional in self.directionals:
                diffuseLight, specularLight = directional(
                    diffuseLight, specularLight, mesh.vertex_normals, mesh.vertices, eyes,
                    mesh.with_specular, mesh.metallic_textures, mesh.roughness_textures)
            # The reference only applies vertex lighting to 4-D / 6-D textures (lighting.py:214-220);
            # the documented vertex texture shape [B, nv, 3] therefore passes through unlit.
            if mesh.textures.dim() == 4:
                mesh.textures = torch.clamp(mesh.textures * diffuseLight[:, :, None, :] +
                                            torch.ones_like(mesh.textures) * specularLight[:, :, None, :], 0.0, 1.0)
            elif mesh.textures.dim() == 6:
                mesh.textures = torch.clamp(mesh.textures * diffuseLight[:, :, None, None, None, :] +
                                            torch.ones_like(mesh.textures) * specularLight[:, :, None, None, None, :], 0.0, 1.0)
        return mesh

    execute = forward
