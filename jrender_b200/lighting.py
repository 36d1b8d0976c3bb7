"""Lighting: the surface-mode path (the renderer's default) runs as ONE fused kernel forward and one backward
(csrc/lighting_api.cu, SURVEY.md section 8f rank 1); everything else is the op-by-op PyTorch mirror below.

Mirrors jrender/renderer/lighting/{ambient_lighting,directional_lighting,lighting}.py for the
paths the rasterizer demos use: ambient + directional light in 'surface' and 'vertex' modes,
including the Cook-Torrance specular branch the reference takes by default
(Mesh.with_specular defaults to True, structures/mesh.py:74).  Normal-mapped meshes
(surface_ResNormals), SSS and the Gbuffer debug modes are not mirrored.
"""
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

    def forward(self, mesh, eyes=None):
        if self.Gbuffer == "albedo":
            return mesh
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
