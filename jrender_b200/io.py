"""OBJ / MTL loading and texture baking, and the textured OBJ export (load-time; SURVEY.md section 8f rank 3).

Mirrors, for the SoftRas loader:
  jrender/io/load_obj.py:9-20
  jrender/io/utils/_load_obj_for_softras.py:19-207   (OBJ fan triangulation, MTL Kd / map_Kd)
  jrender/io/utils/load_textures.py:3-101            (bilinear bake of the image into R*R texels
                                                      per face -- a CUDA kernel in the reference,
                                                      restated here in numpy because it runs once
                                                      per mesh, not per frame)
and for the NMR loader (dr_type='n3mr'):
  jrender/io/utils/_load_obj_for_n3mr.py:11-155      (same parsing; [nf, ts, ts, ts, 3] textures, default colour 0.5)
  jrender/io/utils/load_textures.py:103-246          (the ts^3 bake with texture wrapping modes -> b200r_bake_textures_n3mr)
and for the export:
  jrender/io/save_obj.py:7-84                        (.obj / .mtl / .png writer; the texture atlas is painted by
                                                      b200r_texture_atlas_softras / _n3mr <- io/utils/create_texture_image.py)
Images are read and written with OpenCV (the reference uses skimage, which is not installed here).
Normal / bump maps and TBN (SSS, render2) are outside the hot-path scope.
"""
import os

import numpy as np
import torch

from . import _lib


def _gpu(what, device):
    """The CUDA device a GPU-only step runs on: `device`, or the current one.  Raises when there is no GPU."""
    if not torch.cuda.is_available():
        raise _lib.B200RasterError("%s runs on the GPU; there is no CPU fallback" % what)
    return torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())


def _placed(x, dev, dtype=torch.float32):
    """x (numpy array or tensor) as a contiguous `dtype` tensor on `dev`."""
    t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))
    return t.to(device=dev, dtype=dtype).contiguous()


def load_mtl(filename_mtl):
    """_load_obj_for_softras.py:19-40: Kd colours and map_Kd filenames per material."""
    texture_filenames, colors, material_name = {}, {}, ''
    with open(filename_mtl) as f:
        for line in f.readlines():
            s = line.split()
            if len(s) == 0:
                continue
            if s[0] == 'newmtl':
                material_name = s[1]
            if s[0] == 'map_Kd':
                texture_filenames[material_name] = s[1]
            if s[0] == 'Kd':
                colors[material_name] = np.array(list(map(float, s[1:4])))
    return colors, texture_filenames


def _imread_rgb01(path):
    import cv2
    img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if img is None:
        raise IOError("cannot read texture image %s" % path)
    if img.ndim == 2:
        img = np.stack((img,) * 3, -1)
    else:
        img = img[:, :, :3][:, :, ::-1]   # BGR(A) -> RGB, drop alpha like the reference
    return img.astype(np.float32) / 255.


def bake_textures_for_softras(image, faces_uv, textures, is_update, device=None):
    """_load_textures_for_softras (load_textures.py:3-101) through the CUDA kernel b200r_bake_textures_softras.

    image [H,W,3] (already flipped vertically by the caller), faces_uv [nf,3,2], textures [nf,R*R,3], is_update [nf]:
    numpy arrays or tensors; returns a CUDA float32 tensor [nf,R*R,3] (updated where is_update != 0).
    There is no CPU implementation in the product (oracle/bake.py is the checker)."""
    dev = _gpu("texture baking (b200r_bake_textures_softras)", device)
    img, uv, upd = _placed(image, dev), _placed(faces_uv, dev), _placed(is_update, dev, torch.int32)
    out = _placed(textures, dev).clone()
    nf, T = out.shape[:2]
    R = int(round(float(np.sqrt(T))))
    if R * R != T or uv.shape != (nf, 3, 2) or img.dim() != 3 or img.shape[2] != 3 or upd.shape != (nf,):
        raise ValueError("bake_textures_for_softras: image [H,W,3], faces_uv [nf,3,2], textures [nf,R*R,3], is_update [nf]")
    _lib.call("b200r_bake_textures_softras", dev, img, uv, upd, out, nf, R, img.shape[0], img.shape[1])
    return out


TEXTURE_WRAPPING = {'REPEAT': 0, 'MIRRORED_REPEAT': 1, 'CLAMP_TO_EDGE': 2, 'CLAMP_TO_BORDER': 3}   # _load_obj_for_n3mr.py:7-8


def bake_textures_for_n3mr(image, faces_uv, textures, is_update, texture_wrapping=0, use_bilinear=True, device=None):
    """_load_textures_for_n3mr (load_textures.py:103-246) through the CUDA kernel b200r_bake_textures_n3mr.

    image [H,W,3] (already flipped vertically by the caller), faces_uv [nf,3,2], textures [nf,ts,ts,ts,3], is_update [nf];
    texture_wrapping 0..3 (TEXTURE_WRAPPING) or its name.  Returns a CUDA float32 tensor [nf,ts,ts,ts,3], updated where
    is_update != 0.  No CPU implementation in the product (oracle/bake.py is the checker)."""
    dev = _gpu("texture baking (b200r_bake_textures_n3mr)", device)
    wrap = TEXTURE_WRAPPING[texture_wrapping] if isinstance(texture_wrapping, str) else int(texture_wrapping)
    img, uv, upd = _placed(image, dev), _placed(faces_uv, dev), _placed(is_update, dev, torch.int32)
    out = _placed(textures, dev).clone()
    if out.dim() != 5 or out.shape[1] != out.shape[2] or out.shape[1] != out.shape[3] or out.shape[4] != 3:
        raise ValueError("bake_textures_for_n3mr: textures must be [nf,ts,ts,ts,3]")
    nf, ts = out.shape[0], out.shape[1]
    if uv.shape != (nf, 3, 2) or img.dim() != 3 or img.shape[2] != 3 or upd.shape != (nf,):
        raise ValueError("bake_textures_for_n3mr: image [H,W,3], faces_uv [nf,3,2], textures [nf,ts,ts,ts,3], is_update [nf]")
    _lib.call("b200r_bake_textures_n3mr", dev, img, uv, upd, out, nf, ts, img.shape[0], img.shape[1], wrap,
              1 if use_bilinear else 0)
    return out


def _parse_texture_faces(filename_obj):
    """UV triangles (fan triangulation, 0 for a missing vt index) and the material of every face
    (_load_obj_for_softras.py:43-83 == _load_obj_for_n3mr.py:30-68)."""
    with open(filename_obj) as f:
        lines = f.readlines()
    vt = [[float(v) for v in line.split()[1:3]] for line in lines if len(line.split()) and line.split()[0] == 'vt']
    faces, material_names, material_name = [], [], ''
    for line in lines:
        s = line.split()
        if len(s) == 0:
            continue
        if s[0] == 'f':
            vs = s[1:]

            def ti(tok):
                return int(tok.split('/')[1]) if ('/' in tok and '//' not in tok) else 0
            v0 = ti(vs[0])
            for i in range(len(vs) - 2):
                faces.append((v0, ti(vs[i + 1]), ti(vs[i + 2])))
                material_names.append(material_name)
        if s[0] == 'usemtl':
            material_name = s[1]
    vt = np.vstack(vt).astype(np.float32)
    faces_uv = vt[np.vstack(faces).astype(np.int32) - 1]
    return faces_uv, material_names


def load_textures_n3mr(filename_obj, filename_mtl, texture_res, texture_wrapping='REPEAT', use_bilinear=True):
    """_load_obj_for_n3mr.py:29-103: [nf, ts, ts, ts, 3] float32; faces without a material keep 0.5, Kd colours are
    broadcast over the ts^3 texels, map_Kd images are baked by b200r_bake_textures_n3mr."""
    faces_uv, material_names = _parse_texture_faces(filename_obj)
    colors, texture_filenames = load_mtl(filename_mtl)
    textures = np.full((faces_uv.shape[0], 3), 0.5, np.float32)
    names = np.array(material_names)
    for material_name, color in colors.items():
        textures[names == material_name] = color
    ts = int(texture_res)
    textures = np.ascontiguousarray(np.broadcast_to(textures[:, None, None, None, :], (faces_uv.shape[0], ts, ts, ts, 3)), dtype=np.float32)
    if ts < 2 and texture_filenames:
        # The reference's kernel divides by (texture_size - 1.): with Mesh.from_obj's default texture_res = 1 every sample
        # point is 0 / 0 and the baked texels are garbage (demo4-optim_textures.py loads the cow this way and then replaces
        # the textures).  Here the material colours are kept and the image is not sampled.
        import warnings
        warnings.warn("load_obj(dr_type='n3mr', texture_res=1): one texel per face cannot be sampled from the texture image "
                      "(the reference divides by texture_res - 1); material colours kept, use texture_res >= 2 to bake")
        return textures
    for material_name, filename_texture in texture_filenames.items():
        image = _imread_rgb01(os.path.join(os.path.dirname(filename_obj), filename_texture))[::-1, :, :]
        textures = bake_textures_for_n3mr(np.ascontiguousarray(image), faces_uv, textures, (names == material_name).astype(np.int32),
                                          TEXTURE_WRAPPING[texture_wrapping], use_bilinear)
    if isinstance(textures, torch.Tensor):
        textures = textures.cpu().numpy()
    return textures


def load_textures(filename_obj, filename_mtl, texture_res):
    """_load_obj_for_softras.py:43-140 without the normal-map branch: [nf, R*R, 3] float32."""
    faces_uv, material_names = _parse_texture_faces(filename_obj)
    colors, texture_filenames = load_mtl(filename_mtl)
    textures = np.ones((faces_uv.shape[0], 3), np.float32)
    names = np.array(material_names)
    for material_name, color in colors.items():
        textures[names == material_name] = color
    textures = np.repeat(textures[:, None, :], texture_res ** 2, axis=1).astype(np.float32)
    for material_name, filename_texture in texture_filenames.items():
        image = _imread_rgb01(os.path.join(os.path.dirname(filename_obj), filename_texture))[::-1, :, :]
        textures = bake_textures_for_softras(np.ascontiguousarray(image), faces_uv, textures, (names == material_name).astype(np.int32))
    if isinstance(textures, torch.Tensor):   # baked on the GPU; loaders hand back host arrays like the geometry
        textures = textures.cpu().numpy()
    return textures


def load_obj(filename_obj, normalization=False, load_texture=False, dr_type='softras', texture_res=4,
             texture_type='surface', texture_wrapping='REPEAT', use_bilinear=True):
    """load_obj.py:9-20 / _load_obj_for_softras.py:142-207.  Returns torch tensors:
    (vertices [nv,3] f32, faces [nf,3] i32) or (+ textures) when load_texture."""
    assert dr_type in ['softras', 'n3mr']
    assert texture_type in ['surface', 'vertex']
    with open(filename_obj) as f:
        lines = f.readlines()
    vertices = np.vstack([[float(v) for v in line.split()[1:4]] for line in lines
                          if len(line.split()) and line.split()[0] == 'v']).astype(np.float32)
    faces = []
    for line in lines:
        s = line.split()
        if len(s) and s[0] == 'f':
            vs = s[1:]
            v0 = int(vs[0].split('/')[0])
            for i in range(len(vs) - 2):
                faces.append((v0, int(vs[i + 1].split('/')[0]), int(vs[i + 2].split('/')[0])))
    faces = np.vstack(faces).astype(np.int32) - 1
    textures = None
    if load_texture and dr_type == 'n3mr':   # _load_obj_for_n3mr.py:139-147 (no texture_type there)
        for line in lines:
            if line.startswith('mtllib'):
                textures = load_textures_n3mr(filename_obj, os.path.join(os.path.dirname(filename_obj), line.split()[1]), texture_res,
                                              texture_wrapping=texture_wrapping, use_bilinear=use_bilinear)
        if textures is None:
            raise Exception('Failed to load textures.')
    elif load_texture and texture_type == 'surface':
        for line in lines:
            if line.startswith('mtllib'):
                textures = load_textures(filename_obj, os.path.join(os.path.dirname(filename_obj), line.split()[1]), texture_res)
        if textures is None:
            raise Exception('Failed to load textures.')
    elif load_texture and texture_type == 'vertex':
        textures = np.vstack([[float(v) for v in line.split()[4:7]] for line in lines
                              if len(line.split()) and line.split()[0] == 'v']).astype(np.float32)
    if normalization:   # unit cube centred at zero (:199-203)
        vertices = vertices - vertices.min(0)
        vertices = vertices / np.abs(vertices).max()
        vertices = vertices * 2
        vertices = vertices - vertices.max(0) / 2
    v, f = torch.from_numpy(vertices.astype(np.float32)), torch.from_numpy(faces)
    if load_texture:
        return v, f, torch.from_numpy(textures)
    return v, f


def texture_atlas(tile_vertices, textures, texture_res_out, tile_width, image_height, image_width, device=None):
    """create_texture_image_cuda_kernel (jrender/io/utils/create_texture_image.py:3-104) through the CUDA kernels
    b200r_texture_atlas_softras (textures [nf, R*R, 3]) / b200r_texture_atlas_n3mr (textures [nf, ts, ts, ts, 3]).

    tile_vertices [nf, 3, 2]: every face's tile triangle in pixel units.  Returns the CUDA float32 image [H, W, 3] as the
    kernel writes it (row 0 at the top, unused tiles 1).  No CPU implementation in the product (oracle/texture_atlas.py
    is the checker)."""
    dev = _gpu("texture-atlas export (b200r_texture_atlas_*)", device)
    tri, tex = _placed(tile_vertices, dev).detach(), _placed(textures, dev).detach()
    nf = tex.shape[0]
    if tri.shape != (nf, 3, 2):
        raise ValueError("texture_atlas: tile_vertices must be [nf, 3, 2] for textures of %d faces" % nf)
    if tex.dim() == 3 and tex.shape[2] == 3 and int(round(np.sqrt(tex.shape[1]))) ** 2 == tex.shape[1]:
        res, name = int(round(np.sqrt(tex.shape[1]))), "b200r_texture_atlas_softras"
    elif tex.dim() == 5 and tex.shape[1] == tex.shape[2] == tex.shape[3] and tex.shape[4] == 3:
        res, name = tex.shape[1], "b200r_texture_atlas_n3mr"
    else:
        raise ValueError("texture_atlas: textures must be [nf, R*R, 3] (SoftRas) or [nf, ts, ts, ts, 3] (NMR), got %s"
                         % (tuple(tex.shape),))
    image = torch.empty((image_height, image_width, 3), dtype=torch.float32, device=dev)
    _lib.call(name, dev, tri, tex, image, nf, res, int(texture_res_out), int(tile_width), int(image_height), int(image_width))
    return image


def create_texture_image(textures, texture_res=16):
    """save_obj.py:7-29: one texture_res x texture_res tile per face in a near-square atlas.  Returns (image [H, W, 3]
    float32 numpy, flipped vertically so that row 0 is the top of the texture as the UVs see it; uv [nf, 3, 2] float32,
    every face's tile triangle normalised by (W - 1, H - 1)).

    textures: [nf, R*R, 3] (SoftRas) or [nf, ts, ts, ts, 3] (NMR), numpy or a tensor on any device (detached).  The tile
    row is the integer face_num // tile_width (the reference divides an int by true division there, save_obj.py:15,
    which puts the UV triangle of every face outside the first column off the tile the kernel paints)."""
    texture_res = int(texture_res)
    if texture_res < 2 or texture_res == 3:
        raise ValueError("create_texture_image: texture_res %d (must be 2 or >= 4; at 3 the tile triangle is degenerate)"
                         % texture_res)
    num_faces = textures.shape[0]
    tile_width = int((num_faces - 1.) ** 0.5) + 1
    tile_height = int((num_faces - 1.) / tile_width) + 1
    face_nums = np.arange(num_faces)
    column, row = face_nums % tile_width, face_nums // tile_width
    R = texture_res
    vertices = np.zeros((num_faces, 3, 2), np.float32)   # [:, :, UV], pixel units
    vertices[:, 0, 0] = column * R + R / 2
    vertices[:, 0, 1] = row * R + 1
    vertices[:, 1, 0] = column * R + 1
    vertices[:, 1, 1] = (row + 1) * R - 1 - 1
    vertices[:, 2, 0] = (column + 1) * R - 1 - 1
    vertices[:, 2, 1] = (row + 1) * R - 1 - 1
    H, W = tile_height * R, tile_width * R
    image = texture_atlas(vertices, textures, R, tile_width, H, W)
    image = image.cpu().numpy() if isinstance(image, torch.Tensor) else np.asarray(image, np.float32)
    vertices[:, :, 0] /= (W - 1)
    vertices[:, :, 1] /= (H - 1)
    return np.ascontiguousarray(image[::-1]), vertices


def _host_array(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def save_obj(filename, vertices, faces, textures=None, texture_res=16, texture_type='surface'):
    """save_obj.py:31-84.  Without textures: the geometry only.  Surface textures ([nf, R*R, 3] or [nf, ts, ts, ts, 3]):
    an atlas of texture_res^2 pixels per face (create_texture_image) written next to the .obj as <name>.png, <name>.mtl
    naming it, and `vt` / `f v/vt` lines.  Vertex textures ([nv, 3]): `v x y z r g b` lines.

    The textured files follow the reference's layout line for line, with two deviations: the integer tile row (see
    create_texture_image) and no `mtllib` line for vertex colours (the reference names a .mtl it never writes, which
    load_obj(load_texture=True) would then fail to open)."""
    assert texture_type in ['surface', 'vertex']
    v, f = _host_array(vertices), _host_array(faces)
    assert v.ndim == 2 and f.ndim == 2
    if textures is None:   # the geometry-only layout this function has always written
        with open(filename, 'w') as fh:
            fh.write('# %s\n\n' % os.path.basename(filename))
            for p in v:
                fh.write('v %.8f %.8f %.8f\n' % (p[0], p[1], p[2]))
            fh.write('\n')
            for t in f:
                fh.write('f %d %d %d\n' % (t[0] + 1, t[1] + 1, t[2] + 1))
        return
    filename_mtl = filename[:-4] + '.mtl'
    if texture_type == 'surface':
        import cv2
        filename_texture = filename[:-4] + '.png'
        material_name = 'material_1'
        texture_image, vertices_textures = create_texture_image(textures, texture_res)
        texture_image = (texture_image.clip(0, 1) * 255).astype('uint8')
        if not cv2.imwrite(filename_texture, np.ascontiguousarray(texture_image[:, :, ::-1])):   # RGB -> BGR
            raise IOError("cannot write texture image %s" % filename_texture)
    else:
        colors = _host_array(textures)
        if colors.shape != (v.shape[0], 3):
            raise ValueError("save_obj: vertex textures must be [nv, 3], got %s" % (colors.shape,))
    with open(filename, 'w') as fh:
        fh.write('# %s\n' % os.path.basename(filename))
        fh.write('#\n')
        fh.write('\n')
        if texture_type == 'surface':
            fh.write('mtllib %s\n\n' % os.path.basename(filename_mtl))
            for p in v:
                fh.write('v %.8f %.8f %.8f\n' % (p[0], p[1], p[2]))
            fh.write('\n')
            for p in vertices_textures.reshape((-1, 2)):
                fh.write('vt %.8f %.8f\n' % (p[0], p[1]))
            fh.write('\n')
            fh.write('usemtl %s\n' % material_name)
            for i, t in enumerate(f):
                fh.write('f %d/%d %d/%d %d/%d\n' % (t[0] + 1, 3 * i + 1, t[1] + 1, 3 * i + 2, t[2] + 1, 3 * i + 3))
            fh.write('\n')
        else:
            for p, c in zip(v, colors):
                fh.write('v %.8f %.8f %.8f %.8f %.8f %.8f\n' % (p[0], p[1], p[2], c[0], c[1], c[2]))
            fh.write('\n')
            for t in f:
                fh.write('f %d %d %d\n' % (t[0] + 1, t[1] + 1, t[2] + 1))
    if texture_type == 'surface':
        with open(filename_mtl, 'w') as fh:
            fh.write('newmtl %s\n' % material_name)
            fh.write('map_Kd %s\n' % os.path.basename(filename_texture))


def save_voxel(filename, voxel):
    """save_obj.py:86-94: one vertex (i / n0, j / n1, k / n2) per voxel equal to 1 of voxel [n0, n1, n2], in the
    reference's i, j, k loop order, written as an OBJ without faces.  The reference hands save_obj a 1-D empty face array,
    which its `len(faces.shape) == 2` assertion rejects, so it never writes a file; this writes the file that call means:
    save_obj's geometry layout (the `#` header, the `v` lines, a blank line) with no `f` lines."""
    v = _host_array(voxel)
    if v.ndim != 3:
        raise ValueError("save_voxel: voxel must be [n0, n1, n2], got %s" % (v.shape,))
    idx = np.argwhere(v == 1)
    vertices = (idx / np.array(v.shape, np.float64)).astype(np.float32)   # Python float division, then float32
    with open(filename, 'w') as fh:
        fh.write('# %s\n#\n\n' % os.path.basename(filename))
        if len(vertices):
            np.savetxt(fh, vertices, fmt='v %.8f %.8f %.8f')
        fh.write('\n')
