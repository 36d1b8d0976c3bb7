"""Stage the few reference DATA files the as-configured demos need (BASELINE configs C1 and C5) into baseline/_ref/assets/.

    python -m tools.stage_assets

/root/reference does not exist on the GPU box; baseline/_ref/ is git-ignored but travels with gpurun, so benches, examples
and GPU tests can run demo1 (spot cow, T=25 baked
textures) and demo2 (sphere_1352 -> data/source.npy silhouettes with data/camera.npy) literally.  Data only -- no
reference source code is copied -- and nothing here is committed.  Consumers fall back to generated stand-ins (and say
so) when the directory is absent.
"""
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE = "/root/reference"
OUT = os.path.join(os.path.dirname(HERE), "baseline", "_ref", "assets")
FILES = [
    "data/obj/spot/spot_triangulated.obj", "data/obj/spot/spot_triangulated.mtl", "data/obj/spot/spot_texture.png",   # demo1-render.py:17,26
    "data/obj/sphere/sphere_1352.obj",                                                                                # demo2-deform.py:55
    "data/source.npy", "data/camera.npy",                                                                             # demo2-deform.py:50-53
    "data/head/head.obj", "data/head/head.mtl", "data/head/lambertian.jpg", "data/head/bump.png",                      # demo1.5-SSS.py:17,23
]


def path(rel):
    """Absolute path of a staged asset, or None when it is not there."""
    p = os.path.join(OUT, rel)
    return p if os.path.exists(p) else None


def stage():
    if not os.path.isdir(REFERENCE):
        return False
    for rel in FILES:
        src, dst = os.path.join(REFERENCE, rel), os.path.join(OUT, rel)
        if not os.path.exists(src):
            continue
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if not os.path.exists(dst) or os.path.getsize(dst) != os.path.getsize(src):
            shutil.copyfile(src, dst)
    return True


if __name__ == "__main__":
    print("staged" if stage() else "no /root/reference here", OUT)
