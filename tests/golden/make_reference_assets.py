"""Packs the reference's material and scene files (data, not code) into the archives the CPU tests read:
  reference_materials.tar.xz  every Assets/Materials/*.material.json and Assets/Materials/*/*.material.json (tests/test_material_json.py)
  reference_scenes.tar.xz     every Assets/*.scene.json and the model files they name that exist in the reference (git-LFS pointer stubs, ~130 B each;
                              tests/test_scene_json.py)
Run where the reference tree lies:   python tests/golden/make_reference_assets.py <reference root>"""
import glob
import io
import json
import os
import sys
import tarfile

HERE = os.path.dirname(os.path.abspath(__file__))


def scene_models(base, scenes):
    models = set()
    for f in scenes:
        try: names = json.load(open(f)).get("models", [])
        except ValueError: continue         # a scene file that is not JSON itself
        models.update(p for p in (os.path.join(base, m.replace("\\", "/")) for m in names) if os.path.isfile(p))
    return sorted(models)


def pack(base, patterns, out, extra=lambda files: []):
    files = sorted(sum((glob.glob(os.path.join(base, p)) for p in patterns), []))
    files += extra(files)
    with tarfile.open(out, "w:xz") as t:
        for f in files:
            data = open(f, "rb").read()
            ti = tarfile.TarInfo(os.path.relpath(f, base)); ti.size = len(data); ti.mtime = 0; ti.mode = 0o644
            t.addfile(ti, io.BytesIO(data))
    print(out, len(files), "files")


if __name__ == "__main__":
    ref = sys.argv[1]
    pack(os.path.join(ref, "Assets", "Materials"), ["*.material.json", "*/*.material.json"], os.path.join(HERE, "reference_materials.tar.xz"))
    assets = os.path.join(ref, "Assets")
    pack(assets, ["*.scene.json"], os.path.join(HERE, "reference_scenes.tar.xz"), lambda scenes: scene_models(assets, scenes))
