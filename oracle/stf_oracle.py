"""ORACLE — TEST INFRASTRUCTURE.  Writes the sources of liboracle_stf.so (stf.mk): the oracle with stochastic texture filtering honoured (rtxpt_b200_set_texture_filtering).

The committed oracle (pt_scene.h, oracle.cpp) samples material textures trilinearly and stays as it is.  This script streams those two files into OUTDIR with pt_stf.h applied:
the scene carries the STF settings, loadSurface opens the vertex's sampler state around sampleGeometryMaterial (PathTracerBridgeDonut.hlsli:637-656), the material fetch runs
STF's Texture2DSampleLevel while that state is active, and oracle.cpp gains oracle_set_texture_filtering.  Every rewrite is an insertion, so with STF off the library computes
what liboracle.so computes; each anchor must occur exactly once, or the script fails.  The other headers are copied into OUTDIR as they are, so that every header that
includes pt_scene.h finds the rewritten one.

    python3 stf_oracle.py OUTDIR
"""
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))

PT_SCENE = [
    ("#include <vector>\n", '#include <vector>\n#include "pt_stf.h"\n'),
    ("    std::vector<RtxptSubInstanceData> subInstances;", "    StfSettings stf;\n    std::vector<RtxptSubInstanceData> subInstances;"),
    ("    return sc.textures[textureIndex].sampleLevel(uv, lambda);\n",
     "    if (stfCurrentVertex().active) return stfSampleLevel(sc.textures[textureIndex], uv, lambda, stfCurrentVertex());\n"
     "    return sc.textures[textureIndex].sampleLevel(uv, lambda);\n"),
    ("    MaterialProperties mat = sampleGeometryMaterial(sc, gs, materialIndex, lambda);\n",
     "    MaterialProperties mat;\n"
     "    {\n"
     "        StfVertexScope stfScope(sc.stf, pixelX, pixelY, pathVertexIndex, sampleIndex);\n"
     "        mat = sampleGeometryMaterial(sc, gs, materialIndex, lambda);\n"
     "    }\n"),
]
ORACLE_CPP = [
    ('} // extern "C"',
     "// rtxpt_b200_set_texture_filtering: the description the product accepts (magnification method NONE)\n"
     "ORC_API int oracle_set_texture_filtering(void* p, const RtxptStochasticTextureFiltering* f)\n"
     "{\n"
     "    OracleCtx* c = (OracleCtx*)p;\n"
     "    if (f->magnificationMethod != 0 || f->filterType > 3) return -1;\n"
     "    c->scene.stf.enable = f->enable; c->scene.stf.filterType = f->filterType; c->scene.stf.sigma = f->gaussianSigma;\n"
     "    return 0;\n"
     "}\n"
     '} // extern "C"'),
]


def rewrite(name, edits, out):
    with open(os.path.join(HERE, name)) as f:
        text = f.read()
    for old, new in edits:
        n = text.count(old)
        if n != 1:
            sys.exit("stf_oracle.py: %s: anchor found %d times (expected once): %r" % (name, n, old[:80]))
        text = text.replace(old, new)
    with open(os.path.join(out, name), "w") as f:
        f.write(text)


if __name__ == "__main__":
    out = sys.argv[1]
    os.makedirs(out, exist_ok=True)
    for name in sorted(os.listdir(HERE)):
        if name.endswith(".h") and name != "pt_scene.h":
            shutil.copy(os.path.join(HERE, name), os.path.join(out, name))
    rewrite("pt_scene.h", PT_SCENE, out)
    rewrite("oracle.cpp", ORACLE_CPP, out)
