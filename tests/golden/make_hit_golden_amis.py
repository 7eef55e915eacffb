"""Generates tests/golden/hit_golden_amis.npz: the records of make_hit_golden.py's three passes run through the UNMODIFIED reference headers compiled with
RTXPT_USE_APPROXIMATE_MIS = 1 (oracle/_ref/ref_kat_bsdf_amis, ref_kat_pt_build_amis, ref_kat_pt_fill_amis of oracle/amis.mk; everything else as for hit_golden.npz), the light-vs-BSDF MIS that RTXPT's
realtime mode compiles by default.  Word 94 of every record is 1: the approximate-MIS oracle's "hit" mode (oracle/amis.mk) reads it as RtxptPathTracerConstants::useApproximateMIS.
Besides make()'s mix (NEE-AT feedback, emissive surfaces without a light record as for ExcludeFromNEE), NEEFullSamples spans 1 .. 63.
Run in the build container only:
    make -C oracle ref && make -C oracle -f amis.mk ref && python tests/golden/make_hit_golden_amis.py"""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden")); sys.path.insert(0, os.path.join(ROOT, "tests"))
from make_bsdf_golden import run  # noqa: E402
from make_hit_golden import make  # noqa: E402


def approximate(u, rng):
    """word 94 = 1; NEEFullSamples 1 (half the records), 2 .. 8 or 9 .. 63, in the constants (84) and in the incoming path's packed MIS info (payload word 18, bits 16-21); most
    records with several samples without feedback insertion (92), which the product refuses together; half the emissive surfaces without a light record (75)"""
    n = len(u); fs = np.where(rng.random(n) < 0.5, 1, np.where(rng.random(n) < 0.7, rng.integers(2, 9, n), rng.integers(9, 64, n))).astype(np.uint32)
    u[:, 84] = fs; u[:, 94] = 1.0
    U = u.view(np.uint32); U[:, 18] = (U[:, 18] & ~np.uint32(0x3F << 16)) | (fs << 16)
    u[(fs > 1) & (rng.random(n) < 0.7), 92] = 0.0
    u[(u[:, 54:57] > 0).any(1) & (rng.random(n) < 0.5), 75] = -1.0
    return u


def with_ops(u, n_init, seed):
    """op 2 (EmptyPathInitialize) on the first n_init records, as in make_hit_golden.py"""
    r2 = np.random.default_rng(seed); u[:n_init, 27] = 2; u[:n_init, 1020] = np.exp(r2.uniform(-9, -5, n_init)); u[:n_init // 4, 80] = 0
    return u


if __name__ == "__main__":
    g = np.load(os.path.join(ROOT, "tests", "golden", "interior_golden.npz")); slots = g["interior_out"].reshape(-1, 12, 6)[:, :, 0:2].reshape(-1, 2).view(np.uint32); slots = slots[(slots != 0).any(1)]
    u = with_ops(approximate(make(np.random.default_rng(877), 120, slots), np.random.default_rng(880)), 8, 1)
    out = run("hit", u, 128, exe="ref_kat_bsdf_amis")
    ub = approximate(make(np.random.default_rng(879), 60, slots, build=True), np.random.default_rng(881))
    outb = run("hit", ub, 128, exe="ref_kat_pt_build_amis")
    uf = approximate(make(np.random.default_rng(878), 120, slots, fill=True), np.random.default_rng(882))
    outf = run("hit", uf, 128, exe="ref_kat_pt_fill_amis")
    src = ("Rtxpt/Shaders/PathTracer/{PathTracer,PathTracerNEE,PathTracerNestedDielectrics,PathTracerStablePlanes,StablePlanes,PathState,PathPayload}.hlsli + Lighting/LightSampler.hlsli + "
           "Utils/SampleGenerators.hlsli at reference commit f08d1c7 with RTXPT_USE_APPROXIMATE_MIS = 1, compiled as C++ by oracle/amis.mk targets _ref/ref_kat_bsdf_amis (PATH_TRACER_MODE 0), "
           "_ref/ref_kat_pt_build_amis (1) and _ref/ref_kat_pt_fill_amis (2) behind oracle/ref_bridge_stub.h")
    path = os.path.join(ROOT, "tests", "golden", "hit_golden_amis.npz")
    np.savez_compressed(path, hit_in=u, hit_out=out, fill_in=uf, fill_out=outf, build_in=ub, build_out=outb, source=np.array(src))
    print(u.shape, out.shape, uf.shape, outf.shape, ub.shape, outb.shape, os.path.getsize(path))
