"""NEEFullSamples > 1 in the CUDA source, held to the reference's shader code and to the oracle on the CPU.

tests/emu/nee_full_samples_host_emu.cu (nee_emu_multi_vertices; it reuses the stub bridge of tests/emu/shade_host_emu.cu) runs the multi-sample shade of shade.cuh -
k_shade< .., MULTI > in reference mode, k_rt_shade< FILL, .., MULTI > - on one vertex, gives every light sample's shadow record the golden stub bridge's visibility answer as k_trace_shadow< .., MULTI > would mark it, and resolves the vertex's NEE block with
k_nee_resolve's body.  HandleNEE takes the samples from the vertex's one uniform stream and rounds the running (radiance, specAvg) sum to fp16 after every visible sample
(PathTracerNEE.hlsli:277-346), so the sample order is part of the result."""
import ctypes as C
import os
import subprocess
import numpy as np
from test_shade_port import PAYLOAD, SHADOW, FEEDBACK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    subprocess.run(["make", "-C", os.path.join(ROOT, "tests", "emu"), "-s", "-f", "nee_full_samples.mk"], check=True)
    L = C.CDLL(os.path.join(ROOT, "tests", "emu", "_build", "libnee_full_samples_emu.so"))
    L.nee_emu_multi_vertices.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int32]; L.nee_emu_multi_vertices.restype = None
    return L


COLS = {0: [c for c in PAYLOAD if c != 15] + SHADOW + FEEDBACK, 2: PAYLOAD + SHADOW + [37] + FEEDBACK + list(range(41, 51))}


def _multi(L, r, mode, reverse=False):
    r = np.ascontiguousarray(r, np.float32)
    out = np.zeros((len(r), 128), np.float32); st = np.zeros(len(r), np.int32)
    L.nee_emu_multi_vertices(r.ctypes.data, len(r), out.ctypes.data, st.ctypes.data, mode, int(reverse))
    return out, st == 0


def test_multi_sample_shade_matches_reference_path_tracer_golden():
    """The golden's hits with NEEFullSamples = 2 and no feedback insertion, in the reference and the FILL pass: the outgoing path state, the number of shadow rays, the last one
    and its answer, the planes and header (FILL) - bit for bit against the unmodified PathTracer.hlsli."""
    L = _lib()
    g = np.load(os.path.join(ROOT, "tests", "golden", "hit_golden.npz"))
    for key, mode in (("hit", 0), ("fill", 2)):
        u, ref = g[key + "_in"], g[key + "_out"]
        sel = (u[:, 27] == 0) & (u[:, 84] == 2) & (u[:, 92] == 0)
        out, ran = _multi(L, u[sel], mode)
        assert ran.all() and sel.sum() >= 20, (key, sel.sum())
        same = ref[sel].view(np.uint32)[:, COLS[mode]] == out.view(np.uint32)[:, COLS[mode]]
        assert same.all(), (key, np.argwhere(~same)[:8])
        assert (ref[sel, 20] == 2).any()            # both samples traced on some vertices


def test_multi_sample_shade_agrees_with_oracle_on_recombined_vertices(oracle):
    """Recombined vertices (as test_shade_port's fourth test) with NEEFullSamples 0, 2, 3, 5, 8 and 63 and no feedback insertion: the host build of the CUDA source equals
    the oracle's HandleNEE loop on every compared word.  From three visible samples on, summing the block in reverse order changes some results: the test would see an order bug."""
    L = _lib()
    O = oracle.lib(); O.oracle_hit_funcs.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]; O.oracle_hit_funcs.restype = None
    g = np.load(os.path.join(ROOT, "tests", "golden", "hit_golden.npz"))
    n = 4000
    reversed_differs = 0
    for key, mode in (("hit", 0), ("fill", 2)):
        rng = np.random.default_rng(200 + mode); u = g[key + "_in"]; u = u[u[:, 27] <= 1]; pick = lambda: rng.integers(0, len(u), n)
        for full in (0, 2, 3, 5, 8, 63):
            r = u[pick()].copy()
            for lo, hi in ((80, 96), (96, 136), (136, 920), (920, 950), (950, 960)): r[:, lo:hi] = u[pick(), lo:hi]
            for w in (14, 17, 18): q = pick(); sel = rng.random(n) < 0.5; r[sel, w] = u[q[sel], w]
            r[:, 84] = full; r[:, 92] = 0
            r = np.ascontiguousarray(r)
            a, ran = _multi(L, r, mode)
            b = np.zeros((n, 128), np.float32); O.oracle_hit_funcs(r.ctypes.data, n, b.ctypes.data, mode)
            same = a.view(np.uint32)[:, COLS[mode]] == b.view(np.uint32)[:, COLS[mode]]
            assert ran.all() and same.all(), (key, full, np.argwhere(~same)[:8])
            hits = r[:, 27] == 0
            if full == 0: assert (b[hits, 20] == 0).all()
            else: assert (b[hits, 20] > 1).mean() > (0.2 if full > 1 else 0), (key, full)
            if full >= 3:
                rev, _ = _multi(L, r, mode, reverse=True)
                reversed_differs += int((rev.view(np.uint32)[:, COLS[mode]] != a.view(np.uint32)[:, COLS[mode]]).any(1).sum())
    assert reversed_differs > 10, reversed_differs
