"""CPU: stochastic texture filtering (rtxpt_b200/csrc/stf.cuh) against the reference.  The host build of stf.cuh (tests/emu/stf.mk) reproduces tests/golden/stf_golden.npz - what
the UNMODIFIED External/Rtxtf headers compute (oracle/_ref/ref_kat_stf) - word for word: sample positions, levels, texels and the sampler state after every fetch.  Its Linear,
Cubic and Gaussian picks average to the bilinear, B-spline and Gaussian filter weights, and every pick is a texel centre of a level of the chain."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "stf_golden.npz")
OUT_WORDS = 4 * 11 + 10


@pytest.fixture(scope="module")
def emu():
    subprocess.run(["make", "-C", os.path.join(ROOT, "tests", "emu"), "-s", "-f", "stf.mk"], check=True)
    L = C.CDLL(os.path.join(ROOT, "tests", "emu", "_build", "libstf_emu.so"))
    L.stf_emu_run.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    L.stf_emu_vertex_random.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    return L


def run(emu, inp):
    inp = np.ascontiguousarray(inp, np.uint32)
    out = np.zeros((len(inp), OUT_WORDS), np.uint32)
    emu.stf_emu_run(inp.ctypes.data, len(inp), out.ctypes.data)
    return out


def test_host_build_reproduces_reference_golden(emu):
    g = np.load(GOLDEN)
    inp, ref = g["inp"], g["out"]
    assert set(np.unique(inp[:, 3])) == {0, 1, 2, 3} and set(np.unique(inp[:, 5])) == {1, 3} and set(np.unique(inp[:, 6])) == {0, 1}
    out = run(emu, inp)
    bad = np.nonzero((out != ref).any(1))[0]
    assert len(bad) == 0, f"{len(bad)} of {len(inp)} cases differ, first {bad[0]}: {inp[bad[0]]} -> {out[bad[0]]} vs {ref[bad[0]]}"


def test_golden_positions_are_texel_centres_of_the_chain():
    g = np.load(GOLDEN)
    inp, out = g["inp"], g["out"]
    for f in range(4):
        o = out[:, 11 * f: 11 * f + 11]
        lod = o[:, 2].astype(np.int64)
        assert (lod < inp[:, 2]).all()
        w = np.maximum(1, inp[:, 0].astype(np.int64) >> lod); h = np.maximum(1, inp[:, 1].astype(np.int64) >> lod)
        pos = o[:, :2].view(np.float32).astype(np.float64)
        for p, n in ((pos[:, 0], w), (pos[:, 1], h)):
            s = p * n - 0.5
            assert np.abs(s - np.round(s)).max() < 1e-3
        texel = o[:, 3:7].view(np.float32)
        assert (texel[:, 0] >= 0).all() and (texel[:, 0] < w).all() and (texel[:, 1] >= 0).all() and (texel[:, 1] < h).all() and (texel[:, 2] == lod).all()
    # the state moves between fetches only when the sampler reseeds
    u0 = inp[:, 7:11]
    for f in range(4):
        after = out[:, 11 * f + 7: 11 * f + 11]
        assert (after[inp[:, 6] == 0] == u0[inp[:, 6] == 0]).all()
    assert (out[inp[:, 6] == 1, 7:11] != u0[inp[:, 6] == 1]).any(1).mean() > 0.5


def _picks(emu, filt, x, y, size, sigma, n, seed):
    """n picks of one position at level 0 (lambda 0) of a size x size texture, wrap sampler"""
    rng = np.random.default_rng(seed)
    inp = np.zeros((n, 28), np.uint32); f = inp.view(np.float32)
    inp[:, 0] = size; inp[:, 1] = size; inp[:, 2] = 1; inp[:, 3] = filt; f[:, 4] = sigma; inp[:, 5] = 1
    f[:, 7:11] = (rng.integers(1, 1 << 24, (n, 4)) * 2.0 ** -24).astype(np.float32)
    for k in range(4): f[:, 11 + 3 * k] = x; f[:, 12 + 3 * k] = y; f[:, 13 + 3 * k] = 0.0
    out = run(emu, inp)
    t = out[:, 3:5].view(np.float32).astype(np.int64)
    return t[:, 0], t[:, 1]


def _weights_1d(filt, s, sigma, size):
    """the filter's weight of every texel of the axis (wrapped) for texel-space coordinate s"""
    w = np.zeros(size)
    base = math.floor(s); t = s - base
    if filt == 1:
        taps = {base: 1 - t, base + 1: t}
    elif filt == 2:
        taps = {base - 1: (1 - t) ** 3 / 6, base: (3 * t ** 3 - 6 * t ** 2 + 4) / 6, base + 1: (-3 * t ** 3 + 3 * t ** 2 + 3 * t + 1) / 6, base + 2: t ** 3 / 6}
    else:
        phi = lambda z: 0.5 * (1 + math.erf(z / math.sqrt(2)))
        taps = {k: phi((k + 0.5 - s) / sigma) - phi((k - 0.5 - s) / sigma) for k in range(base - 12, base + 14)}
    for k, v in taps.items(): w[k % size] += v
    return w


@pytest.mark.parametrize("filt,sigma", [(1, 0.3), (2, 0.3), (3, 0.3), (3, 1.7)])
def test_picks_converge_to_filter_weights(emu, filt, sigma):
    """Linear -> bilinear, Cubic -> cubic B-spline, Gaussian -> the Gaussian's mass over each texel; the bar is five binomial standard deviations of the sample count"""
    size, n = 16, 200000
    for (x, y, seed) in ((0.3712, 0.8127, 1), (0.0213, 0.9902, 2)):
        px, py = _picks(emu, filt, x, y, size, sigma, n, seed)
        sx, sy = np.float32(x) * size - 0.5, np.float32(y) * size - 0.5
        expect = np.outer(_weights_1d(filt, float(sy), sigma, size), _weights_1d(filt, float(sx), sigma, size))
        got = np.bincount(py * size + px, minlength=size * size).reshape(size, size) / n
        bar = 5 * np.sqrt(np.maximum(expect * (1 - expect), 1e-12) / n) + 1e-5
        assert (np.abs(got - expect) <= bar).all(), np.abs(got - expect).max()


def test_vertex_random_is_the_bridges_uniform_generator(emu):
    """u = four draws of a fresh UniformSampleSequenceGenerator of (pixel, vertex, sample), effect seed Base (PathTracerBridgeDonut.hlsli:648-650), written out in Python"""
    M = 0xFFFFFFFF
    def h32(x):
        x ^= x >> 16; x = (x * 0x21f0aaad) & M; x ^= x >> 15; x = (x * 0xf35a2d97) & M; x ^= x >> 15; return x
    def comb(seed, v): return (seed ^ ((h32(v) + 0x9e3779b9 + ((seed << 6) & M) + (seed >> 2)) & M)) & M
    for pix, vtx, smp in ((0x00030007, 1, 0), (0x01200045, 3, 17), (0xFFFF0000, 9, 123456)):
        h = comb(comb(comb(h32((vtx + 0x035F9F29) & M), pix), 0), smp)
        want = []
        for _ in range(4):
            h = h32(h); want.append(np.float32((h >> 8) * 2.0 ** -24))
        got = np.zeros(4, np.float32); emu.stf_emu_vertex_random(pix, vtx, smp, got.ctypes.data)
        assert got.tolist() == want


def test_stf_oracle_off_is_the_oracle_and_on_is_another_image():
    """liboracle_stf.so with STF off renders what liboracle.so renders, bit for bit; with each filter on, the textured Cornell box is another image, and the same one twice"""
    import oracle_lib
    import oracle_stf_lib
    from rtxpt_b200 import scene_builder as sb
    from test_gpu_stf_parity import textured_cornell, _camera
    oracle_stf_lib.build()
    W = H = 24
    scene = textured_cornell()
    consts = sb.make_constants(W, H, _camera(W, H), bounce_count=3, diffuse_bounce_count=3)
    def render(mod, filt=None):
        o = mod.Oracle(scene); o.set_constants(consts)
        if filt is not None: oracle_stf_lib.set_texture_filtering(o, True, filt, 0.3)
        acc = o.render(0, 1)[0]; o.close()
        return acc
    base = render(oracle_lib)
    assert np.array_equal(render(oracle_stf_lib.oracle), base)
    for filt in range(4):
        a = render(oracle_stf_lib.oracle, filt)
        assert not np.array_equal(a, base) and np.array_equal(a, render(oracle_stf_lib.oracle, filt)) and np.isfinite(a).all()


def test_stf_struct_layout_matches_the_header():
    """RtxptStochasticTextureFiltering: the Python mirror's size and offsets are the C compiler's"""
    import tempfile
    from rtxpt_b200 import structs as S
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "rtxpt_b200.h"\nint main(void) { printf("%zu %zu %zu %zu %zu\\n", sizeof(RtxptStochasticTextureFiltering), '
           'offsetof(RtxptStochasticTextureFiltering, enable), offsetof(RtxptStochasticTextureFiltering, filterType), '
           'offsetof(RtxptStochasticTextureFiltering, magnificationMethod), offsetof(RtxptStochasticTextureFiltering, gaussianSigma)); return 0; }\n')
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "l.c"), "w") as f: f.write(src)
        subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "l.c"), "-o", os.path.join(d, "l")], check=True)
        got = [int(x) for x in subprocess.run([os.path.join(d, "l")], capture_output=True, text=True, check=True).stdout.split()]
    T = S.StochasticTextureFiltering
    assert got == [C.sizeof(T), T.enable.offset, T.filterType.offset, T.magnificationMethod.offset, T.gaussianSigma.offset]
