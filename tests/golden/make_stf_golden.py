"""Generates tests/golden/stf_golden.npz: stochastic texture filtering as RTXPT's material fetches run it (STF_SamplerState::Texture2DSampleLevel at magnification method NONE),
from the UNMODIFIED External/Rtxtf headers (oracle/_ref/ref_kat_stf of oracle/stf.mk).  Each case is one sampler state - the four filters, random u, Gaussian sigma 0.05 .. 3,
reseedOnSample off and on, a wrap or clamp sampler - over one texture (power-of-two and odd sizes, 1 x 1 up to 4096 x 4096, full or partial mip chains) with four fetches at
random uv (also outside [0, 1], and at exact half-texel multiples j / (2 size): the rounding ties of Point and Gaussian and the probability-0 / 1 picks of Linear) and lambda (also below 0 and beyond the chain, integers included).  Records: the input words (`inp`, 28 per case) and what the reference wrote
(`out`: per fetch the position, level, texel and the state's u after the fetch; per case STF_ApplyAddressingMode1D of the last position for the five address modes).
Run in the build container only:
    make -C oracle -f stf.mk ref && python tests/golden/make_stf_golden.py"""
import os, subprocess
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
KAT = os.path.join(ROOT, "oracle", "_ref", "ref_kat_stf")
IN_WORDS, OUT_WORDS = 28, 4 * 11 + 10


def make(n, seed):
    rng = np.random.default_rng(seed)
    inp = np.zeros((n, IN_WORDS), np.uint32); f = inp.view(np.float32)
    sizes = np.array([1, 2, 3, 4, 5, 7, 8, 13, 16, 31, 64, 100, 127, 256, 333, 512, 1024, 4096])
    w = rng.choice(sizes, n); h = np.where(rng.random(n) < 0.5, w, rng.choice(sizes, n))
    full = np.floor(np.log2(np.maximum(w, h))).astype(np.int64) + 1
    levels = np.where(rng.random(n) < 0.8, full, np.maximum(1, (full * rng.random(n)).astype(np.int64) + 1))
    inp[:, 0] = w; inp[:, 1] = h; inp[:, 2] = levels
    inp[:, 3] = rng.integers(0, 4, n)
    f[:, 4] = np.exp(rng.uniform(np.log(0.05), np.log(3.0), n)).astype(np.float32); f[rng.random(n) < 0.3, 4] = 0.3          # RTXPT's UI default
    inp[:, 5] = np.where(rng.random(n) < 0.7, 1, 3)
    inp[:, 6] = rng.random(n) < 0.5
    u = (rng.integers(0, 1 << 24, (n, 4)) * 2.0 ** -24).astype(np.float32)                                                       # what a uniform generator draws
    u[:, 0] = np.where(inp[:, 3] == 3, np.maximum(u[:, 0], np.float32(2.0 ** -24)), u[:, 0])                                     # Gaussian: log(0) is not a sample
    f[:, 7:11] = u
    for k in range(4):
        uv = rng.uniform(0.0, 1.0, (n, 2)); wide = rng.random(n) < 0.25
        uv[wide] = rng.uniform(-3.0, 4.0, (wide.sum(), 2))
        lam = rng.uniform(-1.5, levels + 1.0); integral = rng.random(n) < 0.15; lam[integral] = np.round(lam[integral])
        # rounding ties and certain picks: uv = j / (2 size) exactly (uv * size - 0.5 a half-integer or an integer at even sizes - uv 0, 0.5, 1 on real meshes)
        tie = rng.random(n) < 0.3
        for a, dim in ((0, w), (1, h)):
            j = rng.integers(-2, 2 * dim + 3); uv[tie, a] = (j / (2.0 * dim))[tie]
        f[:, 11 + 3 * k] = uv[:, 0]; f[:, 12 + 3 * k] = uv[:, 1]; f[:, 13 + 3 * k] = lam
    return inp


def run(inp):
    r = subprocess.run([KAT], input=inp.tobytes(), stdout=subprocess.PIPE, check=True)
    return np.frombuffer(r.stdout, np.uint32).reshape(len(inp), OUT_WORDS)


if __name__ == "__main__":
    inp = make(3000, 20261017)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "stf_golden.npz"), inp=inp, out=run(inp))
