"""Generates tests/golden/debug_view_golden.npz: RTXPT's debug-view colour functions from the UNMODIFIED reference (oracle/_ref/ref_kat_debug of oracle/debug_views_ref.mk):
ColorFromHash over hashed material IDs, raw words and the R11G11B10 edge patterns (zero, infinity and NaN exponents); GradientHeatMap over [-0.5, 1.5] and every breakpoint
(0.3, 0.7, 0.8, 0.9) with its float neighbours; StablePlaneDebugVizColor for planes 0..5; StablePlaneDebugVizFourWaySplitCoord for plane indices -1..2 at odd and even
screen sizes, every quadrant edge included; DbgShowNormalSRGB on random and axis-aligned unit vectors.  Records: `inp` (op, a, b, c) and `out` (3 words per record).
Run in the build container only:
    make -C oracle -f debug_views_ref.mk ref && python tests/golden/make_debug_view_golden.py"""
import os, subprocess
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
KAT = os.path.join(ROOT, "oracle", "_ref", "ref_kat_debug")


def _hash32(x):
    x = x.astype(np.uint64)
    x ^= x >> 16; x = (x * 0x21f0aaad) & 0xFFFFFFFF; x ^= x >> 15; x = (x * 0xf35a2d97) & 0xFFFFFFFF; x ^= x >> 15
    return x.astype(np.uint32)


def make(seed=11):
    rng = np.random.default_rng(seed)
    recs = []
    words = np.concatenate([_hash32(np.arange(4096, dtype=np.uint32)), _hash32(np.uint32([0xFFFFFFFF])), rng.integers(0, 2**32, 4000, dtype=np.uint64).astype(np.uint32),
                            np.uint32([0, 0x7C0, 0x7FF, 0x3E0000, 0xFFC00000, 0xFFFFFFFF, 0x1F << 6, 0x1F << 17, 0x1F << 27])])
    recs += [(0, int(w), 0, 0) for w in words]
    grey = np.concatenate([rng.uniform(-0.5, 1.5, 4000), np.linspace(0, 1, 1001)]).astype(np.float32)
    for b in (0.0, 0.3, 0.7, 0.8, 0.9, 1.0):
        b = np.float32(b); grey = np.concatenate([grey, np.float32([np.nextafter(b, np.float32(-1)), b, np.nextafter(b, np.float32(2))])])
    recs += [(1, int(w), 0, 0) for w in grey.view(np.uint32)]
    recs += [(2, p, 0, 0) for p in range(6)]
    for W, H in ((1920, 1080), (37, 19), (8, 8), (1, 1)):
        for plane in (-1, 0, 1, 2):
            xs = np.unique(np.concatenate([rng.integers(0, W, 40), [0, W // 2 - 1, W // 2, W - 1]]).clip(0, W - 1))
            ys = np.unique(np.concatenate([rng.integers(0, H, 40), [0, H // 2 - 1, H // 2, H - 1]]).clip(0, H - 1))
            recs += [(3, plane & 0xFFFFFFFF, int(x) | (int(y) << 16), W | (H << 16)) for x in xs[::3] for y in ys]
    n = rng.normal(size=(3000, 3)); n /= np.linalg.norm(n, axis=1, keepdims=True)
    n = np.concatenate([n, np.eye(3), -np.eye(3)]).astype(np.float32)
    recs += [(4, int(a), int(b), int(c)) for a, b, c in n.view(np.uint32)]
    return np.array(recs, np.uint32)


def main():
    inp = make()
    out = subprocess.run([KAT], input=inp.tobytes(), capture_output=True, check=True).stdout
    out = np.frombuffer(out, np.uint32).reshape(len(inp), 3)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "debug_view_golden.npz"), inp=inp, out=out)
    print(len(inp), "records")


if __name__ == "__main__":
    main()
