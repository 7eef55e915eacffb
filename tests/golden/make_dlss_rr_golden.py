"""Generates tests/golden/dlss_rr_golden.npz: RTXPT's DLSS-RR input pass (PostProcess.hlsl DENOISER_DLSS_RR, :175-440, with ComputeSpecularMotionVector, :94-160) from the
UNMODIFIED reference (oracle/_ref/ref_kat_dlss_rr of oracle/dlss_rr_ref.mk) on synthetic single pixels: random plane records with 1, 2 and 3 active planes; invalid planes and
sky planes (infinite SceneLength); dark diffuse BSDF estimates with bright specular ones, and both dark (the 0.05 albedo floor from both sides); zero stable radiance and radiance above the clamp (DLSSRRBrightnessClampK 4096 and 0.5); plane roughness on both sides of 0.25 and specular
hit distances at and around 1e-3; normals with n.z < 0 and reflection rays behind the normal (zObj < 0); static and moving cameras.
Records: `inp` (104 words, the layout ref_kat_dlss_rr_main.cpp documents) and `out` (15 floats per record).  Run in the build container only:
    make -C oracle -f dlss_rr_ref.mk ref && python tests/golden/make_dlss_rr_golden.py"""
import os, subprocess
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
KAT = os.path.join(ROOT, "oracle", "_ref", "ref_kat_dlss_rr")
INVALID = 0xFFFFFFFF
W, H = 1920, 1080


def f16(x):
    return np.asarray(x, np.float16).view(np.uint16).astype(np.uint32)


def pack2(hi, lo):
    return (f16(hi) << 16) | f16(lo)


def world_to_clip(eye, target, fov_y=1.0, aspect=W / H, near=0.1):
    """Row-vector view-projection (float4(p, 1) x M), reverse-Z infinite projection like RTXPT's camera."""
    eye, target = np.asarray(eye, np.float64), np.asarray(target, np.float64)
    f = target - eye; f /= np.linalg.norm(f)
    r = np.cross(f, [0.0, 1.0, 0.0]); r /= np.linalg.norm(r)
    u = np.cross(r, f)
    view = np.eye(4); view[:3, 0], view[:3, 1], view[:3, 2] = r, u, f; view[3, :3] = [-r @ eye, -u @ eye, -f @ eye]
    t = 1.0 / np.tan(fov_y / 2)
    proj = np.zeros((4, 4)); proj[0, 0] = t / aspect; proj[1, 1] = t; proj[3, 2] = near; proj[2, 3] = 1.0
    return (view @ proj).astype(np.float32)


def cameras(rng):
    eye = np.array([0.0, 1.0, -5.0]); target = np.array([0.0, 0.5, 0.0])
    cur = world_to_clip(eye, target)
    moved = [world_to_clip(eye + rng.normal(scale=0.05, size=3), target + rng.normal(scale=0.05, size=3)) for _ in range(4)]
    return cur, [cur] + moved          # the first previous view is the same camera (static)


def oct_word(n):
    """NDirToOctUnorm32 of unit vectors (Utils.hlsli): enough to produce valid normal words of a chosen direction."""
    n = n / np.abs(n).sum(-1, keepdims=True)
    xy = n[..., :2].copy()
    neg = n[..., 2] < 0
    wrap = (1 - np.abs(xy[..., ::-1])) * np.where(xy >= 0, 1.0, -1.0)
    xy[neg] = wrap[neg]
    u = np.clip(xy * 0.5 + 0.5, 0, 1)
    u = np.clip(u * 0.5 + 0.5, 0, 1)            # the [0, 1] mapping is applied twice (see lights_bake.cpp)
    q = np.round(u * 0xFFFE).astype(np.uint32)
    return q[..., 0] | (q[..., 1] << 16)


def make(seed=23, count=2000):
    rng = np.random.default_rng(seed)
    cur, prevs = cameras(rng)
    recs = np.zeros((count, 104), np.uint32)
    for i in range(count):
        r = recs[i]
        active = 1 + i % 3
        r[0] = active
        r[1] = np.float32(4096.0 if i % 4 else 0.5).view(np.uint32)
        valid = rng.random(3) < 0.75
        if i % 11 == 0: valid[:] = False
        for k in range(3):
            r[2 + k] = rng.integers(1, 1 << 12) if valid[k] else INVALID
        r[5] = (np.float32(rng.uniform(0.5, 20)).view(np.uint32) & 0xFFFFFFFC) | rng.integers(0, 3)
        eye = np.array([0.0, 1.0, -5.0], np.float32)
        for k in range(3):
            s = r[6 + 20 * k: 26 + 20 * k]
            d = rng.normal(size=3); d[2] = abs(d[2]) + 0.3; d /= np.linalg.norm(d)
            s[0:3] = (eye + rng.normal(scale=0.5, size=3) * (k > 0)).astype(np.float32).view(np.uint32)
            s[3] = np.float32(rng.uniform(0, 5)).view(np.uint32)
            s[4:7] = d.astype(np.float32).view(np.uint32)
            sky = rng.random() < 0.15
            s[7] = np.float32(np.inf if sky else rng.uniform(0.1, 30)).view(np.uint32)
            thp = rng.uniform(0, 1.3, 3); mv = rng.normal(scale=4, size=3)
            s[8:11] = pack2(thp, mv)
            rough = rng.choice([rng.uniform(0, 1), np.float32(0.25), np.nextafter(np.float32(0.25), np.float32(0)), np.nextafter(np.float32(0.25), np.float32(1)), rng.uniform(0, 0.2)])
            s[11] = (rng.integers(1, 8) << 16) | f16(rough)
            kind = rng.random()         # BSDF estimates: ordinary; a dark diffuse one the specular estimate alone lifts over the 0.05 albedo floor; both below the floor
            if kind < 0.25: est = (rng.uniform(0.0, 0.03, 3), rng.uniform(0.1, 1.0, 3))
            elif kind < 0.35: est = (rng.uniform(0.0, 0.02, 3), rng.uniform(0.0, 0.02, 3))
            else: est = (rng.uniform(0.04, 1.0, 3), rng.uniform(0.04, 1.0, 3))
            s[12:15] = pack2(*est)
            n = rng.normal(size=3); n /= np.linalg.norm(n)
            if rng.random() < 0.5: n = -d + rng.normal(scale=0.2, size=3); n /= np.linalg.norm(n)     # facing the camera (zObj > 0); else any direction, n.z < 0 included
            s[15] = oct_word(n) if rng.random() < 0.9 else rng.integers(0, 2**32, dtype=np.uint64)
            rad = rng.choice([0.0, rng.uniform(0, 2), rng.uniform(0, 50), 6000.0])
            radv = rng.uniform(0, 1, 3) * rad
            s[16] = f16(radv[0]) | (f16(radv[1]) << 16); s[17] = f16(radv[2]) | (f16(rng.uniform(0, 1) * rad) << 16)
            s[18] = s[19] = 0                  # FlagsAndVertexIndex, PackedCounters: the pass reads neither
        sr = rng.choice([0.0, rng.uniform(0, 1), rng.uniform(0, 100), 30000.0]) * rng.uniform(0, 1, 3)
        if i % 7 == 0: sr[:] = 0
        r[66] = f16(sr[0]) | (f16(sr[1]) << 16); r[67] = f16(sr[2]) | (f16(1.0) << 16)
        t = np.float32(0.001)
        r[68] = np.float32(rng.choice([0.0, t, np.nextafter(t, np.float32(0)), np.nextafter(t, np.float32(1)), rng.uniform(0, 0.002), rng.uniform(0, 50)])).view(np.uint32)
        mv = rng.normal(scale=3, size=2)
        r[69] = f16(mv[0]) | (f16(mv[1]) << 16)
        r[70:86] = cur.reshape(-1).view(np.uint32)
        r[86:102] = prevs[i % len(prevs)].reshape(-1).view(np.uint32)
        r[102:104] = np.float32([0.5 * W, -0.5 * H]).view(np.uint32)
    return recs


def main():
    inp = make()
    out = subprocess.run([KAT], input=inp.tobytes(), capture_output=True, check=True).stdout
    out = np.frombuffer(out, np.float32).reshape(len(inp), 15)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "dlss_rr_golden.npz"), inp=inp, out=out)
    print(len(inp), "records")


if __name__ == "__main__":
    main()
