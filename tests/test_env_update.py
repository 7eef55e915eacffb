"""CPU: the importance / radiance map that rtxpt_b200_update_env_map builds on the GPU (rtxpt_b200/csrc/envbake.cuh: importanceTexel, importanceReduceTexel), compiled for the host
by tests/emu, equals the oracle's LightBaker::buildEnvRadianceMap bit for bit on random, constant and seam-heavy cubes.  On the GPU only libdevice's cos / sin differ from the
host's: tests/test_gpu_env_update.py (-m gpu) measures that."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest

IMPORTANCE_FLOATS = sum((1024 >> m) ** 2 * 4 for m in range(11))
EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
EMU_LIB, ORACLE_ENV_LIB = os.path.join(EMU, "_build", "libenv_update_emu.so"), os.path.join(EMU, "_build", "liboracle_env.so")
_libs = {}


def env_lib(path):
    """One of the two test libraries of tests/emu/env_update.mk (built by build(); made here when missing)."""
    if path not in _libs:
        if not os.path.exists(path):
            subprocess.run(["make", "-C", EMU, "-s", "-f", "env_update.mk", os.path.relpath(path, EMU)], check=True)
        _libs[path] = C.CDLL(path)
    return _libs[path]


def _chain(L, name, cube):
    cube = np.ascontiguousarray(cube, np.float32); n = cube.shape[1]
    out = np.zeros(IMPORTANCE_FLOATS, np.float32)
    f = getattr(L, name); f.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p]; f.restype = C.c_int
    assert f(n, cube.ctypes.data, out.ctypes.data) == 0
    return out


def _cubes():
    rng = np.random.default_rng(11)
    yield "random16", rng.gamma(2.0, 0.5, (6, 16, 16, 4)).astype(np.float32)
    yield "random256", rng.gamma(1.5, 2.0, (6, 256, 256, 4)).astype(np.float32)
    const = np.zeros((6, 64, 64, 4), np.float32); const[..., :3] = (0.75, 1.5, 3.25); const[..., 3] = 1
    yield "constant64", const
    # seam-heavy: every face its own level, a one-texel frame of a different level along its edges and a checkerboard inside, so that every clamp at a face border and every
    # face selection near an edge or corner of the cube decides texels
    n = 32; seam = np.zeros((6, n, n, 4), np.float32)
    yy, xx = np.mgrid[0:n, 0:n]
    for f in range(6):
        seam[f, ..., :3] = np.float32([0.1 + f, 2.0 + 0.5 * f, 7.0 - f])
        seam[f][((xx + yy) & 1) == 1, :3] *= 3.0
        for e in (seam[f, 0], seam[f, -1], seam[f, :, 0], seam[f, :, -1]): e[:, :3] = 60000.0 / (f + 1)
    yield "seam32", seam
    yield "bright128", (rng.random((6, 128, 128, 4)) ** 8 * 5e4).astype(np.float32)


@pytest.mark.parametrize("name,cube", list(_cubes()), ids=lambda v: v if isinstance(v, str) else "")
def test_importance_bodies_equal_the_oracle(name, cube):
    want = _chain(env_lib(ORACLE_ENV_LIB), "oracle_env_radiance_map", cube)
    got = _chain(env_lib(EMU_LIB), "emu_env_importance_map", cube)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, int((got != want).sum()), np.abs(got - want).max())
    assert np.array_equal(got, got.astype(np.float16).astype(np.float32))          # the RGBA16F target's rounding
    assert got[3::4].min() > 0                                                      # every texel of every MIP carries importance
