"""TEST INFRASTRUCTURE ONLY: ctypes bindings of the two CPU builds of RTXPT's DLSS-RR input pass - the oracle's restatement (oracle/dlss_rr.mk, oracle/pt_dlss_rr.h) and the host
build of the product's pixel bodies (tests/emu/dlss_rr.mk) - with the same calling convention: `records` on single pixels in the layout of tests/golden/dlss_rr_golden.npz,
`frame` over a frame's realtime buffers as Context.readback_realtime returns them, giving what Context.readback_dlss_rr returns."""
import ctypes as C
import importlib.util
import os
import subprocess

import numpy as np

from rtxpt_b200 import structs as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "dlss_rr_golden.npz")
_libs = {}


def _load(which):
    if which not in _libs:
        if which == "oracle":
            subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "-f", "dlss_rr.mk"], check=True)
            L = C.CDLL(os.path.join(ROOT, "oracle", "_build", "dlss_rr", "liboracle_dlss_rr.so"))
            L.oracle_dlss_rr_records.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]; L.oracle_dlss_rr_records.restype = None
            L.oracle_dlss_rr_frame.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(S.RealtimeConstants), C.c_float, C.c_void_p] + [C.c_void_p] * 5
            L.oracle_dlss_rr_frame.restype = C.c_int
        else:
            subprocess.run(["make", "-C", os.path.join(ROOT, "tests", "emu"), "-s", "-f", "dlss_rr.mk"], check=True)
            L = C.CDLL(os.path.join(ROOT, "tests", "emu", "_build", "libdlss_rr_emu.so"))
            L.dlss_rr_emu_records.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]; L.dlss_rr_emu_records.restype = None
            L.dlss_rr_emu_frame.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(S.RealtimeConstants), C.c_float] + [C.c_void_p] * 10
            L.dlss_rr_emu_frame.restype = None
        _libs[which] = L
    return _libs[which]


def golden():
    g = np.load(GOLDEN)
    return g["inp"], g["out"]


def generator():
    """tests/golden/make_dlss_rr_golden.py as a module (record helpers: f16, pack2, oct_word, world_to_clip)."""
    spec = importlib.util.spec_from_file_location("make_dlss_rr_golden", os.path.join(ROOT, "tests", "golden", "make_dlss_rr_golden.py"))
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)
    return m


def records(which, inp):
    """15 floats per 104-word record: colour rgb, diffuse albedo, specular albedo, normal xyz + roughness, specular motion vector."""
    inp = np.ascontiguousarray(inp, np.uint32)
    out = np.zeros((len(inp), 15), np.float32)
    L = _load(which)
    (L.oracle_dlss_rr_records if which == "oracle" else L.dlss_rr_emu_records)(inp.ctypes.data, len(inp), out.ctypes.data)
    return out


def frame(which, rt, bufs, brightness_clamp_k=S.DLSS_RR_BRIGHTNESS_CLAMP_K):
    """bufs: planes, header, stable_radiance, motion, spec_hit_t as Context.readback_realtime returns them (motion: float16 [H, W, 4])."""
    H, W = bufs["spec_hit_t"].shape
    planes, header = np.ascontiguousarray(bufs["planes"]), np.ascontiguousarray(bufs["header"], np.uint32)
    sr, mv, sh = (np.ascontiguousarray(bufs["stable_radiance"], np.float16), np.ascontiguousarray(bufs["motion"], np.float16), np.ascontiguousarray(bufs["spec_hit_t"], np.float32))
    out = dict(color=np.zeros((H, W, 4), np.float16), diff_albedo=np.zeros((H, W), np.uint32), spec_albedo=np.zeros((H, W), np.uint32),
               normals_roughness=np.zeros((H, W, 4), np.float16), spec_motion=np.zeros((H, W, 2), np.float16))
    o = [out[k].ctypes.data for k in ("color", "diff_albedo", "spec_albedo", "normals_roughness", "spec_motion")]
    L = _load(which)
    if which == "oracle":
        targets = (C.c_void_p * 7)(planes.ctypes.data, header.ctypes.data, sr.ctypes.data, None, mv.ctypes.data, None, sh.ctypes.data)
        assert L.oracle_dlss_rr_frame(W, H, C.byref(rt), float(brightness_clamp_k), C.cast(targets, C.c_void_p), *o) == 0
    else:
        L.dlss_rr_emu_frame(W, H, C.byref(rt), float(brightness_clamp_k), planes.ctypes.data, header.ctypes.data, sr.ctypes.data, mv.ctypes.data, sh.ctypes.data, *o)
    return out



def mismatches(a, b, mask=None):
    """Per target, the pixels whose words differ between two DLSS-RR sets (fp16 words: a NaN equals any NaN - fp16 conversions keep different NaN payloads); mask: pixels to compare."""
    out = {}
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        if x.dtype == np.float16:
            same = (x.view(np.uint16) == y.view(np.uint16)) | (np.isnan(x) & np.isnan(y))
        else:
            same = x == y
        if same.ndim == 3: same = same.all(-1)
        if mask is not None: same = same | ~mask
        out[k] = int((~same).sum())
    return out
