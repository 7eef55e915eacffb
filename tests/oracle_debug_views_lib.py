"""ctypes binding of oracle/_build/debug_views/liboracle_debug_views.so — TEST INFRASTRUCTURE ONLY: the oracle plus RTXPT's debug views (oracle/debug_views.mk,
oracle/pt_debug_views.h).  The library exports liboracle.so's entry points too, so this is oracle_lib.py loaded a second time as its own module with the library path swapped,
plus the debug-view entries for an `Oracle` of it."""
import ctypes as C
import importlib.util
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build():
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "-f", "debug_views.mk"], check=True)


def _load():
    spec = importlib.util.spec_from_file_location("oracle_lib_debug_views", os.path.join(ROOT, "tests", "oracle_lib.py"))
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)
    m.LIB_PATH = os.path.join(ROOT, "oracle", "_build", "debug_views", "liboracle_debug_views.so")
    m.build = build
    return m


oracle = _load()


def _lib():
    from rtxpt_b200 import structs as S
    L = oracle.lib()
    L.oracle_debug_first_hit.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_int]
    L.oracle_debug_stable_planes.argtypes = [C.c_void_p, C.POINTER(S.RealtimeConstants), C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p]
    L.oracle_debug_first_hit_records.argtypes = [C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
    return L


def first_hit(o, view, sample_index):
    """surfaceDebugViz at vertex 1 of every pixel's camera ray of `sample_index`: float32 [H, W, 4], 0 where the ray misses"""
    W, H = o.consts.imageWidth, o.consts.imageHeight
    out = np.zeros((H, W, 4), np.float32)
    assert _lib().oracle_debug_first_hit(o.h, view, sample_index, out.ctypes.data, 0) == 0
    return out


def stable_planes(o, rt, view, plane_index, realtime):
    """StablePlanesDebugViz over the targets of Oracle.render_realtime (or the library's, in the same layout): float32 [H, W, 4], 0 where nothing is drawn"""
    W, H = o.consts.imageWidth, o.consts.imageHeight
    out = np.zeros((H, W, 4), np.float32)
    r = o._ptr_table([realtime[n] for n in ("planes", "header", "stable_radiance", "depth", "motion", "throughput", "spec_hit_t")])
    assert _lib().oracle_debug_stable_planes(o.h, C.byref(rt), view, int(plane_index), r, out.ctypes.data) == 0
    return out


def first_hit_records(view, records):
    """surfaceDebugViz on surfaces given as records of 28 words (see oracle/debug_views_oracle.cpp): float32 [N, 4]"""
    records = np.ascontiguousarray(records, np.uint32)
    out = np.zeros((len(records), 4), np.float32)
    _lib().oracle_debug_first_hit_records(view, records.ctypes.data, len(records), out.ctypes.data)
    return out


def pixel_funcs(records):
    """the colour functions on records of (op, a, b, c) as oracle/ref_kat_debug_main.cpp takes them: uint32 [N, 3]"""
    records = np.ascontiguousarray(records, np.uint32)
    out = np.zeros((len(records), 3), np.uint32)
    L = oracle.lib(); L.oracle_debug_pixel_funcs.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    L.oracle_debug_pixel_funcs(records.ctypes.data, len(records), out.ctypes.data)
    return out


def denoiser_merge(o, rt, plane, dbg_plane_index, view, realtime, denoiser, denoised_diff, denoised_spec, viz):
    """the final merge's debug views of `plane` drawn into `viz` (float32 [H, W, 4], kept where the merge draws nothing); targets as for Oracle.denoiser_final_merge"""
    from rtxpt_b200 import structs as S
    L = oracle.lib()
    L.oracle_debug_denoiser_merge.argtypes = [C.c_void_p, C.POINTER(S.RealtimeConstants), C.c_uint32, C.c_int32, C.c_uint32] + [C.c_void_p] * 5
    r = o._ptr_table([realtime[n] for n in ("planes", "header", "stable_radiance", "depth", "motion", "throughput", "spec_hit_t")])
    d = o._ptr_table([denoiser[n] for n in ("view_z", "motion", "normal_roughness", "diff", "spec", "disocclusion_mix", "history_clamp_relax", "output")])
    dd = np.ascontiguousarray(denoised_diff, np.float16); ds = np.ascontiguousarray(denoised_spec, np.float16)
    assert viz.dtype == np.float32 and viz.flags.c_contiguous
    assert L.oracle_debug_denoiser_merge(o.h, C.byref(rt), plane, int(dbg_plane_index), view, r, d, dd.ctypes.data, ds.ctypes.data, viz.ctypes.data) == 0
