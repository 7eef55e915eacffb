"""ctypes binding of oracle/_build/stf/liboracle_stf.so — TEST INFRASTRUCTURE ONLY: the oracle with stochastic texture filtering honoured (oracle/stf.mk, oracle/pt_stf.h).

The library exports liboracle.so's entry points plus oracle_set_texture_filtering, so this is oracle_lib.py loaded a second time as its own module with the library path swapped,
and `set_texture_filtering(o, ...)` for an `Oracle` of it.  With STF off the library computes what liboracle.so computes."""
import ctypes as C
import importlib.util
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build():
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "-f", "stf.mk"], check=True)


def _load():
    spec = importlib.util.spec_from_file_location("oracle_lib_stf", os.path.join(ROOT, "tests", "oracle_lib.py"))
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)
    m.LIB_PATH = os.path.join(ROOT, "oracle", "_build", "stf", "liboracle_stf.so")
    m.build = build
    return m


oracle = _load()


def set_texture_filtering(o, enable=True, filter_type=1, gaussian_sigma=0.3):
    from rtxpt_b200 import structs as S
    L = oracle.lib()
    L.oracle_set_texture_filtering.argtypes = [C.c_void_p, C.POINTER(S.StochasticTextureFiltering)]
    assert L.oracle_set_texture_filtering(o.h, C.byref(S.StochasticTextureFiltering(int(enable), filter_type, 0, gaussian_sigma))) == 0
