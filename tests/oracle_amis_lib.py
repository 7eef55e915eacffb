"""ctypes binding of oracle/_build/amis/liboracle_amis.so — TEST INFRASTRUCTURE ONLY: the oracle with RtxptPathTracerConstants::useApproximateMIS honoured (oracle/amis.mk).

The library exports liboracle.so's entry points, so this is oracle_lib.py loaded a second time as its own module with the library path swapped: `Oracle`, `lib()` and the
rest behave as there.  With the switch at 0 the library computes what liboracle.so computes."""
import importlib.util
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build():
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "-f", "amis.mk"], check=True)


def _load():
    spec = importlib.util.spec_from_file_location("oracle_lib_amis", os.path.join(ROOT, "tests", "oracle_lib.py"))
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)
    m.LIB_PATH = os.path.join(ROOT, "oracle", "_build", "amis", "liboracle_amis.so")
    m.build = build
    return m


oracle = _load()
