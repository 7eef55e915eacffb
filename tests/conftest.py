import os
import sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with `-m gpu`)")
    config.addinivalue_line("markers", "gpu_unverified: GPU tests of code that has compiled but not yet run on an H100 (select with `-m gpu_unverified`); skipped without a device")


def pytest_collection_modifyitems(config, items):
    def cuda_device_present():
        import ctypes
        try:
            cu = ctypes.CDLL("libcuda.so.1"); n = ctypes.c_int(0)
            return cu.cuInit(0) == 0 and cu.cuDeviceGetCount(ctypes.byref(n)) == 0 and n.value > 0
        except OSError:
            return False
    have_gpu = cuda_device_present()
    for item in items:
        if "gpu_unverified" in item.keywords and (not have_gpu or config.getoption("-m") != "gpu_unverified"):
            item.add_marker(pytest.mark.skip(reason="not yet verified on a GPU; run with -m gpu_unverified on an H100"))


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle library (test infrastructure; built on demand with g++)."""
    import oracle_lib
    oracle_lib.build()
    return oracle_lib


@pytest.fixture(scope="session")
def product():
    """The CUDA product library; GPU tests fail loudly if it is missing or no device is present."""
    from rtxpt_b200 import lib
    lib.load()
    return lib


@pytest.fixture(scope="session")
def cornell():
    from rtxpt_b200 import scenes
    return scenes.cornell_box(256, 256)


@pytest.fixture(scope="session")
def small_city():
    from rtxpt_b200 import scenes
    return scenes.city_block(target_triangles=120000, width=320, height=180, texture_size=128, n_textures=6, n_materials=64)
