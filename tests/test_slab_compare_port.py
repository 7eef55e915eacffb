"""The traversal's node step on the CPU: the integer slab compare and the packed hit-word build of traverse.cuh (nodeHitMask) against the float formulation they replaced.

tests/emu/slab_compare_host_emu.cu compiles the product's function for the host and keeps the earlier formulation as the reference; both are run over every node of the host
builder's tree of the small city and a few thousand rays - random ones, origins on the geometry (inside leaf boxes), origins outside the scene looking away (every box behind
the ray), axis-parallel and signed-zero directions, tiny and huge tMax.  The hit word has to be the same on every (node, ray) pair: same children entered, same bits, same order."""
import ctypes as C
import os
import subprocess
import sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def _lib():
    subprocess.run(["make", "-C", os.path.join(ROOT, "tests", "emu"), "-s", "-f", "slab_compare.mk"], check=True)
    L = C.CDLL(os.path.join(ROOT, "tests", "emu", "_build", "libslab_compare_emu.so"))
    L.emu_slab_compare.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.POINTER(C.c_uint64)]; L.emu_slab_compare.restype = C.c_uint64
    return L


def _compare(L, nodes, rays, tmin_zero):
    nodes = np.ascontiguousarray(nodes, np.uint32); rays = np.ascontiguousarray(rays, np.float32)
    first = np.zeros(4, np.uint32); hits = C.c_uint64()
    bad = L.emu_slab_compare(nodes.ctypes.data, len(nodes), rays.ctypes.data, len(rays), int(tmin_zero), first.ctypes.data, C.byref(hits))
    return bad, hits.value, first


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _rays(tris, rng, n):
    """n x 8 float32 (origin, tMin = 0, direction, tMax), a seventh each of the kinds the docstring lists."""
    v = tris.reshape(-1, 3); lo, hi = v.min(0), v.max(0); k = n // 7
    r = np.zeros((7 * k, 8), np.float32)
    r[:, :3] = rng.uniform(lo, hi, (7 * k, 3)); r[:, 4:7] = _unit(rng.normal(size=(7 * k, 3))); r[:, 7] = 1e15
    r[k:2 * k, :3] = v[rng.integers(0, len(v), k)]                                                        # on a vertex: inside the leaf's box, on faces of the quantisation grid
    r[2 * k:3 * k, :3] = tris.reshape(-1, 3, 3)[rng.integers(0, len(tris), k)].mean(1)                    # on a triangle
    out = _unit(rng.normal(size=(k, 3))); r[3 * k:4 * k, :3] = (lo + hi) / 2 + out * np.linalg.norm(hi - lo); r[3 * k:4 * k, 4:7] = out      # outside, looking away
    axes = np.eye(3, dtype=np.float32)[rng.integers(0, 3, k)] * rng.choice([-1.0, 1.0], (k, 1))
    r[4 * k:5 * k, 4:7] = axes * rng.choice([-1.0, 1.0], (k, 3))                                          # axis-parallel, the zeros of either sign
    two = _unit(rng.normal(size=(k, 3)) * (np.arange(3) != rng.integers(0, 3, (k, 1)))); r[5 * k:6 * k, 4:7] = two      # one component exactly zero
    r[5 * k:6 * k:2, :3] = v[rng.integers(0, len(v), (k + 1) // 2)]
    r[6 * k:, 7] = 10.0 ** rng.uniform(-6, 1, k)                                                           # short rays: bestT decides
    r[6 * k::3, :3] = v[rng.integers(0, len(v), len(r[6 * k::3]))]
    return r


def test_hit_word_of_the_integer_compare_equals_the_float_formulation(product, small_city):
    from bvh_quality import scene_triangles
    L = _lib()
    tris = scene_triangles(small_city[0]).reshape(-1, 9)
    nodes, _, _ = product.debug_build_bvh(tris)
    rays = _rays(tris, np.random.default_rng(77), 2800)
    bad, hits, first = _compare(L, nodes, rays, True)
    assert bad == 0, "node %d ray %d: reference %08x, product %08x" % tuple(first)
    assert hits > 4 * len(rays) and len(nodes) > 10000                  # the pairs are not all misses: a ray enters several nodes per level of the tree


def test_general_interval_keeps_the_float_compare(product, small_city):
    """k_trace_rays' instantiation: any tMin, negative included (then boxes behind the origin are entered) - word for word the reference on the same pairs."""
    from bvh_quality import scene_triangles
    L = _lib()
    tris = scene_triangles(small_city[0]).reshape(-1, 9)
    nodes, _, _ = product.debug_build_bvh(tris)
    rng = np.random.default_rng(78)
    rays = _rays(tris, rng, 700); rays[:, 3] = rng.choice([0.0, -1.0, -1e3, 1e-3, 5.0], len(rays)).astype(np.float32)
    bad, hits, first = _compare(L, nodes[::4], rays, False)
    assert bad == 0, "node %d ray %d: reference %08x, product %08x" % tuple(first)
    behind = rays[:, 3] < 0
    assert _compare(L, nodes[::4], rays[behind], False)[1] > _compare(L, nodes[::4], np.c_[rays[behind, :3], np.zeros(behind.sum(), np.float32), rays[behind, 4:]], False)[1]
