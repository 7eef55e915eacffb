"""CPU: rigid-instance animation (SURVEY §8f row 4): the product's refit bodies (rtxpt_b200/csrc/refit.cuh, compiled for the host by tests/emu) on BVHs from the product's
builder.  The reference delegates this to the driver (BLAS / TLAS updates), so there is nothing of RTXPT's to restate; the refit is held to its own contract: unmoved
geometry gives back the built tree bit for bit, and after motion every quantised child box still encloses what lies under it - by at most one grid step.
GPU: tests/test_gpu_refit.py (-m gpu)."""
import ctypes as C
import numpy as np
import pytest
from rtxpt_b200 import structs as S


def _soup(n, rng, clusters=6):
    """Triangles in `clusters` groups (one instance each), object space."""
    inst = rng.integers(0, clusters, n)
    centre = rng.uniform(-10, 10, (clusters, 3))[inst]
    v0 = centre + rng.normal(0, 1.5, (n, 3)); e1 = rng.normal(0, 0.3, (n, 3)); e2 = rng.normal(0, 0.3, (n, 3))
    return np.concatenate([v0, v0 + e1, v0 + e2], 1).astype(np.float32), inst.astype(np.uint32)


def _shade_records(soup, inst):
    """triShade as the scene upload builds it: 6 uint4 per source triangle: object-space positions in [k].xyz, instance index in [5].y."""
    n = len(soup); rec = np.zeros((n, 6, 4), np.uint32)
    rec[:, 0:3, 0:3] = soup.reshape(n, 3, 3).view(np.uint32); rec[:, 5, 1] = inst
    return rec


def _instances(mats):
    arr = (S.InstanceData * len(mats))()
    for i, m in enumerate(mats): arr[i].transform[:] = np.float32(m).reshape(12).tolist(); arr[i].prevTransform[:] = np.float32(m).reshape(12).tolist()
    return arr


def _refit(emu, nodes, tris, rec, mats, levels):
    nodes = nodes.copy(); tris = tris.copy(); box = np.zeros((len(nodes), 6), np.float32); inst = _instances(mats)
    f = emu.lib().emu_refit; f.argtypes = [C.c_void_p] * 5 + [C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32]
    assert f(nodes.ctypes.data, tris.ctypes.data, rec.ctypes.data, C.cast(inst, C.c_void_p), box.ctypes.data, len(nodes), len(tris), levels.ctypes.data, len(levels) - 1) == 0
    return nodes, tris, box


def _decode_children(node):
    p = node[0:3].view(np.float32); e = np.uint32([node[3] & 0xFF, (node[3] >> 8) & 0xFF, (node[3] >> 16) & 0xFF]); imask = int(node[3] >> 24)
    meta = node[6:8].view(np.uint8); q = node[8:20].view(np.uint8).reshape(6, 8)
    scale = np.ldexp(1.0, e.astype(np.int64) - 127)
    out = []
    for s in range(8):
        if meta[s] == 0: continue
        lo = p + q[0:3, s] * scale; hi = p + q[3:6, s] * scale
        out.append((s, bool(imask >> s & 1), int(meta[s]), lo, hi, scale))
    return imask, out


def _check_tree(nodes, tris, box):
    """Every child box encloses its content (exactly conservative) and is tight to one grid step; every node's exact box is the union of its children's."""
    verts = tris.view(np.float32).reshape(-1, 3, 4)[:, :, :3]
    for ni, node in enumerate(nodes):
        imask, children = _decode_children(node)
        lo_all, hi_all = np.full(3, np.inf), np.full(3, -np.inf)
        for s, internal, meta, lo, hi, scale in children:
            if internal:
                ci = int(node[4]) + bin(imask & ((1 << s) - 1)).count("1"); clo, chi = box[ci, :3].astype(np.float64), box[ci, 3:].astype(np.float64)
            else:
                first = int(node[5]) + (meta & 31); cnt = bin(meta >> 5).count("1"); v = verts[first:first + cnt].reshape(-1, 3).astype(np.float64); clo, chi = v.min(0), v.max(0)
            assert (lo <= clo).all() and (hi >= chi).all(), (ni, s)
            q = node[8:20].view(np.uint8).reshape(6, 8)
            assert ((clo - lo <= scale * (1 + 1e-9)) | (q[0:3, s] == 0)).all() and ((hi - chi <= scale * (1 + 1e-9)) | (q[3:6, s] == 255)).all(), (ni, s)
            lo_all = np.minimum(lo_all, clo); hi_all = np.maximum(hi_all, chi)
        if children: assert np.array_equal(box[ni, :3], lo_all.astype(np.float32)) and np.array_equal(box[ni, 3:], hi_all.astype(np.float32)), ni


def test_refit_contract(product):
    import host_build_lib as emu
    rng = np.random.default_rng(5)
    soup, inst = _soup(6000, rng)
    nodes, tris, levels = product.debug_build_bvh(soup)
    assert levels[0] == 0 and levels[1] == 1 and levels[-1] == len(nodes) and (np.diff(levels.astype(np.int64)) > 0).all()
    assert np.array_equal(np.sort(tris[:, 3]), np.arange(len(soup)))                          # gid = soup index, each once
    rec = _shade_records(soup, inst)
    ident = [np.hstack([np.eye(3), np.zeros((3, 1))])] * 6
    n1, t1, b1 = _refit(emu, nodes, tris, rec, ident, levels)
    assert np.array_equal(n1, nodes) and np.array_equal(t1, tris)                              # unmoved: the builder's tree, bit for bit
    _check_tree(n1, t1, b1)
    # every instance moves: rotation about y + translation, one of them far away
    mats = []
    for k in range(6):
        a = 0.4 * k; R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]); t = rng.uniform(-3, 3, 3) + (40 if k == 5 else 0)
        mats.append(np.hstack([R, t[:, None]]))
    n2, t2, b2 = _refit(emu, nodes, tris, rec, mats, levels)
    assert np.array_equal(n2[:, 4:8], nodes[:, 4:8]) and np.array_equal(t2[:, [3, 7, 11]], tris[:, [3, 7, 11]])      # topology, metadata, ids untouched
    moved = np.einsum("nij,nkj->nki", np.float32(mats)[inst][:, :, :3], soup.reshape(-1, 3, 3)) + np.float32(mats)[inst][:, None, :, 3]
    got = t2.view(np.float32).reshape(-1, 3, 4)[:, :, :3]
    assert np.allclose(got, moved[t2[:, 3]], rtol=1e-5, atol=1e-5)
    _check_tree(n2, t2, b2)
    assert np.allclose(b2[0, :3], got.reshape(-1, 3).min(0)) and np.allclose(b2[0, 3:], got.reshape(-1, 3).max(0))    # the root follows the scene
    # moving back restores the original tree exactly (nothing accumulates)
    n3, t3, _ = _refit(emu, n2, t2, rec, ident, levels)
    assert np.array_equal(n3, nodes) and np.array_equal(t3, tris)


def test_refit_edge_cases(product):
    import host_build_lib as emu
    rng = np.random.default_rng(8)
    for n in (1, 2, 9, 70):
        soup, inst = _soup(n, rng, clusters=2)
        nodes, tris, levels = product.debug_build_bvh(soup)
        rec = _shade_records(soup, inst)
        flat = [np.hstack([np.diag([1.0, 0.0, 1.0]), np.array([[0.0], [2.0], [0.0]])])] * 2           # squashes everything into the plane y = 2: zero-extent axes
        n2, t2, b2 = _refit(emu, nodes, tris, rec, flat, levels)
        _check_tree(n2, t2, b2)
        assert (t2.view(np.float32).reshape(-1, 3, 4)[:, :, 1] == 2.0).all()
        # scale 0 on every axis (how hosts hide an instance): every triangle of it collapses onto the translation.  All instances collapsed: every node is a point box
        # with the smallest frame exponent (bvh8FrameExponent(0) = -126, stored biased as 1), zero child grid offsets and finite corners
        point = np.float32([3.5, -2.25, 7.0])
        collapsed = np.hstack([np.zeros((3, 3)), point[:, None]])
        n3, t3, b3 = _refit(emu, nodes, tris, rec, [collapsed] * 2, levels)
        _check_tree(n3, t3, b3)
        assert (t3.view(np.float32).reshape(-1, 3, 4)[:, :, :3] == point).all()
        assert np.isfinite(b3).all() and (b3[:, :3] == point).all() and (b3[:, 3:] == point).all()
        assert (n3[:, 0:3].view(np.float32) == point).all()
        assert ((n3[:, 3] & 0xFF) == 1).all() and (((n3[:, 3] >> 8) & 0xFF) == 1).all() and (((n3[:, 3] >> 16) & 0xFF) == 1).all()
        assert (n3[:, 8:20] == 0).all()
        assert np.array_equal(n3[:, 3] >> 24, nodes[:, 3] >> 24) and np.array_equal(n3[:, 4:8], nodes[:, 4:8])
        # one instance collapsed inside a moving scene: the tree stays conservative and the collapsed triangles sit on the point
        n4, t4, b4 = _refit(emu, nodes, tris, rec, [collapsed, flat[0]], levels)
        _check_tree(n4, t4, b4)
        assert np.isfinite(b4).all() and (t4.view(np.float32).reshape(-1, 3, 4)[inst[t4[:, 3]] == 0, :, :3] == point).all()
