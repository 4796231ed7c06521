"""Error behaviour of the C-ABI: bad arguments come back as error codes with a message, never as a crash or a
silent fallback (reference behaviour cited per case)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _tri():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    return v, np.array([[0, 1, 2]], np.uint32)


def test_build_rejects_bad_options():
    from nanort_b200 import api

    v, f = _tri()
    L = api.lib()
    h = C.c_void_p()
    # Build returns false for zero primitives (nanort.h:1907-1909)
    assert L.nrt_build(api._p(v), 12, 3, api._p(f), 0, None, C.byref(h)) == -1 and not h.value
    assert b"num_primitives" in L.nrt_last_error()
    for okw, needle in ((dict(bin_size=1), b"bin_size"),          # the reference asserts bin_size > 1 (nanort.h:1905)
                        (dict(bin_size=512), b"bin_size"),        # implementation limit
                        (dict(max_tree_depth=600), b"max_tree_depth")):  # 512-entry traversal stack
        with pytest.raises(api.NanortB200Error) as e:
            api.BVHAccel().Build(1, v, f, api.BVHBuildOptions(**okw))
        assert needle in str(e.value).encode()
    assert L.nrt_build(None, 12, 3, api._p(f), 1, None, C.byref(h)) == -1
    assert L.nrt_build(api._p(v), 8, 3, api._p(f), 1, None, C.byref(h)) == -1  # stride smaller than a float3


def test_adopt_rejects_malformed_trees():
    from nanort_b200 import api, scenes as S

    v, f = S.make_scene("cornell")
    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    nodes, idx = acc.GetNodes(), acc.GetIndices()
    bad = nodes.copy()
    br = np.nonzero(bad["flag"] == 0)[0][0]
    bad["data"][br, 0] = len(bad) + 5  # child outside the array
    with pytest.raises(api.NanortB200Error):
        api.BVHAccel().Adopt(bad, idx, v, f)
    bad = nodes.copy()
    bad["data"][br, 1] = br  # cycle
    with pytest.raises(api.NanortB200Error):
        api.BVHAccel().Adopt(bad, idx, v, f)
    bad_idx = idx.copy()
    bad_idx[0] = len(f) + 7  # primitive id outside the mesh
    with pytest.raises(api.NanortB200Error):
        api.BVHAccel().Adopt(nodes, bad_idx, v, f)
    leaf = np.nonzero(nodes["flag"] == 1)[0][0]
    bad = nodes.copy()
    bad["data"][leaf, 0] = len(f) + 1  # leaf range outside indices_
    with pytest.raises(api.NanortB200Error):
        api.BVHAccel().Adopt(bad, idx, v, f)


def test_traverse_and_render_reject_null_and_bad_tiles():
    import torch
    from nanort_b200 import api

    v, f = _tri()
    acc = api.BVHAccel()
    acc.Build(1, v, f)
    L = api.lib()
    assert L.nrt_traverse(acc._h, None, 5, None, None, None, 0) == -1
    assert L.nrt_traverse(acc._h, None, 0, None, None, None, 0) == 0  # zero rays is a no-op
    p = api.AoParams()
    p.width, p.height, p.spp, p.tile_w, p.tile_h, p.n_shards = 64, 64, 1, 60, 8, 1  # tile_w not a multiple of 8
    accum = torch.zeros(64 * 64, device="cuda")
    with pytest.raises(api.NanortB200Error):
        acc.RenderAO(p, accum.data_ptr())
    p.tile_w, p.shard, p.n_shards = 64, 3, 2  # shard outside the shard count
    with pytest.raises(api.NanortB200Error):
        acc.RenderAO(p, accum.data_ptr())
    # a non-zero value in the reserved flags bits 8..15 is refused, not ignored
    rays = np.zeros(4, np.dtype([("o", "<f4", 3), ("d", "<f4", 3), ("a", "<f4"), ("b", "<f4"), ("t", "<u4")]))
    for sel in (1, 100, 200):
        with pytest.raises(api.NanortB200Error):
            acc.Traverse(rays, flags=(sel << 8))
    # the same for the two-level scene's production walk (a shallow scene: the deep-stack and list-only walks
    # ignore those bits)
    sc = api.Scene()
    sc.AddNode(acc, np.eye(4, dtype=np.float32))
    assert sc.Commit()
    rays["o"] = (0.2, 0.2, -1.0)
    rays["d"] = (0.0, 0.0, 1.0)
    rays["b"] = 1e30
    h, m = sc.Traverse(rays)
    assert m.all()
    with pytest.raises(api.NanortB200Error):
        sc.Traverse(rays, flags=(2 << 8))
