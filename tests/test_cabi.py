"""CPU: the C-ABI library loads and exports every symbol include/nanort_b200.h declares (no compute)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "nanort_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(nrt_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from nanort_b200 import api

    names = _declared()
    assert len(names) >= 14
    assert sorted(api.EXPORTS) == names, "api.EXPORTS must list exactly the header's entry points"
    L = ctypes.CDLL(api.LIB_PATH)
    for n in names:
        assert hasattr(L, n), n


def test_record_sizes_match_reference_layouts():
    from nanort_b200 import api, scenes

    assert scenes.RAY_DTYPE.itemsize == 36 and scenes.HIT_DTYPE.itemsize == 16 and scenes.NODE_DTYPE.itemsize == 40
    assert api.BUILD_OPT_DTYPE.itemsize == 28 and api.TRACE_OPT_DTYPE.itemsize == 16 and api.STATS_DTYPE.itemsize == 16
    o = api.BVHBuildOptions()
    assert (o["min_leaf_primitives"][0], o["max_tree_depth"][0], o["bin_size"][0]) == (4, 256, 64)
    t = api.BVHTraceOptions()
    assert tuple(t["prim_ids_range"][0]) == (0, 0x7FFFFFFF) and t["skip_prim_id"][0] == 0xFFFFFFFF


def test_no_cpu_fallback_without_device():
    """On a box without a GPU every compute entry point must fail loudly (never fall back)."""
    import numpy as np
    import pytest
    from nanort_b200 import api

    if api.lib().nrt_device_count() > 0:
        pytest.skip("a CUDA device is present")
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    f = np.array([[0, 1, 2]], np.uint32)
    with pytest.raises(api.NanortB200Error):
        api.BVHAccel().Build(1, v, f)


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "nanort_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, fn)).read()
                assert "import oracle" not in txt and "from oracle" not in txt and "liborc" not in txt, fn


def test_python_mirror_constants_equal_the_header_defines():
    """The ctypes mirror's flag constants are the header's #defines (a drifted constant would silently select another
    kernel or record layout), and the mirrored structs have the header's sizes."""
    import ctypes as C
    from nanort_b200 import api

    src = open(os.path.join(ROOT, "include", "nanort_b200.h")).read()
    defs = {m.group(1): int(m.group(2).rstrip("u"), 0) for m in re.finditer(r"#define\s+(NRT_[A-Z0-9_]+)\s+(-?(?:0x[0-9A-Fa-f]+|\d+)u?)\b", src)}
    pairs = {"NRT_TRAVERSE_FAST": api.TRAVERSE_FAST, "NRT_TRAVERSE_CONFORMANCE": api.TRAVERSE_CONFORMANCE,
             "NRT_TRAVERSE_CPP03_INVERSE": api.TRAVERSE_CPP03_INVERSE, "NRT_TRAVERSE_RAY32": api.TRAVERSE_RAY32,
             "NRT_TRAVERSE_ANY_HIT": api.TRAVERSE_ANY_HIT, "NRT_AO_UNFUSED": api.AO_UNFUSED,
             "NRT_AO_PACKED_TILES": api.AO_PACKED_TILES, "NRT_BUILD_FAST": api.BUILD_FAST,
             "NRT_BUILD_REFERENCE_TREE": api.BUILD_REFERENCE_TREE, "NRT_PRIM_SPHERES": api.PRIM_SPHERES,
             "NRT_PRIM_BOXES": api.PRIM_BOXES}
    for name, value in pairs.items():
        assert name in defs, name
        assert defs[name] == value, (name, defs[name], value)
    # the traverse flag bits do not collide with each other or with the reserved bits 8..15
    bits = [defs[n] for n in ("NRT_TRAVERSE_CONFORMANCE", "NRT_TRAVERSE_CPP03_INVERSE", "NRT_TRAVERSE_RAY32", "NRT_TRAVERSE_ANY_HIT")]
    assert len(set(bits)) == 4 and all(b & (b - 1) == 0 and b < 0x100 for b in bits)
    assert defs["NRT_AO_UNFUSED"] > 0xFFFF and defs["NRT_AO_PACKED_TILES"] > 0xFFFF
    # struct sizes the header documents
    assert C.sizeof(api.AoResult) == 48 and C.sizeof(api.AoParams) == 104
