"""CPU: the path tracer over two-level scenes has its own header (include/nanort_b200_scene_path.h); the library exports
what it declares, the ctypes mirror lists exactly that, and the header stands alone as C and as C++ (no compute)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "nanort_b200_scene_path.h")


def test_library_exports_every_scene_path_symbol():
    from nanort_b200 import api

    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    names = sorted(set(re.findall(r"\b(nrt_[a-z0-9_]+)\s*\(", src)))
    assert sorted(api.SCENE_PATH_EXPORTS) == names
    assert not set(names) & set(api.EXPORTS), "declared in one header only"
    L = ctypes.CDLL(api.LIB_PATH)
    for n in names:
        assert hasattr(L, n), n


def test_scene_shading_mirror_has_the_header_layout():
    from nanort_b200 import api

    assert ctypes.sizeof(api.SceneShading) == 2 * ctypes.sizeof(ctypes.c_void_p)
    assert [f for f, _ in api.SceneShading._fields_] == ["d_material_ids", "d_facevarying_normals"]


@pytest.mark.parametrize("lang", ["c", "c++"])
def test_header_compiles_on_its_own(lang, tmp_path):
    cc = shutil.which("gcc" if lang == "c" else "g++")
    if cc is None:
        pytest.skip("no host compiler")
    src = tmp_path / ("t.c" if lang == "c" else "t.cc")
    src.write_text('#include "nanort_b200_scene_path.h"\nint main(void) { nrt_scene_shading s = {0, 0}; return s.d_material_ids != 0; }\n')
    r = subprocess.run([cc, "-fsyntax-only", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
