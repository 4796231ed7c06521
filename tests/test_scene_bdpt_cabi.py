"""CPU: the bidirectional path tracer over two-level scenes has its own header (include/nanort_b200_scene_bdpt.h); the
library exports what it declares, the ctypes mirror lists exactly that, and the header stands alone as C and as C++
(no compute)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "nanort_b200_scene_bdpt.h")


def test_library_exports_every_scene_bdpt_symbol():
    from nanort_b200 import api

    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    names = sorted(set(re.findall(r"\b(nrt_[a-z0-9_]+)\s*\(", src)))
    assert sorted(api.SCENE_BDPT_EXPORTS) == names
    for other in (api.EXPORTS, api.SCENE_PATH_EXPORTS, api.BAKE_EXPORTS, api.BDPT_EXPORTS):
        assert not set(names) & set(other), "declared in one header only"
    L = ctypes.CDLL(api.LIB_PATH)
    for n in names:
        assert hasattr(L, n), n


@pytest.mark.parametrize("lang", ["c", "c++"])
def test_header_compiles_on_its_own(lang, tmp_path):
    cc = shutil.which("gcc" if lang == "c" else "g++")
    if cc is None:
        pytest.skip("no host compiler")
    src = tmp_path / ("t.c" if lang == "c" else "t.cc")
    src.write_text('#include "nanort_b200_scene_bdpt.h"\n'
                   "int main(void) {\n"
                   "  nrt_scene_shading s = {0, 0};\n"
                   "  nrt_bdpt_params p;\n"
                   "  p.max_bounces = 10;\n"
                   "  return (s.d_material_ids != 0) + (int)p.max_bounces +\n"
                   "         nrt_scene_render_bdpt_device(0, &p, &s, 0, 0, 0) +\n"
                   "         nrt_scene_bdpt_export_device(0, &p, &s, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0);\n"
                   "}\n")
    r = subprocess.run([cc, "-fsyntax-only", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
