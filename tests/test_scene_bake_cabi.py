"""CPU: the scene bakes have their own header (include/nanort_b200_scene_bake.h); the library exports what it declares,
the ctypes mirror lists exactly that with the header's chart layout, and the header stands alone as C and as C++ (no
compute)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "nanort_b200_scene_bake.h")


def test_library_exports_every_scene_bake_symbol():
    from nanort_b200 import api

    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    names = sorted(set(re.findall(r"\b(nrt_[a-z0-9_]+)\s*\(", src)))
    assert sorted(api.SCENE_BAKE_EXPORTS) == names
    for other in (api.EXPORTS, api.SCENE_PATH_EXPORTS, api.BAKE_EXPORTS, api.BDPT_EXPORTS, api.SCENE_BDPT_EXPORTS,
                  api.LIGHTMAP_EXPORTS):
        assert not set(names) & set(other), "declared in one header only"
    L = ctypes.CDLL(api.LIB_PATH)
    for n in names:
        assert hasattr(L, n), n


def test_chart_mirror_has_the_header_layout(tmp_path):
    from nanort_b200 import api

    cc = shutil.which("gcc")
    if cc is None:
        pytest.skip("no host compiler")
    t, cls = "nrt_scene_chart", api.SceneChart
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "nanort_b200_scene_bake.h"', "int main(void) {",
             f'  printf("%zu", sizeof({t}));']
    for f, _ in cls._fields_:
        lines.append(f'  printf(" {f}=%zu", offsetof({t}, {f}));')
    lines.append("  return 0; }")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines) + "\n")
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    size, *rest = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert ctypes.sizeof(cls) == int(size)
    assert [(f, getattr(cls, f).offset) for f, _ in cls._fields_] == [(kv.split("=")[0], int(kv.split("=")[1]))
                                                                      for kv in rest]
    assert ctypes.sizeof(cls) == cls.flip_y.offset + 4  # no tail the mirror misses


@pytest.mark.parametrize("lang", ["c", "c++"])
def test_header_compiles_on_its_own(lang, tmp_path):
    cc = shutil.which("gcc" if lang == "c" else "g++")
    if cc is None:
        pytest.skip("no host compiler")
    src = tmp_path / ("t.c" if lang == "c" else "t.cc")
    src.write_text('#include "nanort_b200_scene_bake.h"\n'
                   "int main(void) {\n"
                   "  nrt_scene_chart c = {0};\n"
                   "  nrt_bake_params b = {0};\n"
                   "  nrt_bake_result br = {0};\n"
                   "  nrt_lightmap_params p = {0};\n"
                   "  nrt_lightmap_result r = {0};\n"
                   "  nrt_scene_shading sh = {0};\n"
                   "  uint64_t n = 0;\n"
                   "  c.width = 4;\n"
                   "  return (int)(c.width + r.traverse_launches + br.launches) +\n"
                   "         nrt_scene_uv_raster_device(0, &c, 4, 4, 0, &sh, 0, 0, 0, 0, &n, 0) +\n"
                   "         nrt_scene_bake_ao_device(0, 0, 0, &sh, &b, 0, &br, 0) +\n"
                   "         nrt_scene_bake_ao_rays_device(0, 0, 0, &sh, &b, 0, 0, &n, 0) +\n"
                   "         nrt_scene_bake_lightmap_device(0, 0, 0, &p, &sh, 0, &r, 0) +\n"
                   "         nrt_scene_bake_lightmap_bounce_device(0, 0, 0, &p, &sh, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,\n"
                   "                                               0, 0, &n, &n, 0, 0);\n"
                   "}\n")
    r = subprocess.run([cc, "-fsyntax-only", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
