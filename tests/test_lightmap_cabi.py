"""CPU: the lightmap bake has its own header (include/nanort_b200_lightmap.h); the library exports what it declares, the
ctypes mirror lists exactly that with the header's struct layouts, and the header stands alone as C and as C++ (no
compute)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "nanort_b200_lightmap.h")


def test_library_exports_every_lightmap_symbol():
    from nanort_b200 import api

    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    names = sorted(set(re.findall(r"\b(nrt_[a-z0-9_]+)\s*\(", src)))
    assert sorted(api.LIGHTMAP_EXPORTS) == names
    for other in (api.EXPORTS, api.SCENE_PATH_EXPORTS, api.BAKE_EXPORTS, api.BDPT_EXPORTS, api.SCENE_BDPT_EXPORTS):
        assert not set(names) & set(other), "declared in one header only"
    L = ctypes.CDLL(api.LIB_PATH)
    for n in names:
        assert hasattr(L, n), n


def test_struct_mirrors_have_the_header_layout(tmp_path):
    from nanort_b200 import api

    cc = shutil.which("gcc")
    if cc is None:
        pytest.skip("no host compiler")
    types = {"nrt_lightmap_params": api.LightmapParams, "nrt_lightmap_result": api.LightmapResult}
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "nanort_b200_lightmap.h"', "int main(void) {"]
    for t, cls in types.items():
        lines.append(f'  printf("{t} %zu", sizeof({t}));')
        for f, _ in cls._fields_:
            lines.append(f'  printf(" {f}=%zu", offsetof({t}, {f}));')
        lines.append('  printf("\\n");')
    lines.append("  return 0; }")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines) + "\n")
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = {}
    for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines():
        t, size, *rest = line.split()
        got[t] = (int(size), [(kv.split("=")[0], int(kv.split("=")[1])) for kv in rest])
    for t, cls in types.items():
        size, offsets = got[t]
        assert ctypes.sizeof(cls) == size, t
        assert [(f, getattr(cls, f).offset) for f, _ in cls._fields_] == offsets, t
    # every field of the C struct is mirrored: the last field ends where the struct does (no tail the mirror misses)
    assert ctypes.sizeof(api.LightmapParams) == api.LightmapParams.pad.offset + 4
    assert ctypes.sizeof(api.LightmapResult) == api.LightmapResult.traverse_launches.offset + 4


@pytest.mark.parametrize("lang", ["c", "c++"])
def test_header_compiles_on_its_own(lang, tmp_path):
    cc = shutil.which("gcc" if lang == "c" else "g++")
    if cc is None:
        pytest.skip("no host compiler")
    src = tmp_path / ("t.c" if lang == "c" else "t.cc")
    src.write_text('#include "nanort_b200_lightmap.h"\n'
                   "int main(void) {\n"
                   "  nrt_lightmap_params p = {0};\n"
                   "  nrt_lightmap_result r = {0};\n"
                   "  p.max_bounces = 4;\n"
                   "  return (int)(p.max_bounces + r.traverse_launches) +\n"
                   "         nrt_bake_lightmap_device(0, 0, &p, 0, &r, 0) +\n"
                   "         nrt_bake_lightmap_bounce_device(0, 0, &p, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,\n"
                   "                                         0);\n"
                   "}\n")
    r = subprocess.run([cc, "-fsyntax-only", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
