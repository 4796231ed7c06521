"""CPU: texture-space baking has its own header (include/nanort_b200_bake.h); the library exports what it declares, the
ctypes mirror lists exactly that with the header's struct layouts, the header stands alone as C and as C++, and the
numpy restatement of the texel ray (tests/bake_model.py: texel_rays) equals the reference uv_raster's expression
(examples/uv_raster/main.cc:752-770) compiled as C (no compute on a GPU)."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import bake_model as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "nanort_b200_bake.h")


def test_library_exports_every_bake_symbol():
    from nanort_b200 import api

    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    names = sorted(set(re.findall(r"\b(nrt_[a-z0-9_]+)\s*\(", src)))
    assert sorted(api.BAKE_EXPORTS) == names
    assert not set(names) & set(api.EXPORTS), "declared in one header only"
    assert not set(names) & set(api.SCENE_PATH_EXPORTS), "declared in one header only"
    L = ctypes.CDLL(api.LIB_PATH)
    for n in names:
        assert hasattr(L, n), n


def _c_layout(tmp_path, cc):
    """sizeof and field offsets of the header's structs, as a C compiler lays them out."""
    fields = {
        "nrt_uv_raster_params": ["width", "height", "uv_region", "texel_offset", "flip_x", "flip_y", "flags"],
        "nrt_bake_params": ["width", "height", "spp", "sample0", "seed", "ao_min_t", "ao_max_t", "flags",
                            "d_facevarying_normals"],
        "nrt_bake_result": ["texels", "ao_rays", "ao_hits", "traverse_ms", "total_ms", "launches", "traverse_launches"],
    }
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "nanort_b200_bake.h"', "int main(void) {"]
    for t, fs in fields.items():
        lines.append(f'  printf("{t} %zu", sizeof({t}));')
        for f in fs:
            lines.append(f'  printf(" {f}=%zu", offsetof({t}, {f}));')
        lines.append('  printf("\\n");')
    lines.append("  return 0; }")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines) + "\n")
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    out = {}
    for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines():
        t, size, *rest = line.split()
        out[t] = (int(size), [(kv.split("=")[0], int(kv.split("=")[1])) for kv in rest])
    return out


def test_struct_mirrors_have_the_header_layout(tmp_path):
    from nanort_b200 import api

    cc = shutil.which("gcc")
    if cc is None:
        pytest.skip("no host compiler")
    want = _c_layout(tmp_path, cc)
    for t, cls in (("nrt_uv_raster_params", api.UvRasterParams), ("nrt_bake_params", api.BakeParams),
                   ("nrt_bake_result", api.BakeResult)):
        size, offsets = want[t]
        assert ctypes.sizeof(cls) == size, t
        assert [(f, getattr(cls, f).offset) for f, _ in cls._fields_] == offsets, t


@pytest.mark.parametrize("lang", ["c", "c++"])
def test_header_compiles_on_its_own(lang, tmp_path):
    cc = shutil.which("gcc" if lang == "c" else "g++")
    if cc is None:
        pytest.skip("no host compiler")
    src = tmp_path / ("t.c" if lang == "c" else "t.cc")
    src.write_text('#include "nanort_b200_bake.h"\n'
                   "int main(void) { nrt_bake_params p = {0}; nrt_uv_raster_params q = {0}; nrt_bake_result r = {0};\n"
                   "  return (int)(p.spp + q.width + r.launches); }\n")
    r = subprocess.run([cc, "-fsyntax-only", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


# uv_raster's ray origin (examples/uv_raster/main.cc:752-770) as C: int x, y promoted to float, float32 arithmetic
# in the source's order, no contraction
_TEXEL_C = r"""
#include <stdio.h>
#include <stdlib.h>
int main(int argc, char **argv) {
  const int width = atoi(argv[1]), height = atoi(argv[2]);
  float uv_region[4], texel_offset[2];
  for (int k = 0; k < 4; k++) uv_region[k] = strtof(argv[3 + k], NULL);
  for (int k = 0; k < 2; k++) texel_offset[k] = strtof(argv[7 + k], NULL);
  FILE *f = fopen(argv[9], "wb");
  for (int y = 0; y < height; y++)
    for (int x = 0; x < width; x++) {
      float org[3];
      const float usize = (uv_region[1] - uv_region[0]);
      const float vsize = (uv_region[3] - uv_region[2]);
      org[0] = uv_region[0] + (x * usize + texel_offset[0]) / (float)(width);
      org[1] = uv_region[2] + (y * vsize + texel_offset[1]) / (float)(height);
      org[2] = 1.0f;
      fwrite(org, sizeof(float), 3, f);
    }
  fclose(f);
  return 0;
}
"""


def test_texel_rays_equal_the_reference_expression(tmp_path):
    cc = shutil.which("gcc")
    if cc is None:
        pytest.skip("no host compiler")
    src, exe = tmp_path / "texel.c", tmp_path / "texel"
    src.write_text(_TEXEL_C)
    subprocess.run([cc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-o", str(exe), str(src)], check=True)
    rng = np.random.default_rng(5)
    cases = [(257, 131, [0, 1, 0, 1], [0.5, 0.5]), (64, 64, [0, 1, 0, 1], [0.5, 0.5])]
    for _ in range(6):
        W, H = (int(x) for x in rng.integers(1, 300, 2))
        lo = rng.uniform(-2, 1, 2)
        region = [lo[0], lo[0] + rng.uniform(0.01, 3), lo[1], lo[1] + rng.uniform(-3, 3)]
        cases.append((W, H, region, list(rng.uniform(-1, 2, 2))))
    for W, H, region, off in cases:
        region = [float(np.float32(r)) for r in region]
        off = [float(np.float32(o)) for o in off]
        out = tmp_path / "org.bin"
        subprocess.run([str(exe), str(W), str(H)] + [repr(r) for r in region] + [repr(o) for o in off] + [str(out)],
                       check=True)
        want = np.fromfile(out, np.float32).reshape(-1, 3)
        got = B.texel_rays(W, H, region, off)
        assert np.array_equal(got["org"].view(np.uint32), want.view(np.uint32)), (W, H, region, off)
        assert np.all(got["dir"] == np.float32([0, 0, -1])) and np.all(got["min_t"] == 0)
        assert np.all(got["max_t"] == np.float32(1e30))
