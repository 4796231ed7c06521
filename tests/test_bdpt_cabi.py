"""CPU: the bidirectional path tracer has its own header (include/nanort_b200_bdpt.h); the library exports what it
declares, the ctypes mirror lists exactly that with the header's struct layouts, the header stands alone as C and as
C++, and the numpy restatement of the sample set-up (tests/bdpt_model.py: the generator, the seed and the camera ray)
equals the reference's own (oracle/_ref/libbdpt_ref.so, examples/bidir_path_tracer/main.cc) (no compute on a GPU)."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import bdpt_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "nanort_b200_bdpt.h")


def test_library_exports_every_bdpt_symbol():
    from nanort_b200 import api

    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    names = sorted(set(re.findall(r"\b(nrt_[a-z0-9_]+)\s*\(", src)))
    assert sorted(api.BDPT_EXPORTS) == names
    for other in (api.EXPORTS, api.SCENE_PATH_EXPORTS, api.BAKE_EXPORTS):
        assert not set(names) & set(other), "declared in one header only"
    L = ctypes.CDLL(api.LIB_PATH)
    for n in names:
        assert hasattr(L, n), n


def _c_layout(tmp_path, cc, fields):
    """sizeof and field offsets of the header's structs, as a C compiler lays them out."""
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "nanort_b200_bdpt.h"', "int main(void) {"]
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
    structs = {"nrt_bdpt_params": api.BdptParams, "nrt_bdpt_result": api.BdptResult}
    fields = {t: [f for f, _ in cls._fields_] for t, cls in structs.items()}
    fields["nrt_bdpt_vertex"] = list(api.BDPT_VERTEX_DTYPE.names)
    want = _c_layout(tmp_path, cc, fields)
    for t, cls in structs.items():
        size, offsets = want[t]
        assert ctypes.sizeof(cls) == size, t
        assert [(f, getattr(cls, f).offset) for f, _ in cls._fields_] == offsets, t
    size, offsets = want["nrt_bdpt_vertex"]
    assert api.BDPT_VERTEX_DTYPE.itemsize == size == 80
    assert [(f, api.BDPT_VERTEX_DTYPE.fields[f][1]) for f in api.BDPT_VERTEX_DTYPE.names] == offsets


@pytest.mark.parametrize("lang", ["c", "c++"])
def test_header_compiles_on_its_own(lang, tmp_path):
    cc = shutil.which("gcc" if lang == "c" else "g++")
    if cc is None:
        pytest.skip("no host compiler")
    src = tmp_path / ("t.c" if lang == "c" else "t.cc")
    src.write_text('#include "nanort_b200_bdpt.h"\n'
                   "int main(void) { nrt_bdpt_params p = {0}; nrt_bdpt_result r = {0}; nrt_bdpt_vertex v = {0};\n"
                   "  return (int)(p.spp + r.launches + v.type); }\n")
    r = subprocess.run([cc, "-fsyntax-only", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


@pytest.fixture(scope="module")
def ref():
    from oracle import bdpt_ref

    if not bdpt_ref.available():
        pytest.skip("oracle/_ref/libbdpt_ref.so not built (no reference tree at build time)")
    return bdpt_ref


def test_random_stream_equals_the_reference(ref):
    seeds = [0, 1, 7, 0xFFFFFFFF, M.seed(511, 0, 512, 100, 99), M.seed(3, 5, 64, 4, 2)]
    big = ((4000 * 8192 + 5000) * 200 + 7)
    assert big >= 1 << 32
    seeds.append(M.seed(5000, 4000, 8192, 200, 7))  # (y*W + x)*spp_total + i wraps 32 bits
    assert seeds[-1] == big & 0xFFFFFFFF
    for s in seeds:
        got, want = M.random_reals(s, 200), ref.random(s, 200)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), s


def test_camera_ray_equals_the_reference_lens_vertex(ref):
    from nanort_b200 import api

    # one emissive triangle behind the camera (which looks down -z from z = 20): every eye subpath is the lens alone
    v = np.float32([[-1, 0, 40], [1, 0, 40], [0, 2, 40]])
    f = np.uint32([[0, 1, 2]])
    mats = np.zeros((1, 16), np.float32)
    mats[0, 9:12] = 5.0
    scene = ref.BdptReference(v, f, np.zeros(1, np.uint32), mats, M.flat_normals(v, f), api.BDPT_VERTEX_DTYPE)
    W, H, spp = 37, 23, 3
    rng = np.random.default_rng(3)
    for _ in range(60):
        x, y, i = int(rng.integers(0, W)), int(rng.integers(0, H)), int(rng.integers(0, spp))
        s = M.seed(x, y, W, spp, i)
        eye, light, rgb = scene.sample(x, y, W, H, s)
        assert len(eye) == 1 and len(light) == 0 and not rgb.any()
        org, d = M.camera_ray(M.REFERENCE_CAMERA, x, y, W, H, s)
        assert eye[0]["type"] == api.BDPT_LENS
        assert np.array_equal(eye[0]["position"].view(np.uint32), org.view(np.uint32))
        assert np.array_equal(eye[0]["norm"].view(np.uint32), d.view(np.uint32)), (x, y, i)
        assert eye[0]["pdf_fwd"] == 1.0 and np.all(eye[0]["beta"] == 1.0)
