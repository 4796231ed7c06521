"""ctypes binding of oracle/_ref/libbdpt_ref.so: the unmodified examples/bidir_path_tracer/main.cc behind
oracle/bdpt_ref_shim.cc (built by oracle/bdpt.mk).  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "_ref", "libbdpt_ref.so")
MAX_BOUNCES = 10  # the reference's uMaxBounces: its subpaths have at most 11 vertices

_L = None


def available():
    return os.path.exists(PATH)


def lib():
    global _L
    if _L is None:
        L = C.CDLL(PATH)
        vp, sz, u32, i32 = C.c_void_p, C.c_size_t, C.c_uint32, C.c_int
        L.bdpt_ref_scene.restype = vp
        L.bdpt_ref_scene.argtypes = [vp, sz, vp, sz, vp, vp, vp, sz]
        L.bdpt_ref_scene_free.argtypes = [vp]
        L.bdpt_ref_sample.argtypes = [vp, i32, i32, i32, i32, u32, vp, vp, vp, vp, vp]
        L.bdpt_ref_connect.argtypes = [vp, vp, u32, vp, u32, vp]
        L.bdpt_ref_random.argtypes = [u32, sz, vp]
        _L = L
    return _L


def random(seed, n):
    """n draws of the reference's Random(seed).nextReal()"""
    out = np.zeros(n, np.float32)
    lib().bdpt_ref_random(int(seed) & 0xFFFFFFFF, n, out.ctypes.data)
    return out


class BdptReference:
    """The reference's mesh, materials (16 floats each), BVH (cache_bbox = false) and LightSampler over borrowed
    arrays.  `vertex_dtype` is nanort_b200.api.BDPT_VERTEX_DTYPE (nrt_bdpt_vertex)."""

    def __init__(self, verts, faces, material_ids, materials16, facevarying_normals, vertex_dtype):
        self.verts = np.ascontiguousarray(verts, np.float32)
        self.faces = np.ascontiguousarray(faces, np.uint32)
        self.ids = np.ascontiguousarray(material_ids, np.uint32)
        self.mats = np.ascontiguousarray(np.asarray(materials16).view(np.float32).reshape(-1, 16))
        self.fvn = np.ascontiguousarray(facevarying_normals, np.float32).reshape(-1, 9)
        self.dtype = vertex_dtype
        self.h = lib().bdpt_ref_scene(self.verts.ctypes.data, len(self.verts), self.faces.ctypes.data, len(self.faces),
                                      self.ids.ctypes.data, self.fvn.ctypes.data, self.mats.ctypes.data, len(self.mats))
        assert self.h, "the reference needs an emissive face"

    def __del__(self):
        try:
            lib().bdpt_ref_scene_free(self.h)
        except Exception:
            pass

    def sample(self, x, y, width, height, seed):
        """main()'s sample loop body for loop pixel (x, y): (eye vertices, light vertices, rgb)"""
        eye = np.zeros(MAX_BOUNCES + 1, self.dtype)
        light = np.zeros(MAX_BOUNCES + 1, self.dtype)
        ne, nl = C.c_uint32(0), C.c_uint32(0)
        rgb = np.zeros(3, np.float32)
        lib().bdpt_ref_sample(self.h, int(x), int(y), int(width), int(height), int(seed) & 0xFFFFFFFF, eye.ctypes.data,
                              C.byref(ne), light.ctypes.data, C.byref(nl), rgb.ctypes.data)
        return eye[:ne.value].copy(), light[:nl.value].copy(), rgb

    def connect(self, eye, light):
        """connectPath over the given subpaths (records of vertex_dtype)"""
        eye = np.ascontiguousarray(eye, self.dtype)
        light = np.ascontiguousarray(light, self.dtype)
        rgb = np.zeros(3, np.float32)
        lib().bdpt_ref_connect(self.h, eye.ctypes.data, len(eye), light.ctypes.data, len(light), rgb.ctypes.data)
        return rgb
