"""TEST INFRASTRUCTURE ONLY: ctypes bindings for the parity oracle.

 * `Port`      -> oracle/liborc.so           (C restatement, oracle/nanort_oracle.c)
 * `Reference` -> oracle/_ref/libnanort_ref{,03}.so (the unmodified reference header behind
                  oracle/ref_shim.cc; present when it was built in the authoring container)

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import
this module.  Nothing under nanort_b200/ does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

RAY_DTYPE = np.dtype(
    [("org", "<f4", (3,)), ("dir", "<f4", (3,)), ("min_t", "<f4"), ("max_t", "<f4"), ("type", "<u4")]
)
HIT_DTYPE = np.dtype([("u", "<f4"), ("v", "<f4"), ("t", "<f4"), ("prim_id", "<u4")])
NODE_DTYPE = np.dtype(
    [("bmin", "<f4", (3,)), ("bmax", "<f4", (3,)), ("flag", "<i4"), ("axis", "<i4"), ("data", "<u4", (2,))]
)
BUILD_OPT_DTYPE = np.dtype(
    [
        ("cost_t_aabb", "<f4"),
        ("min_leaf_primitives", "<u4"),
        ("max_tree_depth", "<u4"),
        ("bin_size", "<u4"),
        ("shallow_depth", "<u4"),
        ("min_primitives_for_parallel_build", "<u4"),
        ("cache_bbox", "u1"),
        ("pad", "u1", (3,)),
    ]
)
TRACE_OPT_DTYPE = np.dtype(
    [("prim_ids_range", "<u4", (2,)), ("skip_prim_id", "<u4"), ("cull_back_face", "u1"), ("pad", "u1", (3,))]
)
assert BUILD_OPT_DTYPE.itemsize == 28 and TRACE_OPT_DTYPE.itemsize == 16

MODE_CPP11 = 1
MODE_FIXBINS = 2  # NOT reference behaviour (all three axes binned); experiments only


def build_options(**kw):
    o = np.zeros(1, BUILD_OPT_DTYPE)
    o["cost_t_aabb"] = 0.2
    o["min_leaf_primitives"] = 4
    o["max_tree_depth"] = 256
    o["bin_size"] = 64
    o["shallow_depth"] = 4
    o["min_primitives_for_parallel_build"] = 8192
    for k, v in kw.items():
        o[k] = v
    return o


def trace_options(**kw):
    o = np.zeros(1, TRACE_OPT_DTYPE)
    o["prim_ids_range"] = (0, 0x7FFFFFFF)
    o["skip_prim_id"] = 0xFFFFFFFF
    for k, v in kw.items():
        o[k] = v
    return o


def make(force=False):
    """Compiles liborc.so (and oracle/_ref where the reference tree is present, see oracle/Makefile)."""
    if force or not os.path.exists(os.path.join(HERE, "liborc.so")):
        subprocess.run(["make", "-C", HERE], check=True, capture_output=True)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Counters(C.Structure):
    _fields_ = [("nodes_popped", C.c_uint64), ("prims_tested", C.c_uint64), ("max_stack", C.c_uint32)]


class Port:
    """The C restatement.  Stateless: trees are plain numpy arrays."""

    def __init__(self):
        path = os.path.join(HERE, "liborc.so")
        if not os.path.exists(path):
            make()
        self.lib = C.CDLL(path)
        L = self.lib
        L.orc_build.restype = C.c_size_t
        L.orc_build.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p]
        L.orc_free.argtypes = [C.c_void_p]
        L.orc_traverse_batch.restype = C.c_size_t
        L.orc_traverse_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                         C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                         C.c_void_p]
        L.orc_test_prim.restype = C.c_int
        L.orc_test_prim.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                    C.c_uint32, C.c_void_p]

    def build(self, verts, faces, opts=None, mode=MODE_CPP11):
        verts = np.ascontiguousarray(verts, np.float32)
        faces = np.ascontiguousarray(faces, np.uint32)
        n = len(faces)
        indices = np.zeros(n, np.uint32)
        stats = np.zeros(3, np.uint32)
        out = C.c_void_p()
        nn = self.lib.orc_build(_p(verts), 12, _p(faces), n, _p(opts) if opts is not None else None, mode,
                                C.byref(out), _p(indices), _p(stats))
        if nn == 0:
            return None
        nodes = np.frombuffer((C.c_char * (nn * 40)).from_address(out.value), NODE_DTYPE).copy()
        self.lib.orc_free(out)
        return nodes, indices, {"max_tree_depth": int(stats[0]), "num_leaf_nodes": int(stats[1]),
                                "num_branch_nodes": int(stats[2])}

    def traverse(self, nodes, indices, verts, faces, rays, topts=None, cpp11=True, threads=1, counters=False):
        nodes = np.ascontiguousarray(nodes)
        indices = np.ascontiguousarray(indices, np.uint32)
        verts = np.ascontiguousarray(verts, np.float32)
        faces = np.ascontiguousarray(faces, np.uint32)
        rays = np.ascontiguousarray(rays)
        assert rays.dtype.itemsize == 36 and nodes.dtype.itemsize == 40
        n = len(rays)
        hits = np.zeros(n, HIT_DTYPE)
        mask = np.zeros(n, np.uint8)
        ctr = Counters()
        self.lib.orc_traverse_batch(_p(nodes), _p(indices), _p(verts), 12, _p(faces), _p(rays), n, _p(hits),
                                    _p(mask), _p(topts) if topts is not None else None, 1 if cpp11 else 0,
                                    threads, C.addressof(ctr) if counters else None)
        if counters:
            return hits, mask, {"nodes_popped": ctr.nodes_popped, "prims_tested": ctr.prims_tested,
                                "max_stack": ctr.max_stack}
        return hits, mask

    def test_prim(self, verts, faces, ray, prim, topts=None, cpp11=True):
        verts = np.ascontiguousarray(verts, np.float32)
        faces = np.ascontiguousarray(faces, np.uint32)
        ray = np.ascontiguousarray(ray).reshape(1)
        out = np.zeros(1, HIT_DTYPE)
        ok = self.lib.orc_test_prim(_p(verts), 12, _p(faces), _p(ray), _p(topts) if topts is not None else None,
                                    1 if cpp11 else 0, int(prim), _p(out))
        return bool(ok), out[0]


class Reference:
    """The unmodified reference header (oracle/_ref).  Raises FileNotFoundError when absent."""

    def __init__(self, cpp11=True):
        name = "libnanort_ref.so" if cpp11 else "libnanort_ref03.so"
        path = os.path.join(HERE, "_ref", name)
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.cpp11 = cpp11
        self.lib = C.CDLL(path)
        L = self.lib
        L.ref_build.restype = C.c_void_p
        L.ref_build.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32, C.c_void_p]
        L.ref_adopt.restype = C.c_void_p
        L.ref_adopt.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
        L.ref_free.argtypes = [C.c_void_p]
        L.ref_stats.argtypes = [C.c_void_p, C.c_void_p]
        L.ref_bounding_box.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.ref_num_nodes.restype = C.c_size_t
        L.ref_num_nodes.argtypes = [C.c_void_p]
        L.ref_num_indices.restype = C.c_size_t
        L.ref_num_indices.argtypes = [C.c_void_p]
        L.ref_copy_nodes.argtypes = [C.c_void_p, C.c_void_p]
        L.ref_copy_indices.argtypes = [C.c_void_p, C.c_void_p]
        L.ref_traverse_batch.restype = C.c_size_t
        L.ref_traverse_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_int]
        L.ref_traverse_one_f64.restype = C.c_int
        L.ref_traverse_one_f64.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_double,
                                           C.c_double, C.c_void_p, C.c_void_p]
        L.ref_sizes.argtypes = [C.c_void_p]

    @staticmethod
    def available(cpp11=True):
        name = "libnanort_ref.so" if cpp11 else "libnanort_ref03.so"
        return os.path.exists(os.path.join(HERE, "_ref", name))

    def sizes(self):
        s = np.zeros(5, np.uint32)
        self.lib.ref_sizes(_p(s))
        return [int(x) for x in s]

    class Accel:
        def __init__(self, ref, handle, verts, faces):
            self.ref, self.h, self.verts, self.faces = ref, handle, verts, faces  # keep geometry alive

        def __del__(self):
            if self.h:
                self.ref.lib.ref_free(self.h)
                self.h = None

        def stats(self):
            s = np.zeros(3, np.uint32)
            self.ref.lib.ref_stats(self.h, _p(s))
            return {"max_tree_depth": int(s[0]), "num_leaf_nodes": int(s[1]), "num_branch_nodes": int(s[2])}

        def bounding_box(self):
            a, b = np.zeros(3, np.float32), np.zeros(3, np.float32)
            self.ref.lib.ref_bounding_box(self.h, _p(a), _p(b))
            return a, b

        def nodes(self):
            n = self.ref.lib.ref_num_nodes(self.h)
            out = np.zeros(n, NODE_DTYPE)
            self.ref.lib.ref_copy_nodes(self.h, _p(out))
            return out

        def indices(self):
            n = self.ref.lib.ref_num_indices(self.h)
            out = np.zeros(n, np.uint32)
            self.ref.lib.ref_copy_indices(self.h, _p(out))
            return out

        def traverse(self, rays, topts=None, threads=1, hits=None, mask=None):
            rays = np.ascontiguousarray(rays)
            assert rays.dtype.itemsize == 36
            n = len(rays)
            if hits is None:
                hits = np.zeros(n, HIT_DTYPE)
            if mask is None:
                mask = np.zeros(n, np.uint8)
            self.ref.lib.ref_traverse_batch(self.h, _p(rays), n, _p(hits), _p(mask),
                                            _p(topts) if topts is not None else None, threads)
            return hits, mask

    def build(self, verts, faces, opts=None):
        verts = np.ascontiguousarray(verts, np.float32)
        faces = np.ascontiguousarray(faces, np.uint32)
        h = self.lib.ref_build(_p(verts), 12, _p(faces), len(faces), _p(opts) if opts is not None else None)
        if not h:
            return None
        return Reference.Accel(self, h, verts, faces)

    def adopt(self, nodes, indices, verts, faces):
        nodes = np.ascontiguousarray(nodes)
        indices = np.ascontiguousarray(indices, np.uint32)
        verts = np.ascontiguousarray(verts, np.float32)
        faces = np.ascontiguousarray(faces, np.uint32)
        h = self.lib.ref_adopt(_p(nodes), len(nodes), _p(indices), len(indices), _p(verts), 12, _p(faces))
        if not h:
            return None
        return Reference.Accel(self, h, verts, faces)

    def traverse_one_f64(self, verts, faces, org, dir, min_t=0.0, max_t=1e30):
        verts = np.ascontiguousarray(verts, np.float64)
        faces = np.ascontiguousarray(faces, np.uint32)
        org = np.ascontiguousarray(org, np.float64)
        dir = np.ascontiguousarray(dir, np.float64)
        out = np.zeros(3, np.float64)
        prim = np.zeros(1, np.uint32)
        r = self.lib.ref_traverse_one_f64(_p(verts), _p(faces), len(faces), _p(org), _p(dir), min_t, max_t,
                                          _p(out), _p(prim))
        return r, out, int(prim[0])


# ------------------------------------------------------------------ two-level scene (examples/nanosg)
SG_HIT_DTYPE = np.dtype([("u", "<f4"), ("v", "<f4"), ("t", "<f4"), ("prim_id", "<u4"), ("node_id", "<u4"),
                         ("P", "<f4", (3,))])
SG_NODE_DTYPE = np.dtype([("xform", "<f4", (4, 4)), ("inv", "<f4", (4, 4)), ("inv33", "<f4", (4, 4)),
                          ("invT33", "<f4", (4, 4)), ("lbmin", "<f4", (3,)), ("lbmax", "<f4", (3,)),
                          ("xbmin", "<f4", (3,)), ("xbmax", "<f4", (3,))])
assert SG_HIT_DTYPE.itemsize == 32 and SG_NODE_DTYPE.itemsize == 76 * 4


class _SgBlas(C.Structure):
    _fields_ = [("nodes", C.c_void_p), ("indices", C.c_void_p), ("verts", C.c_void_p), ("stride", C.c_size_t),
                ("faces", C.c_void_p)]


class PortScene:
    """Port of nanosg::Scene: instances = [(verts, faces, xform4x4)], Commit() at construction.
    Every instance builds its own bottom-level tree, like Node::Update does."""

    def __init__(self, instances, cpp11=True, port=None):
        self.port = port or Port()
        L = self.port.lib
        L.orc_build_boxes.restype = C.c_size_t
        L.orc_build_boxes.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p),
                                      C.c_void_p, C.c_void_p]
        L.orc_sg_node_update.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_sg_list.restype = C.c_int
        L.orc_sg_list.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                  C.c_void_p, C.c_void_p]
        L.orc_sg_traverse_batch.restype = C.c_size_t
        L.orc_sg_traverse_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                            C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.orc_sg_local_hit_batch.restype = None
        L.orc_sg_local_hit_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                             C.c_int, C.c_void_p, C.c_void_p]
        self.cpp11 = cpp11
        mode = MODE_CPP11 if cpp11 else 0
        n = len(instances)
        self.sg = np.zeros(n, SG_NODE_DTYPE)
        self.blas = []  # (nodes, indices, verts, faces) kept alive
        self._blas_c = (_SgBlas * n)()
        cache = {}
        for i, (v, f, x) in enumerate(instances):
            v = np.ascontiguousarray(v, np.float32)
            f = np.ascontiguousarray(f, np.uint32)
            key = (v.ctypes.data, f.ctypes.data, len(f))
            if key not in cache:  # identical arrays give identical trees: build once
                nodes, idx, _ = self.port.build(v, f, None, mode)
                cache[key] = (nodes, idx, v, f)
            nodes, idx, v, f = cache[key]
            self.blas.append(cache[key])
            self._blas_c[i] = _SgBlas(nodes.ctypes.data, idx.ctypes.data, v.ctypes.data, 12, f.ctypes.data)
            x = np.ascontiguousarray(x, np.float32).reshape(16)
            lb0 = np.ascontiguousarray(nodes["bmin"][0])
            lb1 = np.ascontiguousarray(nodes["bmax"][0])
            L.orc_sg_node_update(self.sg[i:i + 1].ctypes.data, _p(x), _p(lb0), _p(lb1))
        boxes = np.ascontiguousarray(np.concatenate([self.sg["xbmin"], self.sg["xbmax"]], axis=1), np.float32)
        self.top_idx = np.zeros(n, np.uint32)
        out = C.c_void_p()
        o = build_options(min_leaf_primitives=1)
        nn = L.orc_build_boxes(_p(boxes), n, _p(o), mode, C.byref(out), _p(self.top_idx), None)
        assert nn > 0
        self.top = np.frombuffer((C.c_char * (nn * 40)).from_address(out.value), NODE_DTYPE).copy()
        L.orc_free(out)

    def _top(self, top, top_idx):
        """this scene's own top-level tree, or any other one built over the same instance boxes (e.g. the tree a
        device Commit produced, Scene.GetTopLevel())"""
        if top is None:
            return self.top, self.top_idx
        top, top_idx = np.ascontiguousarray(top), np.ascontiguousarray(top_idx, np.uint32)
        assert top.dtype.itemsize == 40 and len(top_idx) == len(self.sg)
        return top, top_idx

    def list_node_intersections(self, ray, max_hits=64, top=None, top_idx=None):
        top, top_idx = self._top(top, top_idx)
        ray = np.ascontiguousarray(ray).reshape(1)
        tmin, tmax, ids = np.zeros(128, np.float32), np.zeros(128, np.float32), np.zeros(128, np.uint32)
        n = self.port.lib.orc_sg_list(_p(top), _p(top_idx), _p(self.sg), _p(ray), max_hits,
                                      1 if self.cpp11 else 0, _p(tmin), _p(tmax), _p(ids))
        return tmin[:n], tmax[:n], ids[:n]

    def traverse(self, rays, threads=1, top=None, top_idx=None, max_hits=64):
        """Scene::Traverse over `top` (default: this scene's own top-level tree); max_hits (<= 128) replaces the
        reference's 64-box limit."""
        assert 1 <= max_hits <= 128
        top, top_idx = self._top(top, top_idx)
        rays = np.ascontiguousarray(rays)
        n = len(rays)
        hits, mask = np.zeros(n, SG_HIT_DTYPE), np.zeros(n, np.uint8)
        self.port.lib.orc_sg_traverse_batch(_p(top), _p(top_idx), _p(self.sg),
                                            C.addressof(self._blas_c), _p(rays), n, _p(hits), _p(mask),
                                            max_hits, 1 if self.cpp11 else 0, threads)
        return hits, mask

    def _local_hits(self, rays, node_ids, prim_ids):
        rays = np.ascontiguousarray(rays).reshape(-1)
        n = len(rays)
        ids = np.ascontiguousarray(np.broadcast_to(np.asarray(node_ids, np.uint32), (n,)))
        assert n == 0 or int(ids.max()) < len(self.sg)
        prims = None if prim_ids is None else np.ascontiguousarray(np.broadcast_to(np.asarray(prim_ids, np.uint32), (n,)))
        hits, ok = np.zeros(n, SG_HIT_DTYPE), np.zeros(n, np.uint8)
        self.port.lib.orc_sg_local_hit_batch(_p(self.sg), C.addressof(self._blas_c), _p(rays), n, _p(ids),
                                             _p(prims) if prims is not None else None, 1 if self.cpp11 else 0,
                                             _p(hits), _p(ok))
        return hits, ok.astype(bool)

    def instance_hit(self, rays, node_ids):
        """(records, ok): the nearest hit of rays[i] inside instance node_ids[i] alone, as Scene::Traverse records
        it (its per-instance body, nanosg.h:831-850)"""
        return self._local_hits(rays, node_ids, None)

    def prim_hit(self, rays, node_ids, prim_ids):
        """(records, ok): the record Scene::Traverse writes when triangle prim_ids[i] of instance node_ids[i] is the
        pick of rays[i] -- the same arithmetic on that one triangle"""
        return self._local_hits(rays, node_ids, prim_ids)


def list_node_intersections_on_tree(port, nodes, indices, sg_nodes, ray, max_hits=64, cpp11=True):
    """BVHAccel::ListNodeIntersections (restatement pinned to nanosg.h by tests/test_oracle_scene.py) over ANY node
    array built on the world boxes sg_nodes["xbmin"/"xbmax"] -- e.g. the one a device build produced.  The list is a
    property of the tree's leaves (NodeBBoxIntersector has no [min_t, max_t] clamp, nanosg.h:597-634: a box behind the
    origin or beyond max_t is listed iff it shares a leaf with a box the range-clamped node test lets through), so a
    device list is compared on the device's own tree."""
    L = port.lib
    L.orc_sg_list.restype = C.c_int
    L.orc_sg_list.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                              C.c_void_p, C.c_void_p]
    nodes = np.ascontiguousarray(nodes)
    indices = np.ascontiguousarray(indices, np.uint32)
    sg_nodes = np.ascontiguousarray(sg_nodes)
    ray = np.ascontiguousarray(ray).reshape(1)
    tmin, tmax, ids = np.zeros(128, np.float32), np.zeros(128, np.float32), np.zeros(128, np.uint32)
    n = L.orc_sg_list(_p(nodes), _p(indices), _p(sg_nodes), _p(ray), max_hits, 1 if cpp11 else 0, _p(tmin), _p(tmax),
                      _p(ids))
    return tmin[:n], tmax[:n], ids[:n]


class ReferenceScene:
    """The unmodified nanosg::Scene (oracle/_ref/libnanosg_ref*.so)."""

    @staticmethod
    def available(cpp11=True):
        return os.path.exists(os.path.join(HERE, "_ref", "libnanosg_ref.so" if cpp11 else "libnanosg_ref03.so"))

    def __init__(self, instances, cpp11=True):
        path = os.path.join(HERE, "_ref", "libnanosg_ref.so" if cpp11 else "libnanosg_ref03.so")
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.lib = L = C.CDLL(path)
        L.refsg_create.restype = C.c_void_p
        L.refsg_free.argtypes = [C.c_void_p]
        L.refsg_add_node.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
        L.refsg_commit.argtypes = [C.c_void_p]
        L.refsg_bounding_box.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.refsg_node_state.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
        L.refsg_top_num_nodes.restype = C.c_size_t
        L.refsg_top_num_nodes.argtypes = [C.c_void_p]
        L.refsg_top_copy.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.refsg_node_num_nodes.restype = C.c_size_t
        L.refsg_node_num_nodes.argtypes = [C.c_void_p, C.c_size_t]
        L.refsg_node_copy.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        L.refsg_list_node_intersections.restype = C.c_int
        L.refsg_list_node_intersections.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                                    C.c_void_p]
        L.refsg_traverse_batch.restype = C.c_size_t
        L.refsg_traverse_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_int]
        self.h = L.refsg_create()
        self.n = len(instances)
        self.n_prims = []
        for v, f, x in instances:
            v = np.ascontiguousarray(v, np.float32)
            f = np.ascontiguousarray(f, np.uint32)
            x = np.ascontiguousarray(x, np.float32).reshape(16)
            assert L.refsg_add_node(self.h, _p(v), len(v), _p(f), len(f), _p(x)) == 0
            self.n_prims.append(len(f))
        assert L.refsg_commit(self.h) == 0

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.refsg_free(self.h)
            self.h = None

    def bounding_box(self):
        a, b = np.zeros(3, np.float32), np.zeros(3, np.float32)
        self.lib.refsg_bounding_box(self.h, _p(a), _p(b))
        return a, b

    def node_states(self):
        out = np.zeros(self.n, SG_NODE_DTYPE)
        for i in range(self.n):
            self.lib.refsg_node_state(self.h, i, out[i:i + 1].ctypes.data)
        return out

    def top(self):
        nn = self.lib.refsg_top_num_nodes(self.h)
        nodes, idx = np.zeros(nn, NODE_DTYPE), np.zeros(self.n, np.uint32)
        self.lib.refsg_top_copy(self.h, _p(nodes), _p(idx))
        return nodes, idx

    def node_tree(self, i):
        nn = self.lib.refsg_node_num_nodes(self.h, i)
        nodes, idx = np.zeros(nn, NODE_DTYPE), np.zeros(self.n_prims[i], np.uint32)
        self.lib.refsg_node_copy(self.h, i, _p(nodes), _p(idx))
        return nodes, idx

    def list_node_intersections(self, ray, max_hits=64):
        ray = np.ascontiguousarray(ray).reshape(1)
        tmin, tmax, ids = np.zeros(128, np.float32), np.zeros(128, np.float32), np.zeros(128, np.uint32)
        n = self.lib.refsg_list_node_intersections(self.h, _p(ray), max_hits, _p(tmin), _p(tmax), _p(ids))
        return tmin[:n], tmax[:n], ids[:n]

    def traverse(self, rays, threads=1):
        rays = np.ascontiguousarray(rays)
        n = len(rays)
        hits, mask = np.zeros(n, SG_HIT_DTYPE), np.zeros(n, np.uint8)
        self.lib.refsg_traverse_batch(self.h, _p(rays), n, _p(hits), _p(mask), threads)
        return hits, mask


# ------------------------------------------------------------------ BVHAccel<double>: the reference itself is the checker
RAY64_DTYPE = np.dtype([("org", "<f8", (3,)), ("dir", "<f8", (3,)), ("min_t", "<f8"), ("max_t", "<f8"),
                        ("type", "<u4"), ("pad", "<u4")])
HIT64_DTYPE = np.dtype([("u", "<f8"), ("v", "<f8"), ("t", "<f8"), ("prim_id", "<u4"), ("pad", "<u4")])
NODE64_DTYPE = np.dtype([("bmin", "<f8", (3,)), ("bmax", "<f8", (3,)), ("flag", "<i4"), ("axis", "<i4"),
                         ("data", "<u4", (2,))])


BUILD_OPT64_DTYPE = np.dtype([("cost_t_aabb", "<f8"), ("min_leaf_primitives", "<u4"), ("max_tree_depth", "<u4"),
                              ("bin_size", "<u4"), ("shallow_depth", "<u4"),
                              ("min_primitives_for_parallel_build", "<u4"), ("cache_bbox", "u1"), ("pad", "u1", (3,))])
assert BUILD_OPT64_DTYPE.itemsize == 32


def build_options_f64(**kw):
    o = np.zeros(1, BUILD_OPT64_DTYPE)
    o["cost_t_aabb"], o["min_leaf_primitives"], o["max_tree_depth"], o["bin_size"] = 0.2, 4, 256, 64
    o["shallow_depth"], o["min_primitives_for_parallel_build"] = 4, 8192
    for k, v in kw.items():
        o[k] = v
    return o


class Port64:
    """The C restatement instantiated for double (oracle/liborc64.so = nanort_oracle.c with -DORC_DOUBLE)."""

    def __init__(self):
        path = os.path.join(HERE, "liborc64.so")
        if not os.path.exists(path):
            make(force=True)
        self.lib = L = C.CDLL(path)
        L.orc_build.restype = C.c_size_t
        L.orc_build.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p]
        L.orc_free.argtypes = [C.c_void_p]
        L.orc_traverse_batch.restype = C.c_size_t
        L.orc_traverse_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                         C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                         C.c_void_p]
        L.orc_sizes.argtypes = [C.c_void_p]

    def sizes(self):
        s = np.zeros(5, np.uint32)
        self.lib.orc_sizes(_p(s))
        return [int(x) for x in s]

    def build(self, verts, faces, opts=None, mode=MODE_CPP11):
        verts = np.ascontiguousarray(verts, np.float64)
        faces = np.ascontiguousarray(faces, np.uint32)
        n = len(faces)
        indices, stats, out = np.zeros(n, np.uint32), np.zeros(3, np.uint32), C.c_void_p()
        nn = self.lib.orc_build(_p(verts), 24, _p(faces), n, _p(opts) if opts is not None else None, mode,
                                C.byref(out), _p(indices), _p(stats))
        if nn == 0:
            return None
        nodes = np.frombuffer((C.c_char * (nn * 64)).from_address(out.value), NODE64_DTYPE).copy()
        self.lib.orc_free(out)
        return nodes, indices, {"max_tree_depth": int(stats[0]), "num_leaf_nodes": int(stats[1]),
                                "num_branch_nodes": int(stats[2])}

    def traverse(self, nodes, indices, verts, faces, rays, topts=None, cpp11=True, threads=1):
        nodes = np.ascontiguousarray(nodes)
        rays = np.ascontiguousarray(rays)
        assert rays.dtype.itemsize == 72 and nodes.dtype.itemsize == 64
        verts = np.ascontiguousarray(verts, np.float64)
        faces = np.ascontiguousarray(faces, np.uint32)
        indices = np.ascontiguousarray(indices, np.uint32)
        n = len(rays)
        hits, mask = np.zeros(n, HIT64_DTYPE), np.zeros(n, np.uint8)
        self.lib.orc_traverse_batch(_p(nodes), _p(indices), _p(verts), 24, _p(faces), _p(rays), n, _p(hits), _p(mask),
                                    _p(topts) if topts is not None else None, 1 if cpp11 else 0, threads, None)
        return hits, mask


class ReferenceF64:
    """nanort::BVHAccel<double> of the unmodified reference (oracle/_ref, ref64_* in oracle/ref_shim.cc); Port64 is
    pinned to it (tests/test_oracle_f64.py)."""

    def __init__(self, cpp11=True):
        name = "libnanort_ref.so" if cpp11 else "libnanort_ref03.so"
        path = os.path.join(HERE, "_ref", name)
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.lib = L = C.CDLL(path)
        L.ref64_sizes.argtypes = [C.c_void_p]
        L.ref64_build.restype = C.c_void_p
        L.ref64_build.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32, C.c_void_p]
        L.ref64_adopt.restype = C.c_void_p
        L.ref64_adopt.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
        L.ref64_free.argtypes = [C.c_void_p]
        L.ref64_num_nodes.restype = C.c_size_t
        L.ref64_num_nodes.argtypes = [C.c_void_p]
        L.ref64_copy_nodes.argtypes = [C.c_void_p, C.c_void_p]
        L.ref64_copy_indices.argtypes = [C.c_void_p, C.c_void_p]
        L.ref64_bounding_box.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.ref64_traverse_batch.restype = C.c_size_t
        L.ref64_traverse_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_int]

    def sizes(self):
        s = np.zeros(5, np.uint32)
        self.lib.ref64_sizes(_p(s))
        return [int(x) for x in s]

    class Accel:
        def __init__(self, ref, handle, verts, faces):
            self.ref, self.h, self.verts, self.faces = ref, handle, verts, faces

        def __del__(self):
            if self.h:
                self.ref.lib.ref64_free(self.h)
                self.h = None

        def nodes(self):
            n = self.ref.lib.ref64_num_nodes(self.h)
            out = np.zeros(n, NODE64_DTYPE)
            self.ref.lib.ref64_copy_nodes(self.h, _p(out))
            return out

        def indices(self):
            out = np.zeros(len(self.faces), np.uint32)
            self.ref.lib.ref64_copy_indices(self.h, _p(out))
            return out

        def bounding_box(self):
            a, b = np.zeros(3), np.zeros(3)
            self.ref.lib.ref64_bounding_box(self.h, _p(a), _p(b))
            return a, b

        def traverse(self, rays, topts=None, threads=1):
            rays = np.ascontiguousarray(rays)
            assert rays.dtype.itemsize == 72
            n = len(rays)
            hits, mask = np.zeros(n, HIT64_DTYPE), np.zeros(n, np.uint8)
            self.ref.lib.ref64_traverse_batch(self.h, _p(rays), n, _p(hits), _p(mask),
                                              _p(topts) if topts is not None else None, threads)
            return hits, mask

    def build(self, verts, faces, opts=None):
        verts = np.ascontiguousarray(verts, np.float64)
        faces = np.ascontiguousarray(faces, np.uint32)
        h = self.lib.ref64_build(_p(verts), 24, _p(faces), len(faces), _p(opts) if opts is not None else None)
        return self.Accel(self, h, verts, faces) if h else None

    def adopt(self, nodes, indices, verts, faces):
        nodes = np.ascontiguousarray(nodes)
        assert nodes.dtype.itemsize == 64
        indices = np.ascontiguousarray(indices, np.uint32)
        verts = np.ascontiguousarray(verts, np.float64)
        faces = np.ascontiguousarray(faces, np.uint32)
        h = self.lib.ref64_adopt(_p(nodes), len(nodes), _p(indices), len(indices), _p(verts), 24, _p(faces))
        acc = self.Accel(self, h, verts, faces) if h else None
        if acc:
            acc._keep = (nodes, indices)
        return acc


class ReferencePathTracer:
    """The reference path tracer's own shading functions (oracle/_ref/libpt_ref.so = the unmodified
    examples/path_tracer/main.cc behind oracle/pt_ref_shim.cc): MeshLight, sampleDirect, directionCosTheta,
    fresnel_schlick, reflect, refract ... driven one bounce at a time with caller-supplied random numbers."""

    @staticmethod
    def available():
        return os.path.exists(os.path.join(HERE, "_ref", "libpt_ref.so"))

    def __init__(self, verts, faces, material_ids, materials16, facevarying_normals=None):
        L = C.CDLL(os.path.join(HERE, "_ref", "libpt_ref.so"))
        vp, sz, u32 = C.c_void_p, C.c_size_t, C.c_uint32
        L.pt_ref_scene.restype = vp
        L.pt_ref_scene.argtypes = [vp, sz, vp, sz, vp, vp, vp, sz]
        L.pt_ref_scene_free.argtypes = [vp]
        L.pt_ref_emissive_faces.restype = sz
        L.pt_ref_emissive_faces.argtypes = [vp, vp, sz]
        L.pt_ref_face_normals.argtypes = [vp, vp, sz, vp]
        L.pt_ref_unexpected_draws.restype = C.c_long
        L.pt_ref_shade.argtypes = [vp, sz, u32, u32] + [vp] * 15
        self.L = L
        self.verts = np.ascontiguousarray(verts, np.float32)
        self.faces = np.ascontiguousarray(faces, np.uint32)
        self.ids = np.ascontiguousarray(material_ids, np.uint32)
        self.mats = np.ascontiguousarray(np.asarray(materials16).view(np.float32).reshape(-1, 16))
        if facevarying_normals is None:  # what the example's loader does for an OBJ without normals (calcNormal)
            fvn = np.zeros((len(self.faces), 9), np.float32)
            L.pt_ref_face_normals(self.verts.ctypes.data, self.faces.ctypes.data, len(self.faces), fvn.ctypes.data)
            facevarying_normals = fvn
        self.fvn = np.ascontiguousarray(facevarying_normals, np.float32)
        self.h = L.pt_ref_scene(self.verts.ctypes.data, len(self.verts), self.faces.ctypes.data, len(self.faces),
                                self.ids.ctypes.data, self.fvn.ctypes.data, self.mats.ctypes.data, len(self.mats))

    def __del__(self):
        try:
            self.L.pt_ref_scene_free(self.h)
        except Exception:
            pass

    def emissive_faces(self):
        out = np.zeros(len(self.faces), np.uint32)
        n = self.L.pt_ref_emissive_faces(self.h, out.ctypes.data, len(out))
        return out[:n].copy()

    def shade(self, bounce, max_bounces, org, dir, hit_uvt, hit_prim, weight_in, draws):
        """One bounce of main.cc's per-hit block for rays that hit; see oracle/pt_ref_shim.cc:pt_ref_shade."""
        n = len(hit_prim)
        f32 = lambda a, w: np.ascontiguousarray(a, np.float32).reshape(n, w)
        org, dir, hit_uvt, weight_in, draws = f32(org, 3), f32(dir, 3), f32(hit_uvt, 3), f32(weight_in, 4), f32(draws, 6)
        hit_prim = np.ascontiguousarray(hit_prim, np.uint32)
        out = {"flags": np.zeros(n, np.uint32), "next_org": np.zeros((n, 3), np.float32), "next_dir": np.zeros((n, 3), np.float32),
               "weight": np.zeros((n, 4), np.float32), "shadow_org": np.zeros((n, 3), np.float32),
               "shadow_dir": np.zeros((n, 3), np.float32), "shadow_max_t": np.zeros(n, np.float32),
               "shadow_contrib": np.zeros((n, 3), np.float32), "emission": np.zeros((n, 3), np.float32)}
        before = self.L.pt_ref_unexpected_draws()
        self.L.pt_ref_shade(self.h, n, int(bounce), int(max_bounces), org.ctypes.data, dir.ctypes.data, hit_uvt.ctypes.data,
                            hit_prim.ctypes.data, weight_in.ctypes.data, draws.ctypes.data, out["flags"].ctypes.data,
                            out["next_org"].ctypes.data, out["next_dir"].ctypes.data, out["weight"].ctypes.data,
                            out["shadow_org"].ctypes.data, out["shadow_dir"].ctypes.data, out["shadow_max_t"].ctypes.data,
                            out["shadow_contrib"].ctypes.data, out["emission"].ctypes.data)
        assert self.L.pt_ref_unexpected_draws() == before, "the reference drew a random number the harness did not queue"
        return out


class ReferenceSpheres:
    """The reference's custom-primitive model (oracle/_ref/libprim_ref{,03}.so = the unmodified
    examples/particle_primitive/main.cc: SphereGeometry, SpherePred, SphereIntersector) on the unmodified BVHAccel.
    `cpp11=False` is the same model built without NANORT_USE_CPP11_FEATURE (the C++03 vsafe_inverse).  The accel is
    the reference's own build (`options`: a BUILD_OPT_DTYPE record, None = the defaults) or, through `adopt`, any
    (nodes, indices) pair -- e.g. the device's tree -- loaded with the reference's own Load."""

    _libs = {}

    @staticmethod
    def _name(cpp11):
        return "libprim_ref.so" if cpp11 else "libprim_ref03.so"

    # the entry points added after the first version of the shim (refsph_build / refsph_traverse / refsph_free /
    # refsph_bounding_box): an oracle/_ref built from that version has none of them
    _EXACT = ("refsph_mode_cpp11", "refsph_build_opts", "refsph_adopt", "refsph_traverse_opts", "refsph_test_prims",
              "refsph_nan_rays", "refsph_node_box_hit")

    @staticmethod
    def available(cpp11=True):
        """the library exists: Build with the default options and Traverse with a prim id range"""
        return os.path.exists(os.path.join(HERE, "_ref", ReferenceSpheres._name(cpp11)))

    @classmethod
    def exact_available(cls, cpp11=True):
        """the library also has adopt, build and trace options, test_prim, nan_rays and box_hit"""
        if not cls.available(cpp11):
            return False
        L = cls._lib(cpp11)
        return all(hasattr(L, f) for f in cls._EXACT)

    @classmethod
    def _lib(cls, cpp11):
        if cpp11 in cls._libs:
            return cls._libs[cpp11]
        L = C.CDLL(os.path.join(HERE, "_ref", cls._name(cpp11)))
        vp, sz = C.c_void_p, C.c_size_t
        L.refsph_build.restype = vp
        L.refsph_build.argtypes = [vp, vp, sz]
        L.refsph_free.argtypes = [vp]
        L.refsph_bounding_box.argtypes = [vp, vp, vp]
        L.refsph_traverse.argtypes = [vp, vp, sz, vp, vp, C.c_uint32, C.c_uint32, C.c_int]
        if all(hasattr(L, f) for f in cls._EXACT):
            L.refsph_mode_cpp11.restype = C.c_int
            L.refsph_build_opts.restype = vp
            L.refsph_build_opts.argtypes = [vp, vp, sz, vp]
            L.refsph_adopt.restype = vp
            L.refsph_adopt.argtypes = [vp, sz, vp, sz, vp, vp, sz]
            L.refsph_num_nodes.restype = sz
            L.refsph_num_nodes.argtypes = [vp]
            L.refsph_num_indices.restype = sz
            L.refsph_num_indices.argtypes = [vp]
            L.refsph_copy_nodes.argtypes = [vp, vp]
            L.refsph_copy_indices.argtypes = [vp, vp]
            L.refsph_traverse_opts.argtypes = [vp, vp, sz, vp, vp, vp, C.c_int]
            L.refsph_test_prims.argtypes = [vp, vp, sz, vp, vp, vp, vp, vp]
            L.refsph_nan_rays.argtypes = [vp, vp, sz, vp, vp, C.c_int]
            L.refsph_node_box_hit.restype = C.c_int
            L.refsph_node_box_hit.argtypes = [vp, vp, sz]
            assert L.refsph_mode_cpp11() == (1 if cpp11 else 0)
        cls._libs[cpp11] = L
        return L

    def _need_exact(self, what):
        if not all(hasattr(self.L, f) for f in self._EXACT):
            raise RuntimeError(f"ReferenceSpheres.{what} needs an oracle/_ref built from the current prim_ref_shim.cc "
                               "(ReferenceSpheres.exact_available())")

    def __init__(self, centers, radii, cpp11=True, options=None, _adopt=None):
        self.L = L = self._lib(cpp11)
        self.cpp11 = cpp11
        self.centers = np.ascontiguousarray(centers, np.float32).reshape(-1, 3)
        self.radii = np.ascontiguousarray(radii, np.float32)
        assert len(self.centers) == len(self.radii)
        if _adopt is None and options is None:
            self.h = L.refsph_build(_p(self.centers), _p(self.radii), len(self.radii))
            assert self.h, "reference Build returned false"
        elif _adopt is None:
            self._need_exact("options")
            self.h = L.refsph_build_opts(_p(self.centers), _p(self.radii), len(self.radii), _p(options))
            assert self.h, "reference Build returned false"
        else:
            self._need_exact("adopt")
            nodes, indices = np.ascontiguousarray(_adopt[0]), np.ascontiguousarray(_adopt[1], np.uint32)
            assert nodes.dtype.itemsize == 40
            self.h = L.refsph_adopt(_p(nodes), len(nodes), _p(indices), len(indices), _p(self.centers), _p(self.radii),
                                    len(self.radii))
            assert self.h, "reference Load returned false"

    @classmethod
    def adopt(cls, nodes, indices, centers, radii, cpp11=True):
        """The reference's Traverse and SphereIntersector over a given tree (BVHAccel::Load of its Dump format)."""
        return cls(centers, radii, cpp11=cpp11, _adopt=(nodes, indices))

    def __del__(self):
        if getattr(self, "h", None):
            self.L.refsph_free(self.h)
            self.h = None

    def bounding_box(self):
        a, b = np.zeros(3, np.float32), np.zeros(3, np.float32)
        self.L.refsph_bounding_box(self.h, _p(a), _p(b))
        return a, b

    def nodes(self):
        self._need_exact("nodes")
        out = np.zeros(self.L.refsph_num_nodes(self.h), NODE_DTYPE)
        self.L.refsph_copy_nodes(self.h, _p(out))
        return out

    def indices(self):
        self._need_exact("indices")
        out = np.zeros(self.L.refsph_num_indices(self.h), np.uint32)
        self.L.refsph_copy_indices(self.h, _p(out))
        return out

    @staticmethod
    def _topts(prim_range, topts):
        if topts is None:
            topts = trace_options()
            if prim_range is not None:
                topts["prim_ids_range"] = prim_range
        else:
            assert prim_range is None
        return np.ascontiguousarray(topts, TRACE_OPT_DTYPE)

    def traverse(self, rays, prim_range=None, threads=8, topts=None):
        """One Traverse per ray: (hits, mask); hits are zero on a miss.  topts: a TRACE_OPT_DTYPE record, passed whole."""
        rays = np.ascontiguousarray(rays)
        assert rays.dtype.itemsize == 36
        hits = np.zeros(len(rays), HIT_DTYPE)
        mask = np.zeros(len(rays), np.uint8)
        t = self._topts(prim_range, topts)
        if hasattr(self.L, "refsph_traverse_opts"):
            self.L.refsph_traverse_opts(self.h, _p(rays), len(rays), _p(hits), _p(mask), _p(t), int(threads))
        else:  # the first version of the shim: the default trace options with an id range
            d = trace_options()
            assert all(int(d[f][0]) == int(t[f][0]) for f in ("skip_prim_id", "cull_back_face")), \
                "trace options other than prim_ids_range need ReferenceSpheres.exact_available()"
            lo, hi = (int(x) for x in t["prim_ids_range"][0])
            self.L.refsph_traverse(self.h, _p(rays), len(rays), _p(hits), _p(mask), lo, hi, int(threads))
        return hits, mask

    def test_prim(self, rays, prims, t_inout=None, prim_range=None, topts=None):
        """SphereIntersector::Intersect of sphere prims[i] on rays[i] from t = t_inout[i] (None: ray.max_t), then
        PostTraversal: (records, ok) -- the reference's full record had its Traverse picked prims[i]; ok = Intersect's
        return value (records are zero where it is False)."""
        self._need_exact("test_prim")
        rays = np.ascontiguousarray(rays).reshape(-1)
        prims = np.ascontiguousarray(np.broadcast_to(np.asarray(prims, np.uint32), (len(rays),)))
        if t_inout is not None:
            t_inout = np.ascontiguousarray(np.broadcast_to(np.asarray(t_inout, np.float32), (len(rays),)))
        hits = np.zeros(len(rays), HIT_DTYPE)
        ok = np.zeros(len(rays), np.uint8)
        self.L.refsph_test_prims(self.h, _p(rays), len(rays), _p(prims), _p(t_inout) if t_inout is not None else None,
                                 _p(self._topts(prim_range, topts)), _p(hits), _p(ok))
        return hits, ok.astype(bool)

    def nan_rays(self, rays, prim_range=None, topts=None, threads=8):
        """Rays for which some sphere inside the id range yields a NaN t (brute force over all spheres)."""
        self._need_exact("nan_rays")
        rays = np.ascontiguousarray(rays)
        out = np.zeros(len(rays), np.uint8)
        self.L.refsph_nan_rays(self.h, _p(rays), len(rays), _p(self._topts(prim_range, topts)), _p(out), int(threads))
        return out.astype(bool)

    def leaf_of(self):
        """leaf node index of every sphere in this accel's tree"""
        nodes, idx = self.nodes(), self.indices()
        leaves = np.flatnonzero(nodes["flag"] == 1)
        cnt, off = nodes["data"][leaves, 0].astype(np.int64), nodes["data"][leaves, 1].astype(np.int64)
        start = np.cumsum(cnt) - cnt
        slot = np.repeat(off, cnt) + (np.arange(int(cnt.sum())) - np.repeat(start, cnt))
        out = np.full(len(self.radii), -1, np.int64)
        out[idx[slot]] = np.repeat(leaves, cnt)
        return out

    def box_hit(self, ray, node):
        """Whether the box of `node` passes the reference's slab test over [ray.min_t, ray.max_t]."""
        self._need_exact("box_hit")
        ray = np.ascontiguousarray(ray).reshape(1)
        r = self.L.refsph_node_box_hit(self.h, _p(ray), int(node))
        assert r >= 0, f"no node {node}"
        return bool(r)
