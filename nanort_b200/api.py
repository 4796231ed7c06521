"""Python host side of the C-ABI (include/nanort_b200.h), mirroring nanort's own interface.

Names and argument meaning follow the reference header (nanort.h):
`BVHBuildOptions`, `BVHTraceOptions`, `BVHAccel.Build / Traverse / GetNodes / GetIndices /
GetStatistics / BoundingBox / IsValid` (nanort.h:559-624, 699-860).  `Traverse` takes a whole
array of 36-byte rays instead of one ray -- the batch form of the per-ray call.

All compute happens in nanort_b200/libnanort_b200.so (hand-written sm_90a CUDA).  There is no CPU
fallback: if the library or a CUDA device is missing, calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .scenes import HIT_DTYPE, NODE_DTYPE, RAY_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libnanort_b200.so")

BUILD_FAST = 0
BUILD_REFERENCE_TREE = 1          # bit-identical to CPU nanort's arrays (conformance build)
BUILD_REFERENCE_CPP03_ORDER = 2   # ... in the serial build's node order
TRAVERSE_FAST = 0
TRAVERSE_CONFORMANCE = 1
TRAVERSE_CPP03_INVERSE = 2
TRAVERSE_ANY_HIT = 8  # occlusion query: stop at the first hit inside [min_t, max_t) (see include/nanort_b200.h)
TRAVERSE_RAY32 = 4  # 32-byte ray records {org[3], dir[3], min_t, max_t} (no `type` word), 16-byte aligned

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
STATS_DTYPE = np.dtype(
    [("max_tree_depth", "<u4"), ("num_leaf_nodes", "<u4"), ("num_branch_nodes", "<u4"), ("build_secs", "<f4")]
)

# every symbol include/nanort_b200.h declares
EXPORTS = [
    "nrt_last_error", "nrt_device_count", "nrt_set_device", "nrt_build", "nrt_build_ex", "nrt_adopt", "nrt_free", "nrt_stats",
    "nrt_bounding_box", "nrt_nodes", "nrt_traverse", "nrt_traverse_device", "nrt_traverse_count_device",
    "nrt_host_alloc", "nrt_host_free", "nrt_render_ao_device", "nrt_ao_workload_device", "nrt_render_path_device",
    "nrt_scene_commit", "nrt_scene_free", "nrt_scene_bounding_box", "nrt_scene_nodes", "nrt_scene_instance_state",
    "nrt_scene_traverse", "nrt_scene_traverse_device", "nrt_scene_render_ao_device",
    "nrt_build_f64", "nrt_adopt_f64", "nrt_free_f64", "nrt_stats_f64", "nrt_bounding_box_f64", "nrt_nodes_f64", "nrt_traverse_f64", "nrt_traverse_f64_device",
    "nrt_path_bounce_device", "nrt_build_prims", "nrt_list_node_intersections",
    "nrt_comm_unique_id", "nrt_comm_init", "nrt_comm_free", "nrt_comm_rank", "nrt_render_ao_sharded",
    "nrt_probe_read_gbs", "nrt_probe_copy_gbs", "nrt_traverse_lane_stats_device", "nrt_build_f64_ex",
]


class NanortB200Error(RuntimeError):
    pass


class AoParams(C.Structure):
    _fields_ = [
        ("cam", C.c_float * 12),
        ("width", C.c_uint32), ("height", C.c_uint32),
        ("spp", C.c_uint32), ("sample0", C.c_uint32), ("seed", C.c_uint32),
        ("tile_w", C.c_uint32), ("tile_h", C.c_uint32),
        ("shard", C.c_uint32), ("n_shards", C.c_uint32),
        ("ray_min_t", C.c_float), ("ray_max_t", C.c_float),
        ("ao_min_t", C.c_float), ("ao_max_t", C.c_float),
        ("flags", C.c_uint32),
    ]


class AoResult(C.Structure):
    _fields_ = [
        ("primary_rays", C.c_uint64), ("ao_rays", C.c_uint64), ("ao_hits", C.c_uint64),
        ("traverse_ms", C.c_float), ("total_ms", C.c_float),
        ("launches", C.c_uint32), ("traverse_launches", C.c_uint32),
        ("primary_traverse_ms", C.c_float), ("ao_traverse_ms", C.c_float),
    ]


class PathParams(C.Structure):
    _fields_ = [
        ("cam", C.c_float * 12),
        ("width", C.c_uint32), ("height", C.c_uint32),
        ("spp", C.c_uint32), ("sample0", C.c_uint32), ("seed", C.c_uint32),
        ("tile_w", C.c_uint32), ("tile_h", C.c_uint32), ("shard", C.c_uint32), ("n_shards", C.c_uint32),
        ("max_bounces", C.c_uint32),
        ("ray_min_t", C.c_float), ("ray_max_t", C.c_float),
        ("n_materials", C.c_uint32), ("n_emissive", C.c_uint32),
        ("d_materials", C.c_void_p), ("d_material_ids", C.c_void_p), ("d_emissive_faces", C.c_void_p),
        ("d_facevarying_normals", C.c_void_p),
        ("flags", C.c_uint32), ("pad", C.c_uint32),
    ]


class PathResult(C.Structure):
    _fields_ = [
        ("camera_rays", C.c_uint64), ("radiance_rays", C.c_uint64), ("shadow_rays", C.c_uint64),
        ("traverse_ms", C.c_float), ("total_ms", C.c_float),
        ("launches", C.c_uint32), ("traverse_launches", C.c_uint32),
    ]


_lib = None


def lib():
    """Loads the CUDA library (fails loudly when it has not been built)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NanortB200Error(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nanort_b200 has no CPU fallback)"
        )
    L = C.CDLL(LIB_PATH)
    vp, sz, u32, u64p = C.c_void_p, C.c_size_t, C.c_uint32, C.POINTER(C.c_uint64)
    L.nrt_last_error.restype = C.c_char_p
    L.nrt_device_count.restype = C.c_int
    L.nrt_set_device.argtypes = [C.c_int]
    L.nrt_build.argtypes = [vp, sz, sz, vp, u32, vp, C.POINTER(vp)]
    L.nrt_build_ex.argtypes = [vp, sz, sz, vp, u32, vp, u32, C.POINTER(vp)]
    L.nrt_adopt.argtypes = [vp, sz, vp, sz, vp, sz, sz, vp, u32, C.POINTER(vp)]
    L.nrt_free.argtypes = [vp]
    L.nrt_free.restype = None
    L.nrt_stats.argtypes = [vp, vp]
    L.nrt_bounding_box.argtypes = [vp, vp, vp]
    L.nrt_nodes.argtypes = [vp, C.POINTER(vp), C.POINTER(sz), C.POINTER(vp), C.POINTER(sz)]
    L.nrt_traverse.argtypes = [vp, vp, sz, vp, vp, vp, u32]
    L.nrt_traverse_device.argtypes = [vp, vp, sz, vp, vp, vp, u32, vp]
    L.nrt_traverse_count_device.argtypes = [vp, vp, sz, vp, u32, u64p, u64p, vp]
    L.nrt_traverse_lane_stats_device.argtypes = [vp, vp, sz, vp, u32, u64p, vp]
    L.nrt_host_alloc.argtypes = [sz]
    L.nrt_host_alloc.restype = vp
    L.nrt_host_free.argtypes = [vp]
    L.nrt_host_free.restype = None
    L.nrt_render_ao_device.argtypes = [vp, C.POINTER(AoParams), vp, C.POINTER(AoResult), vp]
    L.nrt_ao_workload_device.argtypes = [vp, C.POINTER(AoParams), vp, vp, vp, u64p, u64p, vp]
    L.nrt_render_path_device.argtypes = [vp, C.POINTER(PathParams), vp, C.POINTER(PathResult), vp]
    L.nrt_scene_commit.argtypes = [vp, u32, u32, C.POINTER(vp)]
    L.nrt_scene_free.argtypes = [vp]
    L.nrt_scene_free.restype = None
    L.nrt_scene_bounding_box.argtypes = [vp, vp, vp]
    L.nrt_scene_nodes.argtypes = [vp, C.POINTER(vp), C.POINTER(sz), C.POINTER(vp), C.POINTER(sz)]
    L.nrt_scene_instance_state.argtypes = [vp, u32, vp]
    L.nrt_scene_traverse.argtypes = [vp, vp, sz, vp, vp, u32]
    L.nrt_scene_traverse_device.argtypes = [vp, vp, sz, vp, vp, u32, vp]
    L.nrt_scene_render_ao_device.argtypes = [vp, vp, vp, vp, vp]
    L.nrt_build_f64.argtypes = [vp, sz, sz, vp, u32, vp, C.POINTER(vp)]
    L.nrt_build_f64_ex.argtypes = [vp, sz, sz, vp, u32, vp, u32, C.POINTER(vp)]
    L.nrt_adopt_f64.argtypes = [vp, sz, vp, sz, vp, sz, sz, vp, u32, C.POINTER(vp)]
    L.nrt_free_f64.argtypes = [vp]
    L.nrt_free_f64.restype = None
    L.nrt_stats_f64.argtypes = [vp, vp]
    L.nrt_bounding_box_f64.argtypes = [vp, vp, vp]
    L.nrt_nodes_f64.argtypes = [vp, C.POINTER(vp), C.POINTER(sz), C.POINTER(vp), C.POINTER(sz)]
    L.nrt_traverse_f64.argtypes = [vp, vp, sz, vp, vp, vp, u32]
    L.nrt_traverse_f64_device.argtypes = [vp, vp, sz, vp, vp, vp, u32, vp]
    L.nrt_path_bounce_device.argtypes = [vp, C.POINTER(PathParams), u32, C.c_uint64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                         vp, u64p, u64p, C.c_int, vp]
    L.nrt_build_prims.argtypes = [u32, vp, sz, vp, u32, vp, C.POINTER(vp)]
    L.nrt_list_node_intersections.argtypes = [vp, vp, sz, C.c_int, vp, vp, u32]
    L.nrt_comm_unique_id.argtypes = [vp]
    L.nrt_comm_init.argtypes = [vp, C.c_int, C.c_int, C.POINTER(vp)]
    L.nrt_comm_free.argtypes = [vp]
    L.nrt_comm_free.restype = None
    L.nrt_comm_rank.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.nrt_render_ao_sharded.argtypes = [vp, vp, C.POINTER(AoParams), vp, C.POINTER(AoResult), vp]
    L.nrt_probe_read_gbs.argtypes = [sz, C.c_int, C.POINTER(C.c_double)]
    L.nrt_probe_copy_gbs.argtypes = [sz, C.c_int, C.c_int, C.POINTER(C.c_double)]
    _lib = L
    return L


def _check(rc):
    if rc != 0:
        raise NanortB200Error(f"nanort_b200 error {rc}: {lib().nrt_last_error().decode()}")


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def BVHBuildOptions(**kw):
    """nanort::BVHBuildOptions<float> with the reference defaults (nanort.h:574-582)."""
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


def BVHTraceOptions(**kw):
    """nanort::BVHTraceOptions with the reference defaults (nanort.h:617-623)."""
    o = np.zeros(1, TRACE_OPT_DTYPE)
    o["prim_ids_range"] = (0, 0x7FFFFFFF)
    o["skip_prim_id"] = 0xFFFFFFFF
    for k, v in kw.items():
        o[k] = v
    return o


AO_UNFUSED = 0x10000
AO_PACKED_TILES = 0x20000


def probe_read_gbs(nbytes, iters=10, device=None):
    """Measured streaming-read bandwidth (GB/s) over nbytes of device memory: L2 roof for <= 64 MB, HBM for >= 1 GB."""
    if device is not None:
        _check(lib().nrt_set_device(int(device)))
    v = C.c_double(0.0)
    _check(lib().nrt_probe_read_gbs(int(nbytes), int(iters), C.byref(v)))
    return v.value


def probe_copy_gbs(nbytes, direction, iters=5, device=None):
    """Measured pinned host<->device copy rate (GB/s); direction 0 = H2D, 1 = D2H."""
    if device is not None:
        _check(lib().nrt_set_device(int(device)))
    v = C.c_double(0.0)
    _check(lib().nrt_probe_copy_gbs(int(nbytes), int(iters), int(direction), C.byref(v)))
    return v.value


class Comm:
    """Multi-GPU communicator of the C-ABI (nrt_comm_*): one per process / GPU, NCCL underneath (bound at run time)."""

    @staticmethod
    def unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        _check(lib().nrt_comm_unique_id(C.cast(buf, C.c_void_p)))
        return buf.raw

    def __init__(self, unique_id: bytes, rank: int, world: int, device: int | None = None):
        assert len(unique_id) == 128
        if device is not None:
            _check(lib().nrt_set_device(int(device)))
        h = C.c_void_p()
        buf = C.create_string_buffer(unique_id, 128)
        _check(lib().nrt_comm_init(C.cast(buf, C.c_void_p), int(rank), int(world), C.byref(h)))
        self._h, self.rank, self.world = h, rank, world

    def free(self):
        if self._h:
            lib().nrt_comm_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def RenderAO(self, accel, params: AoParams, d_frame_full_ptr, stream=None, want_result=True):
        """nrt_render_ao_sharded: this rank's tiles + framebuffer all-gather; every rank's d_frame_full holds the frame."""
        res = AoResult()
        _check(lib().nrt_render_ao_sharded(accel._h, self._h, C.byref(params), C.c_void_p(d_frame_full_ptr),
                                           C.byref(res) if want_result else None, C.c_void_p(stream) if stream else None))
        return res if want_result else None


PRIM_SPHERES = 1
PRIM_BOXES = 2
NODE_HIT_DTYPE = np.dtype([("t_min", np.float32), ("t_max", np.float32), ("node_id", np.uint32)])


class PinnedArray:
    """numpy view over cudaMallocHost memory (nrt_host_alloc)."""

    def __init__(self, shape, dtype):
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) * dtype.itemsize
        self._ptr = lib().nrt_host_alloc(max(n, 1))
        if not self._ptr:
            raise NanortB200Error("nrt_host_alloc failed: " + lib().nrt_last_error().decode())
        buf = (C.c_char * max(n, 1)).from_address(self._ptr)
        self.array = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    def free(self):
        if self._ptr:
            self.array = None
            lib().nrt_host_free(self._ptr)
            self._ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class BVHAccel:
    """nanort::BVHAccel<float> over TriangleMesh / TriangleSAHPred / TriangleIntersector."""

    def __init__(self, device: int | None = None):
        self._h = None
        self._device = device

    # -- lifetime
    def _set_device(self):
        if self._device is not None:
            _check(lib().nrt_set_device(int(self._device)))

    def free(self):
        if self._h:
            lib().nrt_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def IsValid(self):
        return self._h is not None

    # -- build
    def Build(self, num_primitives, vertices, faces, options=None, vertex_stride_bytes=12, flags=BUILD_FAST):
        """BVHAccel::Build(num_primitives, TriangleMesh(vertices, faces, stride), pred, options)
        (nanort.h:716-718).  Returns False for num_primitives == 0 like the reference."""
        self.free()
        if num_primitives == 0:
            return False
        vertices = np.ascontiguousarray(vertices, np.float32)
        faces = np.ascontiguousarray(faces, np.uint32)
        self._set_device()
        h = C.c_void_p()
        n_verts = vertices.size * 4 // vertex_stride_bytes
        _check(lib().nrt_build_ex(_p(vertices), vertex_stride_bytes, n_verts, _p(faces), int(num_primitives),
                                  _p(options), int(flags), C.byref(h)))
        self._h = h
        return True

    def Adopt(self, nodes, indices, vertices, faces, vertex_stride_bytes=12):
        """Conformance entry: traverse an existing nanort-layout tree (nrt_adopt)."""
        self.free()
        nodes = np.ascontiguousarray(nodes)
        assert nodes.dtype.itemsize == 40
        indices = np.ascontiguousarray(indices, np.uint32)
        vertices = np.ascontiguousarray(vertices, np.float32)
        faces = np.ascontiguousarray(faces, np.uint32)
        self._set_device()
        h = C.c_void_p()
        n_verts = vertices.size * 4 // vertex_stride_bytes
        _check(lib().nrt_adopt(_p(nodes), len(nodes), _p(indices), len(indices), _p(vertices), vertex_stride_bytes,
                               n_verts, _p(faces), faces.size // 3, C.byref(h)))
        self._h = h
        return True

    # -- accessors
    def GetStatistics(self):
        s = np.zeros(1, STATS_DTYPE)
        _check(lib().nrt_stats(self._h, _p(s)))
        return {k: s[k][0].item() for k in STATS_DTYPE.names}

    def BoundingBox(self):
        if not self._h:  # nanort.h:793-795
            m = np.finfo(np.float32).max
            return np.full(3, m, np.float32), np.full(3, -m, np.float32)
        a, b = np.zeros(3, np.float32), np.zeros(3, np.float32)
        _check(lib().nrt_bounding_box(self._h, _p(a), _p(b)))
        return a, b

    def _mirrors(self):
        pn, pi = C.c_void_p(), C.c_void_p()
        nn, ni = C.c_size_t(), C.c_size_t()
        _check(lib().nrt_nodes(self._h, C.byref(pn), C.byref(nn), C.byref(pi), C.byref(ni)))
        nodes = np.frombuffer((C.c_char * (nn.value * 40)).from_address(pn.value), NODE_DTYPE)
        idx = np.frombuffer((C.c_char * (ni.value * 4)).from_address(pi.value), np.uint32)
        return nodes, idx

    def GetNodes(self):
        return self._mirrors()[0].copy()

    def GetIndices(self):
        return self._mirrors()[1].copy()

    # -- traversal
    def Traverse(self, rays, options=None, flags=TRAVERSE_FAST, hits=None, mask=None):
        """Batch of BVHAccel::Traverse calls on HOST arrays (nrt_traverse): returns (hits, mask);
        mask[i] is Traverse's bool, hits[i] = {u,v,t,prim_id} where mask[i] == 1."""
        rays = np.ascontiguousarray(rays)
        assert rays.dtype.itemsize == (32 if int(flags) & TRAVERSE_RAY32 else 36)
        n = len(rays)
        if hits is None:
            hits = np.zeros(n, HIT_DTYPE)
        if mask is None:
            mask = np.zeros(n, np.uint8)
        elif mask is False:  # no hit flags wanted: a miss is prim_id == 0xFFFFFFFF
            mask = None
        _check(lib().nrt_traverse(self._h, _p(rays), n, _p(hits), _p(mask), _p(options), int(flags)))
        return hits, mask

    def TraverseDevice(self, d_rays_ptr, n, d_hits_ptr, d_mask_ptr=None, options=None, flags=TRAVERSE_FAST,
                       stream=None):
        """Device-pointer form (nrt_traverse_device); pointers are ints (e.g. torch.Tensor.data_ptr())."""
        _check(lib().nrt_traverse_device(self._h, C.c_void_p(d_rays_ptr), int(n), C.c_void_p(d_hits_ptr),
                                         C.c_void_p(d_mask_ptr) if d_mask_ptr else None, _p(options), int(flags),
                                         C.c_void_p(stream) if stream else None))

    def CountDevice(self, d_rays_ptr, n, options=None, flags=TRAVERSE_FAST, stream=None):
        """Visit counters for the roofline arithmetic (nrt_traverse_count_device)."""
        b, p = C.c_uint64(), C.c_uint64()
        _check(lib().nrt_traverse_count_device(self._h, C.c_void_p(d_rays_ptr), int(n), _p(options), int(flags),
                                               C.byref(b), C.byref(p), C.c_void_p(stream) if stream else None))
        return b.value, p.value

    LANE_STAT_NAMES = ("boxes", "prims", "refill_events", "lanes_refilled", "node_steps", "lanes_testing", "lanes_no_ray",
                       "lanes_finished", "lanes_parked_on_leaves", "leaf_rounds", "lanes_with_leaf", "tri_steps",
                       "retire_events", "lanes_retired", "outer_iterations", "reserved")

    def LaneStatsDevice(self, d_rays_ptr, n, options=None, flags=TRAVERSE_FAST, stream=None):
        """How the persistent warps' lanes spent their steps on these rays (nrt_traverse_lane_stats_device)."""
        out = (C.c_uint64 * 16)()
        _check(lib().nrt_traverse_lane_stats_device(self._h, C.c_void_p(d_rays_ptr), int(n), _p(options), int(flags), out,
                                                    C.c_void_p(stream) if stream else None))
        return dict(zip(self.LANE_STAT_NAMES, [int(x) for x in out]))

    def ExportAOWorkload(self, params: AoParams, d_accum_ptr, d_primary_ptr, d_ao_ptr, stream=None):
        """Same pass, also writing both ray queues as 36-byte rays (nrt_ao_workload_device)."""
        n_p, n_a = C.c_uint64(), C.c_uint64()
        _check(lib().nrt_ao_workload_device(self._h, C.byref(params), C.c_void_p(d_accum_ptr),
                                            C.c_void_p(d_primary_ptr), C.c_void_p(d_ao_ptr), C.byref(n_p),
                                            C.byref(n_a), C.c_void_p(stream) if stream else None))
        return n_p.value, n_a.value

    def RenderPath(self, params: PathParams, d_accum_rgb_ptr, stream=None, want_result=True):
        """Wavefront path tracing pass (nrt_render_path_device)."""
        res = PathResult()
        _check(lib().nrt_render_path_device(self._h, C.byref(params), C.c_void_p(d_accum_rgb_ptr),
                                            C.byref(res) if want_result else None,
                                            C.c_void_p(stream) if stream else None))
        return res

    def BuildSpheres(self, centers, radii, options=None, center_stride_bytes=12):
        """BVHAccel::Build(n, SphereGeometry(centers, radii), SpherePred(centers), options) of the reference's
        particle_primitive model (nrt_build_prims, NRT_PRIM_SPHERES).  Traverse() then returns sphere hit records.
        Centre i is the three floats at byte offset i * center_stride_bytes of `centers` (a multiple of 4, >= 12).
        Traverse flags on the result: TRAVERSE_CPP03_INVERSE as for triangles; TRAVERSE_CONFORMANCE and TRAVERSE_ANY_HIT
        are ignored (closest hit, the same records); TRAVERSE_RAY32, CountDevice and LaneStatsDevice are refused."""
        self.free()
        self._set_device()
        radii = np.ascontiguousarray(radii, np.float32)
        centers = np.ascontiguousarray(centers, np.float32).reshape(-1)
        assert center_stride_bytes >= 12 and center_stride_bytes % 4 == 0
        assert len(radii) == 0 or centers.size * 4 >= (len(radii) - 1) * center_stride_bytes + 12
        h = C.c_void_p()
        rc = lib().nrt_build_prims(PRIM_SPHERES, _p(centers), int(center_stride_bytes), _p(radii), len(radii), _p(options),
                                   C.byref(h))
        if rc != 0:
            if len(radii) == 0:
                return False
            _check(rc)
        self._h = h
        self._keep = (centers, radii)
        return True

    def BuildBoxes(self, boxes6, options=None):
        """A tree over axis-aligned boxes {bmin, bmax} (the node-level primitive of the two-level API); query with
        ListNodeIntersections()."""
        self.free()
        self._set_device()
        boxes6 = np.ascontiguousarray(boxes6, np.float32).reshape(-1, 6)
        h = C.c_void_p()
        rc = lib().nrt_build_prims(PRIM_BOXES, _p(boxes6), 24, None, len(boxes6), _p(options), C.byref(h))
        if rc != 0:
            if len(boxes6) == 0:
                return False
            _check(rc)
        self._h = h
        return True

    def ListNodeIntersections(self, rays, max_intersections=64, flags=0):
        """BVHAccel::ListNodeIntersections for every ray: (hits[n, max], counts[n]); hits[i, :counts[i]] nearest first."""
        rays = np.ascontiguousarray(rays)
        n = len(rays)
        hits = np.zeros((n, max_intersections), NODE_HIT_DTYPE)
        counts = np.zeros(n, np.uint32)
        _check(lib().nrt_list_node_intersections(self._h, _p(rays), n, int(max_intersections), _p(hits), _p(counts), int(flags)))
        return hits, counts

    def PathBounce(self, params: PathParams, bounce, n_rays, d_org_tmin, d_dir_tmax, d_path_id, d_weight, d_out_org_tmin,
                   d_out_dir_tmax, d_out_path_id, d_sh_org_tmin, d_sh_dir_tmax, d_sh_contrib_pix, d_accum_rgb,
                   skip_shadow_pass=False, stream=None):
        """nrt_path_bounce_device: one bounce on caller-owned device queues; returns (n_continue, n_shadow)."""
        nc, ns = C.c_uint64(0), C.c_uint64(0)
        vp = C.c_void_p
        _check(lib().nrt_path_bounce_device(self._h, C.byref(params), int(bounce), int(n_rays), vp(d_org_tmin), vp(d_dir_tmax),
                                            vp(d_path_id), vp(d_weight), vp(d_out_org_tmin), vp(d_out_dir_tmax),
                                            vp(d_out_path_id), vp(d_sh_org_tmin), vp(d_sh_dir_tmax), vp(d_sh_contrib_pix),
                                            vp(d_accum_rgb), C.byref(nc), C.byref(ns), 1 if skip_shadow_pass else 0,
                                            vp(stream) if stream else None))
        return int(nc.value), int(ns.value)

    def RenderAO(self, params: AoParams, d_accum_ptr, stream=None, want_result=True):
        res = AoResult()
        _check(lib().nrt_render_ao_device(self._h, C.byref(params), C.c_void_p(d_accum_ptr),
                                          C.byref(res) if want_result else None,
                                          C.c_void_p(stream) if stream else None))
        return res


# ------------------------------------------------------------------ two-level scene (examples/nanosg)
SCENE_HIT_DTYPE = np.dtype([("u", "<f4"), ("v", "<f4"), ("t", "<f4"), ("prim_id", "<u4"), ("node_id", "<u4"),
                            ("P", "<f4", (3,))])
INSTANCE_STATE_DTYPE = np.dtype([("xform", "<f4", (4, 4)), ("inv", "<f4", (4, 4)), ("inv33", "<f4", (4, 4)),
                                 ("invT33", "<f4", (4, 4)), ("lbmin", "<f4", (3,)), ("lbmax", "<f4", (3,)),
                                 ("xbmin", "<f4", (3,)), ("xbmax", "<f4", (3,))])


class Instance(C.Structure):
    _fields_ = [("accel", C.c_void_p), ("xform", C.c_float * 16)]


class Scene:
    """Mirror of nanosg::Scene (examples/nanosg/nanosg.h:664-905): AddNode(accel, xform) ..., Commit(), Traverse.
    The accels are borrowed and kept alive by this object."""

    def __init__(self):
        self._h = None
        self._nodes = []

    def __del__(self):
        try:
            if self._h:
                lib().nrt_scene_free(self._h)
                self._h = None
        except Exception:
            pass

    def AddNode(self, accel: "BVHAccel", xform) -> bool:
        x = np.ascontiguousarray(xform, np.float32).reshape(16)
        self._nodes.append((accel, x))
        return True

    def Commit(self, flags=BUILD_FAST) -> bool:
        if self._h:
            lib().nrt_scene_free(self._h)
            self._h = None
        n = len(self._nodes)
        arr = (Instance * max(n, 1))()
        for i, (a, x) in enumerate(self._nodes):
            arr[i].accel = a._h
            arr[i].xform[:] = x.tolist()
        h = C.c_void_p()
        rc = lib().nrt_scene_commit(C.cast(arr, C.c_void_p), n, int(flags), C.byref(h))
        if rc == -1 and n == 0:  # Commit() returns false for an empty scene (nanosg.h:708-711)
            return False
        _check(rc)
        self._h = h
        return True

    def GetBoundingBox(self):
        a, b = np.zeros(3, np.float32), np.zeros(3, np.float32)
        _check(lib().nrt_scene_bounding_box(self._h, _p(a), _p(b)))
        return a, b

    def GetTopLevel(self):
        pn, nn, pi, ni = C.c_void_p(), C.c_size_t(), C.c_void_p(), C.c_size_t()
        _check(lib().nrt_scene_nodes(self._h, C.byref(pn), C.byref(nn), C.byref(pi), C.byref(ni)))
        nodes = np.frombuffer((C.c_char * (nn.value * 40)).from_address(pn.value), NODE_DTYPE).copy()
        idx = np.frombuffer((C.c_char * (ni.value * 4)).from_address(pi.value), np.uint32).copy()
        return nodes, idx

    def InstanceStates(self):
        out = np.zeros(len(self._nodes), INSTANCE_STATE_DTYPE)
        for i in range(len(self._nodes)):
            _check(lib().nrt_scene_instance_state(self._h, i, out[i:i + 1].ctypes.data))
        return out

    def Traverse(self, rays, flags=TRAVERSE_FAST):
        """Batch of Scene::Traverse calls on HOST arrays: (hits, mask)."""
        rays = np.ascontiguousarray(rays)
        assert rays.dtype.itemsize == 36
        n = len(rays)
        hits, mask = np.zeros(n, SCENE_HIT_DTYPE), np.zeros(n, np.uint8)
        _check(lib().nrt_scene_traverse(self._h, _p(rays), n, _p(hits), _p(mask), int(flags)))
        return hits, mask

    def TraverseDevice(self, d_rays_ptr, n, d_hits_ptr, d_mask_ptr=None, flags=TRAVERSE_FAST, stream=None):
        """Asynchronous on `stream`.  Any number of calls (and scene AO passes) on one scene may be in flight on any
        streams at once: a call is ordered on the device after the earlier call that used the same one of the
        scene's four scratch sets; the host does not wait."""
        _check(lib().nrt_scene_traverse_device(self._h, C.c_void_p(d_rays_ptr), int(n), C.c_void_p(d_hits_ptr),
                                               C.c_void_p(d_mask_ptr) if d_mask_ptr else None, int(flags),
                                               C.c_void_p(stream) if stream else None))

    def RenderAO(self, params: "AoParams", d_accum_ptr, stream=None):
        """Primary + 1-bounce AO over the two-level scene (nrt_scene_render_ao_device); same parameters as
        BVHAccel.RenderAO."""
        res = AoResult()
        _check(lib().nrt_scene_render_ao_device(self._h, C.byref(params), C.c_void_p(d_accum_ptr), C.byref(res),
                                                C.c_void_p(stream) if stream else None))
        return res


# ------------------------------------------------------------------ BVHAccel<double>
RAY64_DTYPE = np.dtype([("org", "<f8", (3,)), ("dir", "<f8", (3,)), ("min_t", "<f8"), ("max_t", "<f8"),
                        ("type", "<u4"), ("pad", "<u4")])
HIT64_DTYPE = np.dtype([("u", "<f8"), ("v", "<f8"), ("t", "<f8"), ("prim_id", "<u4"), ("pad", "<u4")])
NODE64_DTYPE = np.dtype([("bmin", "<f8", (3,)), ("bmax", "<f8", (3,)), ("flag", "<i4"), ("axis", "<i4"),
                         ("data", "<u4", (2,))])
BUILD_OPT64_DTYPE = np.dtype([("cost_t_aabb", "<f8"), ("min_leaf_primitives", "<u4"), ("max_tree_depth", "<u4"),
                              ("bin_size", "<u4"), ("shallow_depth", "<u4"),
                              ("min_primitives_for_parallel_build", "<u4"), ("cache_bbox", "u1"), ("pad", "u1", (3,))])
assert (RAY64_DTYPE.itemsize, HIT64_DTYPE.itemsize, NODE64_DTYPE.itemsize, BUILD_OPT64_DTYPE.itemsize) == (72, 32, 64, 32)


class BVHAccelF64:
    """Mirror of nanort::BVHAccel<double> (nrt_build_f64 / nrt_traverse_f64)."""

    def __init__(self, device=None):
        self._h = None
        self._device = device

    def free(self):
        if self._h:
            lib().nrt_free_f64(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def Build(self, num_primitives, vertices, faces, options=None, vertex_stride_bytes=24, flags=BUILD_FAST):
        """flags=BUILD_REFERENCE_TREE: the reference's own BVHNode<double> array, bit for bit (nrt_build_f64_ex)."""
        self.free()
        if num_primitives == 0:
            return False
        vertices = np.ascontiguousarray(vertices, np.float64)
        faces = np.ascontiguousarray(faces, np.uint32)
        if self._device is not None:
            _check(lib().nrt_set_device(int(self._device)))
        h = C.c_void_p()
        n_verts = vertices.size * 8 // vertex_stride_bytes
        _check(lib().nrt_build_f64_ex(_p(vertices), vertex_stride_bytes, n_verts, _p(faces), int(num_primitives),
                                      _p(options), int(flags), C.byref(h)))
        self._h = h
        return True

    def Adopt(self, nodes, indices, vertices, faces):
        """Traverse an existing BVHNode<double> array (e.g. the CPU reference's), nrt_adopt_f64."""
        self.free()
        nodes = np.ascontiguousarray(nodes)
        assert nodes.dtype.itemsize == 64
        indices = np.ascontiguousarray(indices, np.uint32)
        vertices = np.ascontiguousarray(vertices, np.float64)
        faces = np.ascontiguousarray(faces, np.uint32)
        if self._device is not None:
            _check(lib().nrt_set_device(int(self._device)))
        h = C.c_void_p()
        _check(lib().nrt_adopt_f64(_p(nodes), len(nodes), _p(indices), len(indices), _p(vertices), 24,
                                   vertices.size // 3, _p(faces), faces.size // 3, C.byref(h)))
        self._h = h
        return True

    def GetStatistics(self):
        s = np.zeros(1, STATS_DTYPE)
        _check(lib().nrt_stats_f64(self._h, _p(s)))
        return {k: s[k][0].item() for k in STATS_DTYPE.names}

    def BoundingBox(self):
        a, b = np.zeros(3, np.float64), np.zeros(3, np.float64)
        _check(lib().nrt_bounding_box_f64(self._h, _p(a), _p(b)))
        return a, b

    def GetNodes(self):
        return self._mirror()[0]

    def GetIndices(self):
        return self._mirror()[1]

    def _mirror(self):
        pn, nn, pi, ni = C.c_void_p(), C.c_size_t(), C.c_void_p(), C.c_size_t()
        _check(lib().nrt_nodes_f64(self._h, C.byref(pn), C.byref(nn), C.byref(pi), C.byref(ni)))
        nodes = np.frombuffer((C.c_char * (nn.value * 64)).from_address(pn.value), NODE64_DTYPE).copy()
        idx = np.frombuffer((C.c_char * (ni.value * 4)).from_address(pi.value), np.uint32).copy()
        return nodes, idx

    def Traverse(self, rays, options=None, flags=0, hits=None, mask=None):
        """Batch of BVHAccel<double>::Traverse calls on HOST arrays (nrt_traverse_f64).  flags: TRAVERSE_FAST (default,
        persistent-warp kernel) or TRAVERSE_CONFORMANCE (the reference's visiting order), TRAVERSE_CPP03_INVERSE."""
        rays = np.ascontiguousarray(rays)
        assert rays.dtype.itemsize == 72
        n = len(rays)
        if hits is None:
            hits = np.zeros(n, HIT64_DTYPE)
        if mask is None:
            mask = np.zeros(n, np.uint8)
        _check(lib().nrt_traverse_f64(self._h, _p(rays), n, _p(hits), _p(mask), _p(options), int(flags)))
        return hits, mask

    def TraverseDevice(self, d_rays_ptr, n, d_hits_ptr, d_mask_ptr=None, options=None, flags=0, stream=None):
        """Device-pointer form (nrt_traverse_f64_device): 72-byte rays in, 32-byte records out."""
        _check(lib().nrt_traverse_f64_device(self._h, C.c_void_p(d_rays_ptr), int(n), C.c_void_p(d_hits_ptr),
                                             C.c_void_p(d_mask_ptr) if d_mask_ptr else None, _p(options), int(flags),
                                             C.c_void_p(stream) if stream else None))
