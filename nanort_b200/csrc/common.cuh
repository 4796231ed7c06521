// Shared types and helpers of the nanort_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <atomic>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/nanort_b200.h"

namespace nrt {

void set_error(const std::string &msg);
int cuda_fail(cudaError_t e, const char *what, const char *file, int line);

#define NRT_CUDA(expr)                                                     \
  do {                                                                     \
    cudaError_t _e = (expr);                                               \
    if (_e != cudaSuccess) return nrt::cuda_fail(_e, #expr, __FILE__, __LINE__); \
  } while (0)

// Every entry point makes the accel's device current for its own duration only and puts the caller's device back:
// a host that drives several GPUs from one thread (or torch, whose current_device() is cudaGetDevice) must not find
// its current device switched by a library call -- nrt_free from a garbage collector included.
struct DeviceGuard {
  int prev = -1;
  cudaError_t err = cudaSuccess;
  DeviceGuard() {  // only remembers the caller's device (for entry points that select one themselves)
    if (cudaGetDevice(&prev) != cudaSuccess) {
      prev = -1;
      cudaGetLastError();
    }
  }
  explicit DeviceGuard(int device) {
    if (cudaGetDevice(&prev) != cudaSuccess) {
      prev = -1;
      cudaGetLastError();
    }
    if (prev != device) err = cudaSetDevice(device);
    if (prev == device) prev = -1;  // nothing to restore
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
  DeviceGuard(const DeviceGuard &) = delete;
  DeviceGuard &operator=(const DeviceGuard &) = delete;
};
#define NRT_DEVICE(dev)            \
  nrt::DeviceGuard _nrt_dg((dev)); \
  NRT_CUDA(_nrt_dg.err)

}  // namespace nrt

#include "host_slots.cuh"

namespace nrt {

// ---- nanort-layout records (byte-compatible, see include/nanort_b200.h) ----
struct Node40 {
  float bmin[3];
  float bmax[3];
  int32_t flag;  // 1 leaf, 0 branch
  int32_t axis;
  uint32_t data[2];  // leaf {count, first}; branch {left, right}
};
static_assert(sizeof(Node40) == 40, "BVHNode<float> layout");

struct Node64 {  // Node40 with double boxes
  double bmin[3];
  double bmax[3];
  int32_t flag;
  int32_t axis;
  uint32_t data[2];
};
static_assert(sizeof(Node64) == 64, "BVHNode<double> layout");

template <typename T>
using BVHNodeOf = typename std::conditional<std::is_same<T, float>::value, Node40, Node64>::type;

struct Ray36 {
  float org[3];
  float dir[3];
  float min_t, max_t;
  uint32_t type;
};
static_assert(sizeof(Ray36) == 36, "Ray<float> layout");

struct Hit16 {
  float u, v, t;
  uint32_t prim_id;
};
static_assert(sizeof(Hit16) == 16, "TriangleIntersection<float> layout");

struct BuildOptions28 {
  float cost_t_aabb;
  uint32_t min_leaf_primitives;
  uint32_t max_tree_depth;
  uint32_t bin_size;
  uint32_t shallow_depth;
  uint32_t min_primitives_for_parallel_build;
  uint8_t cache_bbox;
  uint8_t pad[3];
};
static_assert(sizeof(BuildOptions28) == 28, "BVHBuildOptions<float> layout");

struct BuildStats16 {
  uint32_t max_tree_depth, num_leaf_nodes, num_branch_nodes;
  float build_secs;
};
static_assert(sizeof(BuildStats16) == 16, "BVHBuildStatistics layout");

struct TraceOptions16 {
  uint32_t prim_ids_range[2];
  uint32_t skip_prim_id;
  uint8_t cull_back_face;
  uint8_t pad[3];
};
static_assert(sizeof(TraceOptions16) == 16, "BVHTraceOptions layout");

// ---- private traversal layout -------------------------------------------------
// One 64-byte record per BRANCH node holding BOTH child boxes, so one aligned
// 4 x 16-byte fetch decides both children (the nanort array needs three
// dependent 40-byte fetches for the same decision).
//   q0 = c0.lo.xyz, c0.hi.x     q1 = c0.hi.yz, c1.lo.xy
//   q2 = c1.lo.z, c1.hi.xyz     q3 = ref0, ref1, axis, unused
// ref >= 0: index of the child's WideNode; ref < 0: leaf, ~ref = first slot in
// the packed triangle array.  A leaf with no triangles is ref == kEmptyLeaf.
// The array holds the branch nodes in the nanort array's (depth-first) order, so the root is wide[0].
struct WideNode {
  float4 q0, q1, q2;
  int4 q3;
};
static_assert(sizeof(WideNode) == 64, "WideNode");
constexpr int kEmptyLeaf = (int)0x80000000;  // ~0x7FFFFFFF: never a valid slot

// Packed triangle, 48 bytes, in leaf (indices_) order:
//   v0.xyz, prim_id | v1.xyz, last_in_leaf flag (1/0 as uint bits) | v2.xyz, 0
struct PackedTri {
  float4 a, b, c;
};
static_assert(sizeof(PackedTri) == 48, "PackedTri");

// Rules of the child-pair layouts for either node type (Node40 -> WideNode, layout.cu; Node64 -> PairNodeD,
// f64_fast.cuh): a branch gets the child-pair record whose index is the exclusive scan of these flags, and a child's
// reference in its parent's record is that index (branch), kEmptyLeaf (leaf without primitives) or ~first slot (leaf).
template <class NodeT>
__global__ void branch_flags_kernel(const NodeT *__restrict__ nodes, uint32_t n, uint32_t *__restrict__ flags) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[i] = nodes[i].flag == 0 ? 1u : 0u;
}

template <class NodeT>
__device__ __forceinline__ int child_ref(const NodeT &c, uint32_t cidx, const uint32_t *widx) {
  if (c.flag == 0) return (int)widx[cidx];
  if (c.data[0] == 0) return kEmptyLeaf;
  return ~(int)c.data[1];
}

// ---- round-2 traversal layout (traverse_fast3_kernel) ------------------------------------------------------
// PairNode, 128 bytes = one L1 line, one per BRANCH node, both child boxes.  Every axis owns one 32-byte sector that
// holds the four planes of that axis in BOTH orders,
//   sector x = { lo0 lo1 hi0 hi1 | hi0 hi1 lo0 lo1 }     (y, z alike)
// so a ray loads ONE aligned float4 per axis at byte offset (dir_sign ? 16 : 0) and finds {near0 near1 far0 far1}
// in fixed registers: the reference's `ray_dir_sign ? bmax : bmin` selection (nanort.h:2291-2302) becomes address
// arithmetic done once per ray instead of 12 selects per visited pair.  Sector 3 = {ref0, ref1, axis, 0, ...}.
struct PairNode {
  float4 x[2], y[2], z[2];
  int4 r, pad;
};
static_assert(sizeof(PairNode) == 128, "PairNode");

// TriCM, 48 bytes, component-major packed triangle in leaf order:
//   X = {a.x b.x c.x w}  Y = {a.y b.y c.y w}  Z = {a.z b.z c.z w},  w = prim_id | last_in_leaf << 31 (in all three)
// The watertight test permutes the components by the ray's (kx, ky, kz) (nanort.h:1073-1081); with this layout the
// permutation is again an address: the ray loads the float4 at byte offset 16 * k and needs no selects.
struct TriCM {
  float4 X, Y, Z;
};
static_assert(sizeof(TriCM) == 48, "TriCM");

// ---- accel object ----------------------------------------------------------------
struct Accel {
  int device = 0;
  uint32_t n_prims = 0;
  size_t n_nodes = 0;
  size_t n_wide = 0;
  bool root_is_leaf = false;
  // device: reference-layout tree + original geometry (conformance walk)
  Node40 *d_nodes = nullptr;
  uint32_t *d_indices = nullptr;
  float *d_verts = nullptr;  // tightly packed float3 (stride 12)
  size_t n_verts = 0;
  uint32_t *d_faces = nullptr;
  // when set, the primitives of this accel are n_prims axis-aligned boxes (6 floats each: bmin, bmax) instead of
  // triangles -- the top-level tree of a two-level scene; such an accel has no private traversal layout
  float *d_prim_boxes = nullptr;
  // 0 = triangles; NRT_PRIM_SPHERES / NRT_PRIM_BOXES: primitives of another kind built through their boxes (prims.cu)
  int prim_kind = 0;
  void *d_prim_data = nullptr;  // spheres: float4 {center.xyz, radius} per primitive
  // device: private traversal layout
  WideNode *d_wide = nullptr;
  PackedTri *d_tris = nullptr;
  PairNode *d_pair = nullptr;  // same indices and refs as d_wide
  TriCM *d_tris_cm = nullptr;  // same slots as d_tris
  // camera-relative copies of d_pair / d_tris_cm (every plane and vertex minus the camera origin rel_origin, bit
  // patterns of three floats), read by the AO pass's camera launch; derived on the pass's stream when the origin changes
  PairNode *d_pair_rel = nullptr;
  TriCM *d_tris_rel = nullptr;
  bool rel_valid = false;
  uint32_t rel_origin[3] = {0, 0, 0};
  // unit geometric normal per primitive (float4, w unused), read by the AO spawn; derived on the first AO pass
  float4 *d_face_n = nullptr;
  // recorded after the last launch of every AO pass, path pass and path bounce; the next one waits on it (any stream),
  // so that the pass scratch (d_wave, d_counters[2..6] and [48..54]) and the camera-relative copies are never
  // rewritten while a pass still reads them
  cudaEvent_t pass_done = nullptr;
  HostMirror<Node40> mirror;
  BuildOptions28 options;
  BuildStats16 stats;
  float root_bmin[3], root_bmax[3];
  // nrt_traverse's chunked copies; its first stream is also the stream every build / layout kernel of the accel runs on
  StagingPipeline staging;
  // orders AO passes, path passes, path bounces and the counting scratch d_counters[64..79]
  std::mutex host_mu;
  // nrt_traverse of <= 64 rays (e.g. the facade's one-ray Traverse).  Slot i launches with the ray cursor
  // d_counters[kSmallCursor0 + i]: a slot is held until its launch has finished, so its cursor is never shared.
  static constexpr int kSmallSlots = 16;
  static constexpr int kSmallCursor0 = 80;
  static_assert(kSmallCursor0 + kSmallSlots <= 96, "small-slot cursors lie inside d_counters");
  SmallCallPool<kSmallSlots, sizeof(Ray36), sizeof(Hit16)> small;
  // wavefront pass scratch (render.cu)
  void *d_wave = nullptr;
  size_t wave_bytes = 0;
  // device counter block (96 words): [0..7] misc, [8..9] visit counts, [16..47] ring of ray cursors, [48..54] path
  // tracer, [64..79] count / lane-stat scratch, [80..95] the small slots' ray cursors
  uint64_t *d_counters = nullptr;
  // persistent traversal launches take the ray cursor d_counters[16 + k] of the ring's slot k
  mutable LaunchRing<32> ring;
};

// The regions of Accel::d_counters the passes keep their counters in (pass scratch, like d_wave)
constexpr int kWaveCounters = 2;   // [2, 4): a wave's or a compaction's counters
constexpr int kPassTotals = 4;     // [4, 7): the AO passes' totals
constexpr int kPathCounters = 48;  // [48, 52): the path queues' counters
constexpr int kPathTotals = 52;    // [52, 55): the path tracers' totals
inline unsigned long long *pass_counters(const Accel *a, int region) {
  return reinterpret_cast<unsigned long long *>(a->d_counters) + region;
}

// Passes on one accel (AO passes, path passes, path bounces) share its pass scratch.  Under host_mu, a pass calls
// wait_previous_pass before it enqueues anything and holds a RecordOnExit for as long as it enqueues, so that every
// pass runs on the device after the one enqueued before it, whatever streams the two are on.
inline int wait_previous_pass(Accel *a, cudaStream_t s) {
  if (!a->pass_done) NRT_CUDA(cudaEventCreateWithFlags(&a->pass_done, cudaEventDisableTiming));
  NRT_CUDA(cudaStreamWaitEvent(s, a->pass_done, 0));
  return NRT_OK;
}
struct RecordOnExit {
  cudaEvent_t e;
  cudaStream_t s;
  ~RecordOnExit() { cudaEventRecord(e, s); }
};
// render.cu: derives Accel::d_face_n on `s` the first time a pass needs it (call under host_mu, inside the pass)
int ensure_face_normals(Accel *a, cudaStream_t s);
// the pass scratch grows only after the pass that last used it has finished
inline int grow_wave(Accel *a, size_t need) {
  if (a->wave_bytes >= need) return NRT_OK;
  NRT_CUDA(cudaEventSynchronize(a->pass_done));
  cudaFree(a->d_wave);
  a->d_wave = nullptr;
  a->wave_bytes = 0;
  NRT_CUDA(cudaMalloc(&a->d_wave, need));
  a->wave_bytes = need;
  return NRT_OK;
}

__host__ __device__ inline TraceOptions16 default_trace_options() {
  TraceOptions16 o;
  o.prim_ids_range[0] = 0;
  o.prim_ids_range[1] = 0x7FFFFFFFu;
  o.skip_prim_id = 0xFFFFFFFFu;
  o.cull_back_face = 0;
  o.pad[0] = o.pad[1] = o.pad[2] = 0;
  return o;
}

inline BuildOptions28 default_build_options() {
  BuildOptions28 o;
  o.cost_t_aabb = 0.2f;
  o.min_leaf_primitives = 4;
  o.max_tree_depth = 256;
  o.bin_size = 64;
  o.shallow_depth = 4;
  o.min_primitives_for_parallel_build = 8192;
  o.cache_bbox = 0;
  o.pad[0] = o.pad[1] = o.pad[2] = 0;
  return o;
}

// ---- kernels / stages implemented in the other translation units -------------------
// traverse.cu
// `cursor`: the persistent kernel's ray cursor (a device word, zeroed on `s` before the launch); nullptr takes the
// next one of the accel's ring
int launch_traverse(const Accel *a, const Ray36 *d_rays, size_t n, Hit16 *d_hits, uint8_t *d_mask,
                    const TraceOptions16 &opt, uint32_t flags, cudaStream_t s, unsigned long long *cursor = nullptr);
int launch_traverse_count(const Accel *a, const Ray36 *d_rays, size_t n, const TraceOptions16 &opt,
                          uint32_t flags, uint64_t *d_counts2, cudaStream_t s);
// SoA wavefront entry used by render.cu: rays as two float4 (org.xyz,min_t | dir.xyz,max_t)
int launch_traverse_soa(const Accel *a, const float4 *d_org_tmin, const float4 *d_dir_tmax, size_t n,
                        Hit16 *d_hits, const TraceOptions16 &opt, uint32_t flags, cudaStream_t s);
// layout.cu
int derive_private_layout(Accel *a, cudaStream_t s);
// (re)derives d_pair_rel / d_tris_rel on `s` unless they already hold this origin; the caller orders `s` after every
// launch that may still read the previous copies
int camera_relative_layout(Accel *a, const float cam[3], cudaStream_t s);
// build.cu
int build_on_device(Accel *a, cudaStream_t s);
// build_ref.cu: the reference-exact builder of BVHAccel<T>, T = float or double.  Inputs on the device: packed T
// vertices + faces, or (T = float only) d_boxes, 6 floats per box primitive.  cpp11_order: emit the node order of the
// C++11 parallel build when n > min_primitives_for_parallel_build.  On success *d_nodes_out (2n+2 capacity) and
// *d_indices_out (n) are device arrays the caller owns.
template <typename T>
int build_reference_tree(const T *d_verts, const uint32_t *d_faces, const float *d_boxes, uint32_t n,
                         uint32_t bin_size, uint32_t min_leaf_primitives, uint32_t max_tree_depth,
                         uint32_t shallow_depth, uint32_t min_primitives_for_parallel_build, bool cpp11_order,
                         BVHNodeOf<T> **d_nodes_out, uint32_t **d_indices_out, size_t *n_nodes_out,
                         BuildStats16 *stats_out, T root_bmin[3], T root_bmax[3], cudaStream_t s);
// the float builder over an accel's geometry (or its box primitives), writing its arrays, statistics and root box
int build_reference_tree_on_device(Accel *a, bool cpp11_order, cudaStream_t s);

// prims.cu
int launch_traverse_prims(const Accel *a, const Ray36 *d_rays, size_t n, Hit16 *d_hits, uint8_t *d_mask,
                          const TraceOptions16 &opt, uint32_t flags, cudaStream_t s);

int device_sm_count(int device);
// api.cu: structure check of a foreign nanort-layout tree (see there); fills the statistics
bool validate_foreign_tree(const Node40 *nodes, size_t n_nodes, const uint32_t *indices, size_t n_indices,
                           uint32_t n_prims, BuildStats16 *stats, std::string *why);
bool validate_foreign_tree64(const void *nodes_64B, size_t n_nodes, const uint32_t *indices, size_t n_indices,
                             uint32_t n_prims, BuildStats16 *stats, std::string *why);
// api.cu: makes the calling thread's selected device current (nrt_set_device); NRT_ERR_CUDA without a usable device
int select_device(int *device_out);
// api.cu: a new accel's device, counter block and staging streams (nrt_build, nrt_adopt, nrt_build_prims)
int common_init(Accel *a);
// api.cu: the vertex count a face array addresses (max index + 1), for callers that pass n_verts == 0
size_t infer_n_verts(const uint32_t *faces, uint32_t n_prims);

}  // namespace nrt
