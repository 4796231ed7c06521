// BVHAccel<double>: the fp64 instantiation of Build / Traverse (sm_90a, --fmad=false).
//
// Replaces (file:line in the reference tree):
//   BVHAccel<double>::Build              nanort.h:1892-2149   nrt_build_f64
//   BVHAccel<double>::Traverse           nanort.h:2487-2556   traverse_f64_kernel (reference_walk<double>)
//   IntersectRayAABB<double>             nanort.h:2327-2370   reference_walk<double> (trav_common.cuh)
//   TriangleIntersector<double>::Intersect / PrepareTraversal  nanort.h:1054-1201
//                                                             tri_test<double> / setup_ray<double> (trav_common.cuh)
//   vsafe_inverse<double>                nanort.h:414-465     safe_inverse<double>
//
// Build: fp64 adds nothing to the SHAPE of a good tree, so the topology comes from the production builder run over the
// float-rounded vertices; what must be double is every box the traversal tests, and those are refitted exactly from the
// double vertices (leaf: min/max of its triangles; branch: union of its children, bottom-up with one atomic arrival
// counter per branch).  The result is a BVHNode<double> array in the reference's layout and order conventions.
// Traverse: one thread per ray in the reference's visiting order, all arithmetic in double with every operation
// individually rounded, so t / u / v equal the reference's bits for the reported primitive.
#include <float.h>
#include <math_constants.h>

#include <algorithm>
#include <cstring>
#include <new>
#include <vector>

#include "common.cuh"
#include "scan.cuh"
#include "trav_common.cuh"

namespace nrt {
namespace {

struct Ray72 {
  double org[3], dir[3], min_t, max_t;
  uint32_t type, pad;
};
static_assert(sizeof(Ray72) == 72, "Ray<double> layout");
struct Hit32 {
  double u, v, t;
  uint32_t prim_id, pad;
};
static_assert(sizeof(Hit32) == 32, "TriangleIntersection<double> layout");
struct BuildOptions32 {
  double cost_t_aabb;
  uint32_t min_leaf_primitives, max_tree_depth, bin_size, shallow_depth, min_primitives_for_parallel_build;
  uint8_t cache_bbox, pad[3];
};
static_assert(sizeof(BuildOptions32) == 32, "BVHBuildOptions<double> layout");

struct AccelF64 {
  int device = 0;
  uint32_t n_prims = 0;
  size_t n_nodes = 0, n_verts = 0;
  Node64 *d_nodes = nullptr;
  uint32_t *d_indices = nullptr, *d_faces = nullptr;
  double *d_verts = nullptr;  // packed xyz
  BuildStats16 stats;
  double root_bmin[3], root_bmax[3];
  HostMirror<Node64> mirror;
  cudaStream_t stream = nullptr;  // build and layout kernels
  StagingPipeline staging;        // nrt_traverse_f64
  // fast-path layout (f64_fast.cuh), derived on the first fast Traverse; mu guards the derivation
  void *d_pair = nullptr, *d_tris_fast = nullptr;
  bool fast_ready = false;
  std::mutex mu;
  // persistent fast launches take the ray cursor d_cursor[k] of the ring's slot k
  static constexpr uint32_t kCursors = 8;
  unsigned long long *d_cursor = nullptr;
  LaunchRing<kCursors> ring;
  // nrt_traverse_f64 of <= 64 rays in the reference's order (the facade's one-ray Traverse)
  SmallCallPool<8, sizeof(Ray72), sizeof(Hit32)> small;
};

void destroy_f64(AccelF64 *a) {
  if (!a) return;
  DeviceGuard dg(a->device);
  cudaFree(a->d_nodes);
  cudaFree(a->d_indices);
  cudaFree(a->d_faces);
  cudaFree(a->d_verts);
  cudaFree(a->d_pair);
  cudaFree(a->d_tris_fast);
  cudaFree(a->d_cursor);
  if (a->stream) cudaStreamDestroy(a->stream);
  delete a;
}

// Packs the (strided) double vertices and uploads them and the faces on a new build stream a->stream (non-blocking,
// so the copies are stream-ordered with the kernels that consume them, see api.cu:upload_geometry).
int upload_geometry_f64(AccelF64 *a, const double *verts, size_t stride_bytes, const uint32_t *faces) {
  const size_t nv = a->n_verts;
  std::vector<double> packed(3 * nv);
  for (size_t i = 0; i < nv; i++) {
    const double *p = reinterpret_cast<const double *>(reinterpret_cast<const char *>(verts) + i * stride_bytes);
    packed[3 * i] = p[0], packed[3 * i + 1] = p[1], packed[3 * i + 2] = p[2];
  }
  NRT_CUDA(cudaStreamCreateWithFlags(&a->stream, cudaStreamNonBlocking));
  NRT_CUDA(cudaMalloc(&a->d_verts, sizeof(double) * 3 * nv));
  NRT_CUDA(cudaMalloc(&a->d_faces, sizeof(uint32_t) * 3 * (size_t)a->n_prims));
  NRT_CUDA(cudaMemcpyAsync(a->d_verts, packed.data(), sizeof(double) * 3 * nv, cudaMemcpyHostToDevice, a->stream));
  NRT_CUDA(cudaMemcpyAsync(a->d_faces, faces, sizeof(uint32_t) * 3 * (size_t)a->n_prims, cudaMemcpyHostToDevice, a->stream));
  NRT_CUDA(cudaStreamSynchronize(a->stream));
  return NRT_OK;
}

// ---- build ---------------------------------------------------------------------------------------------------
__global__ void f64_round_kernel(const double *__restrict__ v, size_t n, float *__restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (float)v[i];
}

constexpr uint32_t kNoParent = 0xFFFFFFFFu;

__global__ void f64_parent_kernel(const Node40 *__restrict__ nodes, uint32_t n, uint32_t *__restrict__ parent) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (i == 0) parent[0] = kNoParent;
  const Node40 nd = nodes[i];
  if (nd.flag == 0) {
    parent[nd.data[0]] = i;
    parent[nd.data[1]] = i;
  }
}

// one thread per node; leaves compute their exact double box and climb: the second child to arrive at a branch
// merges both child boxes (the first one leaves), so every branch is written once, after both children
__global__ void f64_refit_kernel(const Node40 *__restrict__ nodes, uint32_t n, const uint32_t *__restrict__ parent,
                                 const uint32_t *__restrict__ indices, const uint32_t *__restrict__ faces,
                                 const double *__restrict__ verts, uint32_t *__restrict__ arrived,
                                 Node64 *__restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Node40 nd = nodes[i];
  Node64 o;
  o.flag = nd.flag;
  o.axis = nd.axis;
  o.data[0] = nd.data[0];
  o.data[1] = nd.data[1];
  if (nd.flag == 0) {  // topology fields now, box by whichever child arrives second
    volatile int32_t *w = reinterpret_cast<volatile int32_t *>(&out[i].flag);
    w[0] = o.flag;
    w[1] = o.axis;
    w[2] = (int32_t)o.data[0];
    w[3] = (int32_t)o.data[1];
    return;
  }
  double lo[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, hi[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
  for (uint32_t k = 0; k < nd.data[0]; k++) {
    const uint32_t prim = indices[nd.data[1] + k];
    for (int c = 0; c < 3; c++) {
      const double *p = verts + 3 * (size_t)faces[3 * (size_t)prim + c];
      for (int a = 0; a < 3; a++) {
        lo[a] = fmin(lo[a], p[a]);
        hi[a] = fmax(hi[a], p[a]);
      }
    }
  }
  for (int a = 0; a < 3; a++) {
    o.bmin[a] = lo[a];
    o.bmax[a] = hi[a];
  }
  out[i] = o;
  uint32_t cur = i;
  for (;;) {
    const uint32_t p = parent[cur];
    if (p == kNoParent) break;
    __threadfence();
    if (atomicAdd(arrived + p, 1u) == 0u) break;  // the sibling subtree is not finished yet
    __threadfence();
    const Node40 pn = nodes[p];
    const volatile double *a = reinterpret_cast<const volatile double *>(out + pn.data[0]);
    const volatile double *b = reinterpret_cast<const volatile double *>(out + pn.data[1]);
    volatile double *d = reinterpret_cast<volatile double *>(out + p);
    for (int k = 0; k < 3; k++) {
      d[k] = fmin(a[k], b[k]);
      d[3 + k] = fmax(a[3 + k], b[3 + k]);
    }
    cur = p;
  }
}

// ---- traversal -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
    traverse_f64_kernel(const Node64 *__restrict__ nodes, const uint32_t *__restrict__ indices,
                        const uint32_t *__restrict__ faces, const double *__restrict__ verts,
                        const Ray72 *__restrict__ rays, size_t n, Hit32 *__restrict__ hits, uint8_t *__restrict__ mask,
                        TraceOptions16 opt, uint32_t flags) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Ray72 r = rays[i];
  RayCtxT<double> c;
  setup_ray(c, r.org[0], r.org[1], r.org[2], r.dir[0], r.dir[1], r.dir[2], r.min_t,
            (flags & NRT_TRAVERSE_CPP03_INVERSE) != 0);
  BestT<double> best;
  best.t = r.max_t;
  best.u = 0.0;
  best.v = 0.0;
  best.prim = 0xFFFFFFFFu;
  // leaf: indices_ -> faces -> double vertices (nanort.h:2394, 1065-1071)
  reference_walk(nodes, c, r.min_t, r.max_t, [&](uint32_t first, uint32_t count, double &hit_t) {
    bool any = false;
    for (uint32_t k = 0; k < count; k++) {
      const uint32_t prim = __ldg(indices + first + k);
      double3 v[3];
      for (int q = 0; q < 3; q++) {
        const double *p = verts + 3 * (size_t)__ldg(faces + 3 * (size_t)prim + q);
        v[q] = make_double3(__ldg(p), __ldg(p + 1), __ldg(p + 2));
      }
      if (tri_test(c, opt, prim, v[0], v[1], v[2], best)) any = true;
    }
    if (any) hit_t = best.t;
  });
  const bool hit = best.t < r.max_t;
  Hit32 h;
  h.u = hit ? best.u : 0.0;
  h.v = hit ? best.v : 0.0;
  h.t = hit ? best.t : r.max_t;
  h.prim_id = hit ? best.prim : 0xFFFFFFFFu;
  h.pad = 0;
  hits[i] = h;
  if (mask) mask[i] = hit ? 1 : 0;
}

#include "f64_fast.cuh"

// PairNodeD / TriD arrays of the fast kernel from the BVHNode<double> array, indices_, faces and double vertices the
// accel already holds on the device, on the first call.
int derive_fast_layout_f64(AccelF64 *a) {
  std::lock_guard<std::mutex> lock(a->mu);
  if (a->fast_ready) return NRT_OK;
  const uint32_t nn = (uint32_t)a->n_nodes;
  uint32_t *d_flags = nullptr, *d_widx = nullptr;
  uint32_t n_branch = 0;
  int rc = NRT_OK;
  cudaStream_t s = a->stream;
  cudaError_t e = cudaMalloc(&d_flags, sizeof(uint32_t) * (size_t)nn);
  if (e == cudaSuccess) e = cudaMalloc(&d_widx, sizeof(uint32_t) * (size_t)nn);
  if (e == cudaSuccess) {
    branch_flags_kernel<<<(nn + 255) / 256, 256, 0, s>>>(a->d_nodes, nn, d_flags);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) rc = exclusive_scan_u32(d_flags, d_widx, nn, &n_branch, s);
  const size_t n_pair = n_branch > 0 ? n_branch : 1;
  if (e == cudaSuccess && rc == NRT_OK) e = cudaMalloc(&a->d_pair, sizeof(PairNodeD) * n_pair);
  if (e == cudaSuccess && rc == NRT_OK) e = cudaMalloc(&a->d_tris_fast, sizeof(TriD) * (size_t)a->n_prims);
  if (e == cudaSuccess && rc == NRT_OK && !a->d_cursor)
    e = cudaMalloc(&a->d_cursor, sizeof(unsigned long long) * AccelF64::kCursors);
  if (e == cudaSuccess && rc == NRT_OK) {
    f64_tris_kernel<<<(a->n_prims + 255) / 256, 256, 0, s>>>(a->d_indices, a->d_faces, a->d_verts, a->n_prims,
                                                            static_cast<TriD *>(a->d_tris_fast));
    f64_pair_kernel<<<(nn + 255) / 256, 256, 0, s>>>(a->d_nodes, nn, d_widx, static_cast<PairNodeD *>(a->d_pair),
                                                    static_cast<TriD *>(a->d_tris_fast));
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  cudaFree(d_flags);
  cudaFree(d_widx);
  if (e != cudaSuccess || rc != NRT_OK) {
    cudaFree(a->d_pair);
    cudaFree(a->d_tris_fast);
    a->d_pair = a->d_tris_fast = nullptr;
    return e != cudaSuccess ? cuda_fail(e, "derive_fast_layout_f64", __FILE__, __LINE__) : rc;
  }
  a->fast_ready = true;
  return NRT_OK;
}

// One launch over m rays on `s`: the reference-order walk, or the fast kernel (its layout derived beforehand) with the
// ray cursor of the next slot of the accel's ring.
int launch_f64(AccelF64 *a, const Ray72 *d_rays, size_t m, Hit32 *d_hits, uint8_t *d_mask, const TraceOptions16 &opt,
               uint32_t flags, cudaStream_t s) {
  if (flags & NRT_TRAVERSE_CONFORMANCE) {
    traverse_f64_kernel<<<(unsigned)((m + 127) / 128), 128, 0, s>>>(a->d_nodes, a->d_indices, a->d_faces, a->d_verts,
                                                                     d_rays, m, d_hits, d_mask, opt, flags);
    NRT_CUDA(cudaGetLastError());
    return NRT_OK;
  }
  size_t grid = (size_t)device_sm_count(a->device) * kFastBlocksPerSmD;  // persistent: every SM holds its complement
  const size_t need = ((m + 31) / 32 + kFastBlockD / 32 - 1) / (kFastBlockD / 32);
  if (grid > need) grid = need;
  if (grid == 0) grid = 1;
  const bool deep = a->stats.max_tree_depth + 2 > 64u;  // adopted reference trees reach depth 256
  const PairNodeD *pair = static_cast<const PairNodeD *>(a->d_pair);
  const TriD *tris = static_cast<const TriD *>(a->d_tris_fast);
  return a->ring.run(s, [&](uint32_t k) {
    unsigned long long *cursor = a->d_cursor + k;
    NRT_CUDA(cudaMemsetAsync(cursor, 0, sizeof(unsigned long long), s));
    if (deep)
      traverse_fast_f64_kernel<512><<<(unsigned)grid, kFastBlockD, 0, s>>>(pair, tris, d_rays, m, d_hits, d_mask, opt, flags,
                                                                          cursor);
    else
      traverse_fast_f64_kernel<64><<<(unsigned)grid, kFastBlockD, 0, s>>>(pair, tris, d_rays, m, d_hits, d_mask, opt, flags,
                                                                         cursor);
    NRT_CUDA(cudaGetLastError());
    return NRT_OK;
  });
}

}  // namespace
}  // namespace nrt

using namespace nrt;

#define F64_CUDA(expr)                                           \
  do {                                                           \
    cudaError_t _e = (expr);                                     \
    if (_e != cudaSuccess) {                                     \
      rc = cuda_fail(_e, #expr, __FILE__, __LINE__);             \
      goto fail;                                                 \
    }                                                            \
  } while (0)

extern "C" {

int nrt_build_f64(const double *verts, size_t stride_bytes, size_t n_verts, const uint32_t *faces, uint32_t n_prims,
                  const void *build_opts_32B, nrt_accel_f64 **out) {
  return nrt_build_f64_ex(verts, stride_bytes, n_verts, faces, n_prims, build_opts_32B, NRT_BUILD_FAST, out);
}

int nrt_build_f64_ex(const double *verts, size_t stride_bytes, size_t n_verts, const uint32_t *faces, uint32_t n_prims,
                     const void *build_opts_32B, uint32_t flags, nrt_accel_f64 **out) {
  if (!out) {
    set_error("nrt_build_f64: out is NULL");
    return NRT_ERR_INVALID;
  }
  *out = nullptr;
  if (n_prims == 0) {  // Build returns false (nanort.h:1907-1909)
    set_error("nrt_build_f64: num_primitives == 0");
    return NRT_ERR_INVALID;
  }
  if (!verts || !faces || stride_bytes < 24) {
    set_error("nrt_build_f64: bad geometry pointers / stride");
    return NRT_ERR_INVALID;
  }
  BuildOptions32 o64;
  {
    const BuildOptions28 d = default_build_options();
    o64.cost_t_aabb = d.cost_t_aabb;
    o64.min_leaf_primitives = d.min_leaf_primitives;
    o64.max_tree_depth = d.max_tree_depth;
    o64.bin_size = d.bin_size;
    o64.shallow_depth = d.shallow_depth;
    o64.min_primitives_for_parallel_build = d.min_primitives_for_parallel_build;
    o64.cache_bbox = 0;
    o64.pad[0] = o64.pad[1] = o64.pad[2] = 0;
  }
  if (build_opts_32B) memcpy(&o64, build_opts_32B, sizeof(o64));
  if (o64.bin_size < 2 || o64.max_tree_depth > 500) {
    set_error("nrt_build_f64: bin_size must be > 1 and max_tree_depth <= 500");
    return NRT_ERR_INVALID;
  }
  int device = 0;
  DeviceGuard dg_caller;  // select_device makes the chosen device current; the caller gets its own back
  int rc = select_device(&device);
  if (rc != NRT_OK) return rc;
  if (n_verts == 0) n_verts = infer_n_verts(faces, n_prims);
  AccelF64 *a = new (std::nothrow) AccelF64();
  Accel *t = new (std::nothrow) Accel();  // float topology, discarded after the refit
  uint32_t *d_parent = nullptr, *d_arrived = nullptr;
  if (!a || !t) {
    delete a;
    delete t;
    return NRT_ERR_NOMEM;
  }
  a->device = t->device = device;
  a->n_prims = t->n_prims = n_prims;
  a->n_verts = t->n_verts = n_verts;
  rc = upload_geometry_f64(a, verts, stride_bytes, faces);
  if (rc != NRT_OK) goto fail;
  if (flags & NRT_BUILD_REFERENCE_TREE) {
    // conformance build: the reference's own BVHNode<double> array and indices_, bit for bit (build_ref.cu)
    rc = build_reference_tree<double>(a->d_verts, a->d_faces, nullptr, n_prims, o64.bin_size, o64.min_leaf_primitives,
                                      o64.max_tree_depth, o64.shallow_depth, o64.min_primitives_for_parallel_build,
                                      (flags & NRT_BUILD_REFERENCE_CPP03_ORDER) == 0, &a->d_nodes, &a->d_indices,
                                      &a->n_nodes, &a->stats, a->root_bmin, a->root_bmax, a->stream);
    if (rc != NRT_OK) goto fail;
    delete t;
    *out = reinterpret_cast<nrt_accel_f64 *>(a);
    return NRT_OK;
  }
  t->d_faces = a->d_faces;  // shared, freed with `a`
  t->options = default_build_options();
  t->options.cost_t_aabb = (float)o64.cost_t_aabb;
  t->options.min_leaf_primitives = o64.min_leaf_primitives;
  t->options.max_tree_depth = o64.max_tree_depth;
  t->options.bin_size = o64.bin_size;
  t->options.shallow_depth = o64.shallow_depth;
  t->options.min_primitives_for_parallel_build = o64.min_primitives_for_parallel_build;
  F64_CUDA(cudaMalloc(&t->d_verts, sizeof(float) * 3 * n_verts));
  f64_round_kernel<<<(unsigned)((3 * n_verts + 255) / 256), 256, 0, a->stream>>>(a->d_verts, 3 * n_verts, t->d_verts);
  F64_CUDA(cudaGetLastError());
  rc = build_on_device(t, a->stream);
  if (rc != NRT_OK) goto fail;
  {
    const uint32_t nn = (uint32_t)t->n_nodes;
    a->n_nodes = nn;
    F64_CUDA(cudaMalloc(&a->d_nodes, sizeof(Node64) * (size_t)nn));
    F64_CUDA(cudaMalloc(&d_parent, sizeof(uint32_t) * (size_t)nn));
    F64_CUDA(cudaMalloc(&d_arrived, sizeof(uint32_t) * (size_t)nn));
    F64_CUDA(cudaMemsetAsync(d_arrived, 0, sizeof(uint32_t) * (size_t)nn, a->stream));
    f64_parent_kernel<<<(nn + 255) / 256, 256, 0, a->stream>>>(t->d_nodes, nn, d_parent);
    f64_refit_kernel<<<(nn + 127) / 128, 128, 0, a->stream>>>(t->d_nodes, nn, d_parent, t->d_indices, a->d_faces,
                                                              a->d_verts, d_arrived, a->d_nodes);
    F64_CUDA(cudaGetLastError());
    Node64 root;
    F64_CUDA(cudaMemcpyAsync(&root, a->d_nodes, sizeof(Node64), cudaMemcpyDeviceToHost, a->stream));
    F64_CUDA(cudaStreamSynchronize(a->stream));
    for (int k = 0; k < 3; k++) {
      a->root_bmin[k] = root.bmin[k];
      a->root_bmax[k] = root.bmax[k];
    }
  }
  a->d_indices = t->d_indices;
  t->d_indices = nullptr;
  a->stats = t->stats;
  cudaFree(d_parent);
  cudaFree(d_arrived);
  cudaFree(t->d_nodes);
  cudaFree(t->d_verts);
  delete t;
  *out = reinterpret_cast<nrt_accel_f64 *>(a);
  return NRT_OK;
fail:
  cudaFree(d_parent);
  cudaFree(d_arrived);
  cudaFree(t->d_nodes);
  cudaFree(t->d_indices);
  cudaFree(t->d_verts);
  delete t;
  destroy_f64(a);
  return rc;
}

int nrt_adopt_f64(const void *nodes_64B, size_t n_nodes, const uint32_t *indices, size_t n_indices, const double *verts,
                  size_t stride_bytes, size_t n_verts, const uint32_t *faces, uint32_t n_prims, nrt_accel_f64 **out) {
  if (!out) {
    set_error("nrt_adopt_f64: out is NULL");
    return NRT_ERR_INVALID;
  }
  *out = nullptr;
  if (!nodes_64B || !indices || !verts || !faces || n_nodes == 0 || n_prims == 0 || n_indices != n_prims ||
      stride_bytes < 24) {
    set_error("nrt_adopt_f64: bad arguments");
    return NRT_ERR_INVALID;
  }
  const Node64 *hn = static_cast<const Node64 *>(nodes_64B);
  BuildStats16 st = {0, 0, 0, 0.0f};
  {  // an adopted tree is foreign data: the same structure check as nrt_adopt (api.cu:validate_foreign_tree)
    std::string why;
    if (!validate_foreign_tree64(nodes_64B, n_nodes, indices, n_indices, n_prims, &st, &why)) {
      set_error("nrt_adopt_f64: " + why);
      return NRT_ERR_INVALID;
    }
  }
  int device = 0;
  DeviceGuard dg_caller;  // select_device makes the chosen device current; the caller gets its own back
  int rc = select_device(&device);
  if (rc != NRT_OK) return rc;
  if (n_verts == 0) n_verts = infer_n_verts(faces, n_prims);
  AccelF64 *a = new (std::nothrow) AccelF64();
  if (!a) return NRT_ERR_NOMEM;
  a->device = device;
  a->n_prims = n_prims;
  a->n_verts = n_verts;
  a->n_nodes = n_nodes;
  a->stats = st;
  rc = upload_geometry_f64(a, verts, stride_bytes, faces);
  if (rc == NRT_OK) {
    cudaError_t e = cudaMalloc(&a->d_nodes, sizeof(Node64) * n_nodes);
    if (e == cudaSuccess) e = cudaMalloc(&a->d_indices, sizeof(uint32_t) * n_indices);
    if (e == cudaSuccess) e = cudaMemcpyAsync(a->d_nodes, hn, sizeof(Node64) * n_nodes, cudaMemcpyHostToDevice, a->stream);
    if (e == cudaSuccess)
      e = cudaMemcpyAsync(a->d_indices, indices, sizeof(uint32_t) * n_indices, cudaMemcpyHostToDevice, a->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(a->stream);
    if (e != cudaSuccess) rc = cuda_fail(e, "nrt_adopt_f64 upload", __FILE__, __LINE__);
  }
  if (rc != NRT_OK) {
    destroy_f64(a);
    return rc;
  }
  for (int k = 0; k < 3; k++) {
    a->root_bmin[k] = hn[0].bmin[k];
    a->root_bmax[k] = hn[0].bmax[k];
  }
  a->mirror.assign(hn, n_nodes, indices, n_indices);
  *out = reinterpret_cast<nrt_accel_f64 *>(a);
  return NRT_OK;
}

void nrt_free_f64(nrt_accel_f64 *a) { destroy_f64(reinterpret_cast<AccelF64 *>(a)); }

int nrt_stats_f64(const nrt_accel_f64 *h, void *stats_16B) {
  if (!h || !stats_16B) {
    set_error("nrt_stats_f64: NULL argument");
    return NRT_ERR_INVALID;
  }
  memcpy(stats_16B, &reinterpret_cast<const AccelF64 *>(h)->stats, sizeof(BuildStats16));
  return NRT_OK;
}

int nrt_bounding_box_f64(const nrt_accel_f64 *h, double bmin[3], double bmax[3]) {
  if (!h || !bmin || !bmax) {
    set_error("nrt_bounding_box_f64: NULL argument");
    return NRT_ERR_INVALID;
  }
  const AccelF64 *a = reinterpret_cast<const AccelF64 *>(h);
  for (int k = 0; k < 3; k++) {
    bmin[k] = a->root_bmin[k];
    bmax[k] = a->root_bmax[k];
  }
  return NRT_OK;
}

int nrt_nodes_f64(nrt_accel_f64 *h, const void **nodes_64B, size_t *n_nodes, const uint32_t **indices,
                  size_t *n_indices) {
  if (!h) {
    set_error("nrt_nodes_f64: NULL accel");
    return NRT_ERR_INVALID;
  }
  AccelF64 *a = reinterpret_cast<AccelF64 *>(h);
  return a->mirror.get(a->device, a->d_nodes, a->n_nodes, a->d_indices, a->n_prims, nodes_64B, n_nodes, indices,
                       n_indices);
}

int nrt_traverse_f64(const nrt_accel_f64 *h, const void *rays_72B, size_t n_rays, void *hits_32B, uint8_t *hit_mask,
                     const void *trace_opts_16B, uint32_t flags) {
  if (!h || (n_rays && (!rays_72B || !hits_32B))) {
    set_error("nrt_traverse_f64: NULL argument");
    return NRT_ERR_INVALID;
  }
  if (n_rays == 0) return NRT_OK;
  AccelF64 *a = const_cast<AccelF64 *>(reinterpret_cast<const AccelF64 *>(h));
  TraceOptions16 opt = default_trace_options();
  if (trace_opts_16B) memcpy(&opt, trace_opts_16B, sizeof(opt));
  NRT_DEVICE(a->device);
  if (n_rays <= decltype(a->small)::kMaxRays && (flags & NRT_TRAVERSE_CONFORMANCE)) {
    // low-latency path of the facade's per-ray Traverse
    return a->small.run(rays_72B, n_rays, sizeof(Ray72), hits_32B, hit_mask,
                        [&](int, void *h_rays, void *h_hits, uint8_t *h_mask, cudaStream_t s) {
                          traverse_f64_kernel<<<1, 64, 0, s>>>(a->d_nodes, a->d_indices, a->d_faces, a->d_verts,
                                                               static_cast<const Ray72 *>(h_rays), n_rays,
                                                               static_cast<Hit32 *>(h_hits), h_mask, opt, flags);
                          NRT_CUDA(cudaGetLastError());
                          return NRT_OK;
                        });
  }
  if (!(flags & NRT_TRAVERSE_CONFORMANCE)) {
    const int rc = derive_fast_layout_f64(a);
    if (rc != NRT_OK) return rc;
  }
  return a->staging.run(rays_72B, n_rays, sizeof(Ray72), hits_32B, sizeof(Hit32), hit_mask,
                        [&](const void *d_rays, size_t m, void *d_hits, uint8_t *d_mask, cudaStream_t s) {
                          return launch_f64(a, static_cast<const Ray72 *>(d_rays), m, static_cast<Hit32 *>(d_hits),
                                            d_mask, opt, flags, s);
                        });
}

// Any number of calls of one accel may be in flight on any streams (launch_f64 orders the ring's slots on the device).
int nrt_traverse_f64_device(const nrt_accel_f64 *h, const void *d_rays_72B, size_t n_rays, void *d_hits_32B,
                            uint8_t *d_hit_mask, const void *trace_opts_16B, uint32_t flags, void *stream) {
  if (!h || (n_rays && (!d_rays_72B || !d_hits_32B))) {
    set_error("nrt_traverse_f64_device: NULL argument");
    return NRT_ERR_INVALID;
  }
  if (n_rays == 0) return NRT_OK;
  AccelF64 *a = const_cast<AccelF64 *>(reinterpret_cast<const AccelF64 *>(h));
  TraceOptions16 opt = default_trace_options();
  if (trace_opts_16B) memcpy(&opt, trace_opts_16B, sizeof(opt));
  NRT_DEVICE(a->device);
  if (!(flags & NRT_TRAVERSE_CONFORMANCE)) {
    const int rc = derive_fast_layout_f64(a);
    if (rc != NRT_OK) return rc;
  }
  return launch_f64(a, static_cast<const Ray72 *>(d_rays_72B), n_rays, static_cast<Hit32 *>(d_hits_32B), d_hit_mask, opt,
                    flags, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
