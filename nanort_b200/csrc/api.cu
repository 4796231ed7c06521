// extern "C" boundary (include/nanort_b200.h): accel lifetime, host<->device plumbing.
#include <string.h>

#include <algorithm>
#include <new>

#include "common.cuh"

namespace nrt {

static thread_local std::string g_err;
static thread_local int g_device = 0;

void set_error(const std::string &msg) { g_err = msg; }

int cuda_fail(cudaError_t e, const char *what, const char *file, int line) {
  g_err = std::string("CUDA error: ") + cudaGetErrorString(e) + " in " + what + " (" + file + ":" +
          std::to_string(line) + ")";
  cudaGetLastError();  // clear sticky-less errors
  return e == cudaErrorMemoryAllocation ? NRT_ERR_NOMEM : NRT_ERR_CUDA;
}

int select_device(int *device_out) {
  if (device_out) *device_out = g_device;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) {
    g_err = std::string("no usable CUDA device (") + (e != cudaSuccess ? cudaGetErrorString(e) : "count = 0") +
            "); nanort_b200 has no CPU fallback";
    cudaGetLastError();
    return NRT_ERR_CUDA;
  }
  if (g_device >= n) {
    g_err = "nrt_set_device: device index out of range";
    return NRT_ERR_INVALID;
  }
  NRT_CUDA(cudaSetDevice(g_device));
  return NRT_OK;
}

static void destroy(Accel *a) {
  if (!a) return;
  DeviceGuard dg(a->device);
  cudaFree(a->d_nodes);
  cudaFree(a->d_indices);
  cudaFree(a->d_verts);
  cudaFree(a->d_faces);
  cudaFree(a->d_wide);
  cudaFree(a->d_tris);
  cudaFree(a->d_pair);
  cudaFree(a->d_tris_cm);
  cudaFree(a->d_pair_rel);
  cudaFree(a->d_tris_rel);
  cudaFree(a->d_face_n);
  if (a->pass_done) cudaEventDestroy(a->pass_done);
  cudaFree(a->d_prim_boxes);
  cudaFree(a->d_prim_data);
  cudaFree(a->d_wave);
  cudaFree(a->d_counters);
  delete a;
}

// Uploads geometry as tightly packed float3 vertices + faces.
// Stream-ordered on a->staging.stream(0), the (non-blocking) stream every build / layout kernel of this accel runs on: a
// synchronous cudaMemcpy from pageable memory on the NULL stream may return before its DMA has finished, and
// non-blocking streams do not order after the NULL stream.
static int upload_geometry(Accel *a, const float *verts, size_t stride, size_t n_verts, const uint32_t *faces,
                           uint32_t n_prims) {
  cudaStream_t s = a->staging.stream(0);
  if (n_verts == 0) n_verts = infer_n_verts(faces, n_prims);
  a->n_verts = n_verts;
  a->n_prims = n_prims;
  NRT_CUDA(cudaMalloc(&a->d_verts, sizeof(float) * 3 * n_verts));
  NRT_CUDA(cudaMalloc(&a->d_faces, sizeof(uint32_t) * 3 * (size_t)n_prims));
  if (stride == 12) {
    NRT_CUDA(cudaMemcpyAsync(a->d_verts, verts, sizeof(float) * 3 * n_verts, cudaMemcpyHostToDevice, s));
  } else {
    NRT_CUDA(cudaMemcpy2DAsync(a->d_verts, 12, verts, stride, 12, n_verts, cudaMemcpyHostToDevice, s));
  }
  NRT_CUDA(cudaMemcpyAsync(a->d_faces, faces, sizeof(uint32_t) * 3 * (size_t)n_prims, cudaMemcpyHostToDevice, s));
  NRT_CUDA(cudaStreamSynchronize(s));  // the caller's buffers are borrowed only for the duration of the call
  return NRT_OK;
}

}  // namespace nrt

// Structure check of a nanort-layout tree that did not come from our builders (nrt_adopt, BVHAccel::Load).  Accepts
// exactly what the reference's Build can emit and the kernels rely on:
//   * every node is reached exactly once from node 0 (a tree, not a DAG: a shared child would also make this walk
//     exponential), children lie behind their parent, axis in 0..2, flag in {0, 1};
//   * the non-empty leaves' ranges [first, first + count) partition [0, n_indices) exactly -- the private layout marks
//     the LAST triangle of a leaf, so overlapping leaves would end early at a foreign mark and skip primitives;
//   * indices address existing primitives; depth <= 500 (512-entry traversal stacks, kNANORT_MAX_STACK_DEPTH).
// Leaves with count == 0 are legal (min_leaf_primitives == 0 produces them); the layout gives them an inverted box.
template <class NodeT>
static bool validate_foreign_tree_t(const NodeT *hn, size_t n_nodes, const uint32_t *indices, size_t n_indices,
                                    uint32_t n_prims, nrt::BuildStats16 *stats, std::string *why) {
  *stats = nrt::BuildStats16{0, 0, 0, 0.0f};
  std::vector<uint8_t> seen(n_nodes, 0);
  std::vector<std::pair<uint32_t, uint32_t> > stack;  // (node, depth)
  std::vector<std::pair<uint32_t, uint32_t> > ranges;
  stack.push_back(std::make_pair(0u, 0u));
  seen[0] = 1;
  while (!stack.empty()) {
    const uint32_t i = stack.back().first, d = stack.back().second;
    stack.pop_back();
    const NodeT &nd = hn[i];
    stats->max_tree_depth = std::max(stats->max_tree_depth, d);
    if (d > 500) {
      *why = "tree deeper than 500 levels (512-entry traversal stack, as the reference's)";
      return false;
    }
    if (nd.flag == 0) {
      stats->num_branch_nodes++;
      const uint32_t c0 = nd.data[0], c1 = nd.data[1];
      if (c0 >= n_nodes || c1 >= n_nodes || c0 <= i || c1 <= i || c0 == c1 || nd.axis < 0 || nd.axis > 2) {
        *why = "branch node with invalid children / axis";
        return false;
      }
      if (seen[c0] || seen[c1]) {
        *why = "node reachable twice (the array is not a tree)";
        return false;
      }
      seen[c0] = seen[c1] = 1;
      stack.push_back(std::make_pair(c0, d + 1));
      stack.push_back(std::make_pair(c1, d + 1));
    } else if (nd.flag == 1) {
      stats->num_leaf_nodes++;
      if ((size_t)nd.data[1] + nd.data[0] > n_indices) {
        *why = "leaf range outside indices";
        return false;
      }
      if (nd.data[0] > 0) ranges.push_back(std::make_pair(nd.data[1], nd.data[0]));
    } else {
      *why = "node flag is neither 0 (branch) nor 1 (leaf)";
      return false;
    }
  }
  std::sort(ranges.begin(), ranges.end());
  size_t next = 0;
  for (size_t k = 0; k < ranges.size(); k++) {
    if (ranges[k].first != next) {
      *why = "leaf ranges do not partition indices (gap or overlap)";
      return false;
    }
    next += ranges[k].second;
  }
  if (next != n_indices) {
    *why = "leaf ranges do not cover indices";
    return false;
  }
  for (size_t i = 0; i < n_indices; i++) {
    if (indices[i] >= n_prims) {
      *why = "index outside primitives";
      return false;
    }
  }
  return true;
}

namespace nrt {
bool validate_foreign_tree(const Node40 *hn, size_t n_nodes, const uint32_t *indices, size_t n_indices,
                           uint32_t n_prims, BuildStats16 *stats, std::string *why) {
  return validate_foreign_tree_t(hn, n_nodes, indices, n_indices, n_prims, stats, why);
}
bool validate_foreign_tree64(const void *nodes_64B, size_t n_nodes, const uint32_t *indices, size_t n_indices,
                             uint32_t n_prims, BuildStats16 *stats, std::string *why) {
  return validate_foreign_tree_t(static_cast<const Node64 *>(nodes_64B), n_nodes, indices, n_indices, n_prims, stats, why);
}

size_t infer_n_verts(const uint32_t *faces, uint32_t n_prims) {
  uint32_t m = 0;
  for (size_t i = 0; i < (size_t)n_prims * 3; i++) m = std::max(m, faces[i]);
  return (size_t)m + 1;
}

int common_init(Accel *a) {
  a->device = g_device;
  NRT_CUDA(cudaMalloc(&a->d_counters, 96 * sizeof(uint64_t)));
  NRT_CUDA(cudaMemset(a->d_counters, 0, 96 * sizeof(uint64_t)));
  return a->staging.create_streams();
}

}  // namespace nrt

using namespace nrt;

extern "C" {

const char *nrt_last_error(void) { return g_err.c_str(); }

int nrt_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

int nrt_set_device(int device) {
  if (device < 0) {
    g_err = "nrt_set_device: negative device";
    return NRT_ERR_INVALID;
  }
  g_device = device;
  return NRT_OK;
}

int nrt_build(const float *verts, size_t stride_bytes, size_t n_verts, const uint32_t *faces, uint32_t n_prims,
              const void *build_opts_28B, nrt_accel **out) {
  return nrt_build_ex(verts, stride_bytes, n_verts, faces, n_prims, build_opts_28B, NRT_BUILD_FAST, out);
}

int nrt_build_ex(const float *verts, size_t stride_bytes, size_t n_verts, const uint32_t *faces, uint32_t n_prims,
                 const void *build_opts_28B, uint32_t flags, nrt_accel **out) {
  if (!out) {
    g_err = "nrt_build: out is NULL";
    return NRT_ERR_INVALID;
  }
  *out = nullptr;
  if (n_prims == 0) {  // reference: Build returns false (nanort.h:1907-1909)
    g_err = "nrt_build: num_primitives == 0";
    return NRT_ERR_INVALID;
  }
  if (!verts || !faces || stride_bytes < 12) {
    g_err = "nrt_build: bad geometry pointers / stride";
    return NRT_ERR_INVALID;
  }
  DeviceGuard dg_caller;  // select_device makes the chosen device current; the caller gets its own back
  int rc = select_device(nullptr);
  if (rc != NRT_OK) return rc;
  Accel *a = new (std::nothrow) Accel();
  if (!a) return NRT_ERR_NOMEM;
  a->options = default_build_options();
  if (build_opts_28B) memcpy(&a->options, build_opts_28B, sizeof(BuildOptions28));
  if (a->options.bin_size < 2) {  // reference asserts bin_size > 1 (nanort.h:1905)
    g_err = "nrt_build: bin_size must be > 1";
    delete a;
    return NRT_ERR_INVALID;
  }
  if (a->options.max_tree_depth > 500) {
    // the traversal stacks hold 512 entries, like the reference's kNANORT_MAX_STACK_DEPTH (nanort.h:63, 2497)
    g_err = "nrt_build: max_tree_depth > 500 is not supported (512-entry traversal stack)";
    delete a;
    return NRT_ERR_INVALID;
  }
  rc = common_init(a);
  if (rc == NRT_OK) rc = upload_geometry(a, verts, stride_bytes, n_verts, faces, n_prims);
  if (rc == NRT_OK) {
    rc = (flags & NRT_BUILD_REFERENCE_TREE)
             ? build_reference_tree_on_device(a, !(flags & NRT_BUILD_REFERENCE_CPP03_ORDER), a->staging.stream(0))
             : build_on_device(a, a->staging.stream(0));
  }
  if (rc == NRT_OK) rc = derive_private_layout(a, a->staging.stream(0));
  if (rc != NRT_OK) {
    destroy(a);
    return rc;
  }
  *out = reinterpret_cast<nrt_accel *>(a);
  return NRT_OK;
}

int nrt_adopt(const void *nodes_40B, size_t n_nodes, const uint32_t *indices, size_t n_indices, const float *verts,
              size_t stride_bytes, size_t n_verts, const uint32_t *faces, uint32_t n_prims, nrt_accel **out) {
  if (!out) {
    g_err = "nrt_adopt: out is NULL";
    return NRT_ERR_INVALID;
  }
  *out = nullptr;
  if (!nodes_40B || !indices || !verts || !faces || n_nodes == 0 || n_prims == 0 || n_indices != n_prims ||
      stride_bytes < 12) {
    g_err = "nrt_adopt: bad arguments";
    return NRT_ERR_INVALID;
  }
  DeviceGuard dg_caller;  // select_device makes the chosen device current; the caller gets its own back
  int rc = select_device(nullptr);
  if (rc != NRT_OK) return rc;
  Accel *a = new (std::nothrow) Accel();
  if (!a) return NRT_ERR_NOMEM;
  a->options = default_build_options();
  const Node40 *hn = static_cast<const Node40 *>(nodes_40B);
  // An adopted tree is foreign data (a dump file): validate it once on the host before any kernel trusts it.
  {
    std::string why;
    if (!validate_foreign_tree(hn, n_nodes, indices, n_indices, n_prims, &a->stats, &why)) {
      g_err = "nrt_adopt: " + why;
      delete a;
      return NRT_ERR_INVALID;
    }
  }
  rc = common_init(a);
  if (rc == NRT_OK) rc = upload_geometry(a, verts, stride_bytes, n_verts, faces, n_prims);
  if (rc == NRT_OK) {
    a->n_nodes = n_nodes;
    cudaStream_t s = a->staging.stream(0);
    cudaError_t e = cudaMalloc(&a->d_nodes, sizeof(Node40) * n_nodes);
    if (e == cudaSuccess) e = cudaMalloc(&a->d_indices, sizeof(uint32_t) * n_indices);
    if (e == cudaSuccess) e = cudaMemcpyAsync(a->d_nodes, hn, sizeof(Node40) * n_nodes, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(a->d_indices, indices, sizeof(uint32_t) * n_indices, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) rc = cuda_fail(e, "nrt_adopt upload", __FILE__, __LINE__);
  }
  if (rc == NRT_OK) rc = derive_private_layout(a, a->staging.stream(0));
  if (rc != NRT_OK) {
    destroy(a);
    return rc;
  }
  a->mirror.assign(hn, n_nodes, indices, n_indices);
  for (int k = 0; k < 3; k++) {
    a->root_bmin[k] = hn[0].bmin[k];
    a->root_bmax[k] = hn[0].bmax[k];
  }
  *out = reinterpret_cast<nrt_accel *>(a);
  return NRT_OK;
}

void nrt_free(nrt_accel *h) { destroy(reinterpret_cast<Accel *>(h)); }

int nrt_stats(const nrt_accel *h, void *stats_16B) {
  if (!h || !stats_16B) {
    g_err = "nrt_stats: NULL argument";
    return NRT_ERR_INVALID;
  }
  memcpy(stats_16B, &reinterpret_cast<const Accel *>(h)->stats, sizeof(BuildStats16));
  return NRT_OK;
}

int nrt_bounding_box(const nrt_accel *h, float bmin[3], float bmax[3]) {
  if (!h || !bmin || !bmax) {
    g_err = "nrt_bounding_box: NULL argument";
    return NRT_ERR_INVALID;
  }
  const Accel *a = reinterpret_cast<const Accel *>(h);
  for (int k = 0; k < 3; k++) {
    bmin[k] = a->root_bmin[k];
    bmax[k] = a->root_bmax[k];
  }
  return NRT_OK;
}

int nrt_nodes(nrt_accel *h, const void **nodes_40B, size_t *n_nodes, const uint32_t **indices, size_t *n_indices) {
  if (!h) {
    g_err = "nrt_nodes: NULL accel";
    return NRT_ERR_INVALID;
  }
  Accel *a = reinterpret_cast<Accel *>(h);
  return a->mirror.get(a->device, a->d_nodes, a->n_nodes, a->d_indices, a->n_prims, nodes_40B, n_nodes, indices,
                       n_indices);
}

// Any number of calls of one accel may be in flight on any streams: fast launches take their ray cursor from the
// accel's ring, whose slots are ordered on the device (traverse.cu:launch_fast3_any).
int nrt_traverse_device(const nrt_accel *h, const void *d_rays_36B, size_t n_rays, void *d_hits_16B,
                        uint8_t *d_hit_mask, const void *trace_opts_16B, uint32_t flags, void *stream) {
  if (!h || (n_rays && (!d_rays_36B || !d_hits_16B))) {
    g_err = "nrt_traverse_device: NULL argument";
    return NRT_ERR_INVALID;
  }
  const Accel *a = reinterpret_cast<const Accel *>(h);
  TraceOptions16 opt = default_trace_options();
  if (trace_opts_16B) memcpy(&opt, trace_opts_16B, sizeof(opt));
  NRT_DEVICE(a->device);
  return launch_traverse(a, static_cast<const Ray36 *>(d_rays_36B), n_rays, static_cast<Hit16 *>(d_hits_16B),
                         d_hit_mask, opt, flags, static_cast<cudaStream_t>(stream));
}

int nrt_traverse_count_device(const nrt_accel *h, const void *d_rays_36B, size_t n_rays, const void *trace_opts_16B,
                              uint32_t flags, uint64_t *boxes_tested, uint64_t *prims_tested, void *stream) {
  if (!h || (n_rays && !d_rays_36B)) {
    g_err = "nrt_traverse_count_device: NULL argument";
    return NRT_ERR_INVALID;
  }
  const Accel *a = reinterpret_cast<const Accel *>(h);
  TraceOptions16 opt = default_trace_options();
  if (trace_opts_16B) memcpy(&opt, trace_opts_16B, sizeof(opt));
  NRT_DEVICE(a->device);
  std::lock_guard<std::mutex> lock(const_cast<Accel *>(a)->host_mu);  // d_counters[64..79] is per-accel scratch
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  uint64_t *d_counts = a->d_counters + 64;
  int rc = launch_traverse_count(a, static_cast<const Ray36 *>(d_rays_36B), n_rays, opt, flags, d_counts, s);
  if (rc != NRT_OK) return rc;
  uint64_t hc[2] = {0, 0};
  NRT_CUDA(cudaMemcpyAsync(hc, d_counts, sizeof(hc), cudaMemcpyDeviceToHost, s));
  NRT_CUDA(cudaStreamSynchronize(s));
  if (boxes_tested) *boxes_tested = hc[0];
  if (prims_tested) *prims_tested = hc[1];
  return NRT_OK;
}

int nrt_traverse_lane_stats_device(const nrt_accel *h, const void *d_rays_36B, size_t n_rays, const void *trace_opts_16B,
                                   uint32_t flags, uint64_t *stats16, void *stream) {
  if (!h || !stats16 || (n_rays && !d_rays_36B)) {
    g_err = "nrt_traverse_lane_stats_device: NULL argument";
    return NRT_ERR_INVALID;
  }
  const Accel *a = reinterpret_cast<const Accel *>(h);
  TraceOptions16 opt = default_trace_options();
  if (trace_opts_16B) memcpy(&opt, trace_opts_16B, sizeof(opt));
  NRT_DEVICE(a->device);
  std::lock_guard<std::mutex> lock(const_cast<Accel *>(a)->host_mu);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  uint64_t *d_counts = a->d_counters + 64;
  int rc = launch_traverse_count(a, static_cast<const Ray36 *>(d_rays_36B), n_rays, opt, flags, d_counts, s);
  if (rc != NRT_OK) return rc;
  NRT_CUDA(cudaMemcpyAsync(stats16, d_counts, 16 * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  NRT_CUDA(cudaStreamSynchronize(s));
  return NRT_OK;
}

// Host-pointer path: a few rays go through the zero-copy pool (not serialised with other host threads), more through
// the staging pipeline.  RAY32 calls move 32 B per ray (the pool's slots are laid out for 36 B).
int nrt_traverse(const nrt_accel *h, const void *rays_36B, size_t n_rays, void *hits_16B, uint8_t *hit_mask,
                 const void *trace_opts_16B, uint32_t flags) {
  if (!h || (n_rays && (!rays_36B || !hits_16B))) {
    g_err = "nrt_traverse: NULL argument";
    return NRT_ERR_INVALID;
  }
  if (n_rays == 0) return NRT_OK;
  Accel *a = const_cast<Accel *>(reinterpret_cast<const Accel *>(h));
  TraceOptions16 opt = default_trace_options();
  if (trace_opts_16B) memcpy(&opt, trace_opts_16B, sizeof(opt));
  const size_t ray_bytes = (flags & NRT_TRAVERSE_RAY32) ? 32 : sizeof(Ray36);
  NRT_DEVICE(a->device);
  if (n_rays <= decltype(a->small)::kMaxRays) {
    return a->small.run(rays_36B, n_rays, ray_bytes, hits_16B, hit_mask,
                        [&](int i, void *h_rays, void *h_hits, uint8_t *h_mask, cudaStream_t s) {
                          return launch_traverse(a, static_cast<const Ray36 *>(h_rays), n_rays, static_cast<Hit16 *>(h_hits),
                                                 h_mask, opt, flags, s,
                                                 reinterpret_cast<unsigned long long *>(a->d_counters) +
                                                     Accel::kSmallCursor0 + i);
                        });
  }
  return a->staging.run(rays_36B, n_rays, ray_bytes, hits_16B, sizeof(Hit16), hit_mask,
                        [&](const void *d_rays, size_t m, void *d_hits, uint8_t *d_mask, cudaStream_t s) {
                          return launch_traverse(a, static_cast<const Ray36 *>(d_rays), m, static_cast<Hit16 *>(d_hits),
                                                 d_mask, opt, flags, s);
                        });
}

void *nrt_host_alloc(size_t bytes) {
  void *p = nullptr;
  if (cudaMallocHost(&p, bytes) != cudaSuccess) {
    cudaGetLastError();
    g_err = "nrt_host_alloc: cudaMallocHost failed";
    return nullptr;
  }
  return p;
}

void nrt_host_free(void *p) {
  if (p) cudaFreeHost(p);
}

}  // extern "C"
