// Non-triangle primitives: the device side of nanort's "bring your own Prim / Pred / Intersector" concept
// (nanort.h:698-860, 1014-1229; model examples/particle_primitive/main.cc:161-291).
//
// The reference takes three user classes: Prim (BoundingBox / BoundingBoxAndCenter per primitive), Pred (the SAH
// partition predicate) and an Intersector (Intersect / Update / PrepareTraversal / PostTraversal).  Host functors
// cannot run inside a CUDA kernel, so the hook is a set of primitive KINDS, each the device restatement of one of the
// reference's own primitive models, selected through the C-ABI (nrt_build_prims) or, in include/nanort.h, by the type of
// the classes handed to BVHAccel::Build / Traverse:
//   NRT_PRIM_SPHERES   examples/particle_primitive: SphereGeometry (box = center -+ radius), SphereIntersector
//                      (quadratic with the cgsociety "q" form, nearest non-negative root, u/v from atan2 / acos)
//   NRT_PRIM_BOXES     the node-level primitive of the two-level API: NodeBBoxGeometry / NodeBBoxIntersector of
//                      examples/nanosg/nanosg.h:447-560 (axis-aligned boxes; BVHAccel::ListNodeIntersections,
//                      nanort.h:2607-2692, lists the boxes a ray pierces, nearest first, at most max_intersections)
// Every kind is a bounding-box build (build.cu's box-primitive path: exact boxes, binned SAH over box centres) plus a
// leaf test in the kind's own arithmetic order, compiled with --fmad=false like everything else.
#include <string.h>

#include <algorithm>
#include <mutex>
#include <new>

#include "common.cuh"
#include "trav_common.cuh"
#include "nodehits.cuh"

namespace nrt {

namespace {

__global__ void sphere_boxes_kernel(const float *__restrict__ centers, size_t stride_floats, const float *__restrict__ radii,
                                    uint32_t n, float *__restrict__ boxes6, float4 *__restrict__ prim4) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float *c = centers + (size_t)i * stride_floats;
  const float r = radii[i];
  // SphereGeometry::BoundingBox (particle_primitive/main.cc:112-119)
  boxes6[6 * (size_t)i + 0] = c[0] - r;
  boxes6[6 * (size_t)i + 1] = c[1] - r;
  boxes6[6 * (size_t)i + 2] = c[2] - r;
  boxes6[6 * (size_t)i + 3] = c[0] + r;
  boxes6[6 * (size_t)i + 4] = c[1] + r;
  boxes6[6 * (size_t)i + 5] = c[2] + r;
  prim4[i] = make_float4(c[0], c[1], c[2], r);
}

// leaf slots of a sphere accel: a = {center.xyz, prim id bits}, b = {radius, -, -, last-in-leaf flag (kept)}
__global__ void sphere_slots_kernel(const uint32_t *__restrict__ indices, const float4 *__restrict__ prim4, uint32_t n,
                                    PackedTri *__restrict__ slots) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const uint32_t prim = indices[s];
  const float4 p = prim4[prim];
  slots[s].a = make_float4(p.x, p.y, p.z, __uint_as_float(prim));
  slots[s].b.x = p.w;
}

struct SphereBest {
  float t;
  uint32_t prim;
};

// SphereIntersector::Intersect (particle_primitive/main.cc:172-245), same operation order.  NOTE what the reference
// does and does not do: no min_t test (only the boxes see the ray's range), ties (t == *t_inout) replace.
__device__ __forceinline__ bool sphere_test(const TraceOptions16 &opt, float ox, float oy, float oz, float dx, float dy,
                                            float dz, float4 a, float radius, float &t_inout) {
  const uint32_t prim = __float_as_uint(a.w);
  if (prim < opt.prim_ids_range[0] || prim >= opt.prim_ids_range[1]) return false;
  const float ocx = ox - a.x, ocy = oy - a.y, ocz = oz - a.z;
  const float A = (dx * dx + dy * dy) + dz * dz;
  const float B = 2.0f * ((dx * ocx + dy * ocy) + dz * ocz);
  const float Cc = ((ocx * ocx + ocy * ocy) + ocz * ocz) - radius * radius;
  const float disc = B * B - (4.0f * A) * Cc;
  float t0, t1;
  if (disc < 0.0f) return false;
  if (fabsf(disc) < FLT_EPSILON) {
    t0 = t1 = -0.5f * (B / A);
  } else {
    const float ds = sqrtf(disc);
    const float q = B < 0.0f ? (-B - ds) / 2.0f : (-B + ds) / 2.0f;
    t0 = q / A;
    t1 = Cc / q;
  }
  if (t0 > t1) {
    const float tmp = t0;
    t0 = t1;
    t1 = tmp;
  }
  if (t1 < 0.0f) return false;
  const float t = t0 < 0.0f ? t1 : t0;
  if (t > t_inout) return false;
  t_inout = t;
  return true;
}

// One thread per ray over the 64-byte child-pair nodes, nearer child first, (ref, entry distance) stack with the same
// cull-at-pop rule as the triangle kernels; leaf test = sphere_test.  Hit record {u, v, t, prim}: PostTraversal's
// spherical coordinates of the hit normal (main.cc:264-277, double-precision atan2 / acos as there).
constexpr int kPrimStack = 512;  // kNANORT_MAX_STACK_DEPTH

__global__ void __launch_bounds__(128)
    traverse_spheres_kernel(const WideNode *__restrict__ wide, const PackedTri *__restrict__ slots, const Ray36 *__restrict__ rays,
                            size_t n, Hit16 *__restrict__ hits, uint8_t *__restrict__ mask, TraceOptions16 opt, uint32_t flags) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float *rp = reinterpret_cast<const float *>(rays + i);
  const float ox = __ldg(rp), oy = __ldg(rp + 1), oz = __ldg(rp + 2), dx = __ldg(rp + 3), dy = __ldg(rp + 4),
              dz = __ldg(rp + 5), min_t = __ldg(rp + 6), max_t = __ldg(rp + 7);
  RayCtx c;
  setup_ray(c, ox, oy, oz, dx, dy, dz, min_t, (flags & NRT_TRAVERSE_CPP03_INVERSE) != 0);
  float best_t = max_t;
  uint32_t best_prim = 0xFFFFFFFFu;
  float bcx = 0.0f, bcy = 0.0f, bcz = 0.0f;  // centre of the best sphere, for PostTraversal
  uint2 stack[kPrimStack];
  int sp = 0;
  int cur = range_has_nan(min_t, max_t) ? kEmptyLeaf : 0;
  for (;;) {
    if (cur == kEmptyLeaf) {
      bool got = false;
      while (sp > 0) {
        const uint2 e = stack[--sp];
        if (__uint_as_float(e.y) <= best_t) {
          cur = (int)e.x;
          got = true;
          break;
        }
      }
      if (!got) break;
    }
    if (cur >= 0) {
      const float4 *p = reinterpret_cast<const float4 *>(wide + cur);
      const float4 q0 = __ldg(p), q1 = __ldg(p + 1), q2 = __ldg(p + 2);
      const int4 q3 = __ldg(reinterpret_cast<const int4 *>(p + 3));
      float t0, t1;
      const bool h0 = slab(c, q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, min_t, best_t, t0);
      const bool h1 = slab(c, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, min_t, best_t, t1);
      if (h0 && h1) {
        const bool swap = t1 < t0;
        if (sp < kPrimStack) stack[sp++] = make_uint2((uint32_t)(swap ? q3.x : q3.y), __float_as_uint(swap ? t0 : t1));
        cur = swap ? q3.y : q3.x;
      } else {
        cur = h0 ? q3.x : (h1 ? q3.y : kEmptyLeaf);
      }
    } else {  // leaf: ~cur = first slot
      const PackedTri *s = slots + (size_t)(~cur);
      for (;;) {
        const float4 a = __ldg(&s->a), b = __ldg(&s->b);
        float t = best_t;
        if (sphere_test(opt, ox, oy, oz, dx, dy, dz, a, b.x, t)) {
          best_t = t;
          best_prim = __float_as_uint(a.w);
          bcx = a.x;
          bcy = a.y;
          bcz = a.z;
        }
        if (__float_as_uint(b.w) != 0u) break;
        s++;
      }
      cur = kEmptyLeaf;
    }
  }
  const bool hit = best_prim != 0xFFFFFFFFu && best_t < max_t;  // nanort.h:2552
  float4 r = make_float4(0.0f, 0.0f, max_t, __uint_as_float(0xFFFFFFFFu));
  if (hit) {  // SphereIntersector::PostTraversal (main.cc:264-277)
    float nx = (ox + best_t * dx) - bcx, ny = (oy + best_t * dy) - bcy, nz = (oz + best_t * dz) - bcz;
    const float len = sqrtf((nx * nx + ny * ny) + nz * nz);  // nanort::vnormalize (nanort.h:387-398)
    if (fabsf(len) > FLT_EPSILON) {
      const float inv = 1.0f / len;
      nx *= inv;
      ny *= inv;
      nz *= inv;
    }
    const float u = (float)(atan2((double)nx, (double)nz) + 3.14159265358979323846) * 0.5f * (float)(1.0 / 3.14159265358979323846);
    const float v = (float)(acos((double)ny) / 3.14159265358979323846);
    r = make_float4(u, v, best_t, __uint_as_float(best_prim));
  }
  reinterpret_cast<float4 *>(hits)[i] = r;
  if (mask) mask[i] = hit ? 1 : 0;
}

// ---- BVHAccel::ListNodeIntersections over a box accel (nanort.h:2607-2692 with NodeBBoxIntersector): the reference's
// walk of the 40-byte node array (hit_t stays at ray.max_t), the at-most-K-nearest heap with libstdc++'s sift rules, the
// result in nearest-first order.  out_hits: K records {t_min, t_max, node_id} per ray; out_count: records filled.
struct NodeHit12 {
  float t_min, t_max;
  uint32_t node_id;
};

__global__ void __launch_bounds__(128)
    list_boxes_kernel(const Node40 *__restrict__ nodes, const uint32_t *__restrict__ indices, const float *__restrict__ boxes6,
                      const Ray36 *__restrict__ rays, size_t n, int max_k, NodeHit12 *__restrict__ out_hits,
                      uint32_t *__restrict__ out_count, uint32_t flags) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const WorldRay w = load_world(rays, i);
  RayCtx c;
  setup_ray(c, w.ox, w.oy, w.oz, w.dx, w.dy, w.dz, w.min_t, (flags & NRT_TRAVERSE_CPP03_INVERSE) != 0);
  NodeHitHeap heap;
  collect_node_hits(nodes, indices, [=](uint32_t id) { return boxes6 + 6 * (size_t)id; }, w, c, max_k, heap);
  // t_max of each listed box, recomputed (cheap: K <= 64)
  const float rix = 1.0f / w.dx, riy = 1.0f / w.dy, riz = 1.0f / w.dz;
  for (int k = 0; k < heap.n; k++) {
    const uint32_t id = heap.id[k];
    float tmin, tmax;
    raw_box(w, rix, riy, riz, boxes6 + 6 * (size_t)id, tmin, tmax);
    out_hits[i * (size_t)max_k + k] = NodeHit12{heap.t[k], tmax, id};
  }
  out_count[i] = (uint32_t)heap.n;
}

}  // namespace
}  // namespace nrt

using namespace nrt;

namespace nrt {
// traverse.cu dispatches here for sphere accels
int launch_traverse_prims(const Accel *a, const Ray36 *d_rays, size_t n, Hit16 *d_hits, uint8_t *d_mask,
                          const TraceOptions16 &opt, uint32_t flags, cudaStream_t s) {
  if (n == 0) return NRT_OK;
  if (a->prim_kind != NRT_PRIM_SPHERES) {
    set_error("nrt_traverse: this accel holds boxes; use nrt_list_node_intersections");
    return NRT_ERR_INVALID;
  }
  traverse_spheres_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(a->d_wide, a->d_tris, d_rays, n, d_hits, d_mask, opt, flags);
  NRT_CUDA(cudaGetLastError());
  return NRT_OK;
}
}  // namespace nrt

extern "C" {

int nrt_build_prims(uint32_t kind, const float *data, size_t stride_bytes, const float *aux, uint32_t n_prims,
                    const void *build_opts_28B, nrt_accel **out) {
  if (!out) {
    set_error("nrt_build_prims: out is NULL");
    return NRT_ERR_INVALID;
  }
  *out = nullptr;
  if (n_prims == 0) {  // reference: Build returns false (nanort.h:1907-1909)
    set_error("nrt_build_prims: num_primitives == 0");
    return NRT_ERR_INVALID;
  }
  if (!data || (kind == NRT_PRIM_SPHERES && (!aux || stride_bytes < 12 || (stride_bytes % 4) != 0)) ||
      (kind == NRT_PRIM_BOXES && stride_bytes != 24) || (kind != NRT_PRIM_SPHERES && kind != NRT_PRIM_BOXES)) {
    set_error("nrt_build_prims: bad kind / pointers / stride (spheres: centers with stride >= 12 + radii; boxes: 6 floats each)");
    return NRT_ERR_INVALID;
  }
  DeviceGuard dg_caller;
  int device = 0;
  int rc = select_device(&device);
  if (rc != NRT_OK) return rc;
  Accel *a = new (std::nothrow) Accel();
  if (!a) return NRT_ERR_NOMEM;
  a->device = device;
  a->prim_kind = (int)kind;
  a->n_prims = n_prims;
  a->options = default_build_options();
  if (build_opts_28B) memcpy(&a->options, build_opts_28B, sizeof(BuildOptions28));
  float *d_in = nullptr, *d_aux = nullptr;
  cudaError_t e = cudaSuccess;
  auto fail = [&](int code) {
    cudaFree(d_in);
    cudaFree(d_aux);
    nrt_free(reinterpret_cast<nrt_accel *>(a));
    return code;
  };
  if (a->options.bin_size < 2 || a->options.max_tree_depth > 500) {
    set_error("nrt_build_prims: bin_size must be > 1 and max_tree_depth <= 500");
    return fail(NRT_ERR_INVALID);
  }
  rc = common_init(a);
  if (rc != NRT_OK) return fail(rc);
  cudaStream_t s = a->staging.stream(0);
  if (e == cudaSuccess) e = cudaMalloc(&a->d_prim_boxes, sizeof(float) * 6 * (size_t)n_prims);
  if (kind == NRT_PRIM_SPHERES) {
    const size_t in_bytes = (size_t)(n_prims - 1) * stride_bytes + 12;
    if (e == cudaSuccess) e = cudaMalloc(&d_in, (in_bytes + 3) & ~(size_t)3);
    if (e == cudaSuccess) e = cudaMalloc(&d_aux, sizeof(float) * (size_t)n_prims);
    if (e == cudaSuccess) e = cudaMalloc(&a->d_prim_data, sizeof(float4) * (size_t)n_prims);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_in, data, in_bytes, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_aux, aux, sizeof(float) * (size_t)n_prims, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) {
      sphere_boxes_kernel<<<(n_prims + 255) / 256, 256, 0, s>>>(d_in, stride_bytes / 4, d_aux, n_prims, a->d_prim_boxes,
                                                               static_cast<float4 *>(a->d_prim_data));
      e = cudaGetLastError();
    }
  } else {
    if (e == cudaSuccess) e = cudaMemcpyAsync(a->d_prim_boxes, data, sizeof(float) * 6 * (size_t)n_prims, cudaMemcpyHostToDevice, s);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return fail(cuda_fail(e, "nrt_build_prims upload", __FILE__, __LINE__));
  rc = build_on_device(a, s);  // box-primitive path of the production builder: exact boxes, binned SAH over box centres
  if (rc == NRT_OK) rc = derive_private_layout(a, s);
  if (rc == NRT_OK && kind == NRT_PRIM_SPHERES) {
    sphere_slots_kernel<<<(n_prims + 255) / 256, 256, 0, s>>>(a->d_indices, static_cast<const float4 *>(a->d_prim_data), n_prims,
                                                             a->d_tris);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) rc = cuda_fail(e, "nrt_build_prims slots", __FILE__, __LINE__);
  }
  if (rc != NRT_OK) return fail(rc);
  cudaFree(d_in);
  cudaFree(d_aux);
  *out = reinterpret_cast<nrt_accel *>(a);
  return NRT_OK;
}

int nrt_list_node_intersections(const nrt_accel *h, const void *rays_36B, size_t n_rays, int max_intersections,
                                void *hits_12B, uint32_t *counts, uint32_t flags) {
  if (!h || (n_rays && (!rays_36B || !hits_12B || !counts)) || max_intersections < 1 || max_intersections > kMaxNodeHits) {
    set_error("nrt_list_node_intersections: bad arguments (1 <= max_intersections <= 64)");
    return NRT_ERR_INVALID;
  }
  const Accel *a = reinterpret_cast<const Accel *>(h);
  if (a->prim_kind != NRT_PRIM_BOXES || !a->d_prim_boxes) {
    set_error("nrt_list_node_intersections: the accel was not built over boxes (nrt_build_prims(NRT_PRIM_BOXES, ...))");
    return NRT_ERR_INVALID;
  }
  if (n_rays == 0) return NRT_OK;
  NRT_DEVICE(a->device);
  std::lock_guard<std::mutex> lock(const_cast<Accel *>(a)->host_mu);
  cudaStream_t s = a->staging.stream(0);
  Ray36 *d_rays = nullptr;
  NodeHit12 *d_hits = nullptr;
  uint32_t *d_cnt = nullptr;
  cudaError_t e = cudaMalloc(&d_rays, sizeof(Ray36) * n_rays);
  if (e == cudaSuccess) e = cudaMalloc(&d_hits, sizeof(NodeHit12) * n_rays * (size_t)max_intersections);
  if (e == cudaSuccess) e = cudaMalloc(&d_cnt, sizeof(uint32_t) * n_rays);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_rays, rays_36B, sizeof(Ray36) * n_rays, cudaMemcpyHostToDevice, s);
  // records beyond counts[ray] are never written by the kernel: hand the caller zeros, not device garbage
  if (e == cudaSuccess) e = cudaMemsetAsync(d_hits, 0, sizeof(NodeHit12) * n_rays * (size_t)max_intersections, s);
  if (e == cudaSuccess) {
    list_boxes_kernel<<<(unsigned)((n_rays + 127) / 128), 128, 0, s>>>(a->d_nodes, a->d_indices, a->d_prim_boxes, d_rays, n_rays,
                                                                     max_intersections, d_hits, d_cnt, flags);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(hits_12B, d_hits, sizeof(NodeHit12) * n_rays * (size_t)max_intersections, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(counts, d_cnt, sizeof(uint32_t) * n_rays, cudaMemcpyDeviceToHost, s);
  const cudaError_t es = cudaStreamSynchronize(s);
  if (e == cudaSuccess) e = es;
  cudaFree(d_rays);
  cudaFree(d_hits);
  cudaFree(d_cnt);
  if (e != cudaSuccess) return cuda_fail(e, "nrt_list_node_intersections", __FILE__, __LINE__);
  return NRT_OK;
}

}  // extern "C"
