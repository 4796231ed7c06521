// Ray traversal kernels (sm_90a).  Compiled with --fmad=false: every float
// operation below is individually rounded, exactly like the reference's x86-64
// SSE2 scalar code (SURVEY.md F2 / Appendix B), so sign decisions on U/V/W and
// the reported t/u/v are bit-identical to CPU nanort for the same triangle.
//
// Replaces (file:line in the reference tree):
//   BVHAccel<float>::Traverse            nanort.h:2487-2556
//   BVHAccel<float>::TestLeafNode        nanort.h:2372-2407
//   IntersectRayAABB<float>              nanort.h:2284-2325
//   TriangleIntersector::Intersect       nanort.h:1054-1150
//   TriangleIntersector::PrepareTraversal nanort.h:1163-1201
//   vsafe_inverse                        nanort.h:414-465
#include <float.h>
#include <math_constants.h>

#include "common.cuh"
#include "trav_common.cuh"
#include "wavefront.cuh"
#include "traverse3.cuh"

namespace nrt {

// ------------------------------------------------------------------ ray loaders
struct AosRays {
  static constexpr int kPayloadWords = 0;
  static constexpr bool kSharedOrigin = false;  // rays start anywhere (wavefront.cuh, CameraRaysT)
  const Ray36 *rays;
  __device__ __forceinline__ void load(size_t i, float &ox, float &oy, float &oz, float &dx, float &dy,
                                       float &dz, float &tmin, float &tmax, uint32_t * = nullptr) const {
    const float *p = reinterpret_cast<const float *>(rays + i);
    ox = __ldcs(p + 0);
    oy = __ldcs(p + 1);
    oz = __ldcs(p + 2);
    dx = __ldcs(p + 3);
    dy = __ldcs(p + 4);
    dz = __ldcs(p + 5);
    tmin = __ldcs(p + 6);
    tmax = __ldcs(p + 7);
  }
};

// 32-byte ray records (NRT_TRAVERSE_RAY32): {org.xyz, dir.x} {dir.yz, min_t, max_t}, two 128-bit loads
struct Aos32Rays {
  static constexpr int kPayloadWords = 0;
  static constexpr bool kSharedOrigin = false;  // rays start anywhere (wavefront.cuh, CameraRaysT)
  const float4 *rays;
  __device__ __forceinline__ void load(size_t i, float &ox, float &oy, float &oz, float &dx, float &dy,
                                       float &dz, float &tmin, float &tmax, uint32_t * = nullptr) const {
    const float4 a = __ldcs(rays + 2 * i), b = __ldcs(rays + 2 * i + 1);
    ox = a.x;
    oy = a.y;
    oz = a.z;
    dx = a.w;
    dy = b.x;
    dz = b.y;
    tmin = b.z;
    tmax = b.w;
  }
};

struct SoaRays {
  static constexpr int kPayloadWords = 0;
  static constexpr bool kSharedOrigin = false;  // rays start anywhere (wavefront.cuh, CameraRaysT)
  const float4 *org_tmin;
  const float4 *dir_tmax;
  __device__ __forceinline__ void load(size_t i, float &ox, float &oy, float &oz, float &dx, float &dy,
                                       float &dz, float &tmin, float &tmax, uint32_t * = nullptr) const {
    float4 o = __ldcs(org_tmin + i);  // read once: evict-first, keep L1/L2 for the tree
    float4 d = __ldcs(dir_tmax + i);
    ox = o.x;
    oy = o.y;
    oz = o.z;
    tmin = o.w;
    dx = d.x;
    dy = d.y;
    dz = d.z;
    tmax = d.w;
  }
};

// ------------------------------------------------------------------ conformance walk
// One thread per ray over the nanort 40-byte node array in the reference's exact order (reference_walk).
template <class Rays, bool COUNT>
__global__ void __launch_bounds__(128)
    traverse_conformance_kernel(const Node40 *__restrict__ nodes, const PackedTri *__restrict__ tris,
                                Rays rays, size_t n, Hit16 *__restrict__ hits, uint8_t *__restrict__ mask,
                                TraceOptions16 opt, uint32_t flags, unsigned long long *counts,
                                const unsigned long long *n_ptr) {
  if (n_ptr) n = (size_t)*n_ptr;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long visits[2] = {0, 0};  // boxes, prims
  if (i < n) {
    float ox, oy, oz, dx, dy, dz, min_t, max_t;
    rays.load(i, ox, oy, oz, dx, dy, dz, min_t, max_t);
    RayCtx c;
    setup_ray(c, ox, oy, oz, dx, dy, dz, min_t, (flags & NRT_TRAVERSE_CPP03_INVERSE) != 0);
    Best best;
    best.t = max_t;
    best.u = 0.0f;
    best.v = 0.0f;
    best.prim = 0xFFFFFFFFu;
    reference_walk(nodes, c, min_t, max_t, PackedTriLeaf{tris, c, opt, best}, COUNT ? visits : nullptr);
    if (hits) write_result(hits, mask, i, best, max_t);
  }
  if (COUNT) {
    for (int o = 16; o > 0; o >>= 1) {
      visits[0] += __shfl_down_sync(FULL_MASK, visits[0], o);
      visits[1] += __shfl_down_sync(FULL_MASK, visits[1], o);
    }
    if ((threadIdx.x & 31) == 0) {
      atomicAdd(counts + 0, visits[0]);
      atomicAdd(counts + 1, visits[1]);
    }
  }
}

// ------------------------------------------------------------------ launchers
static int g_sm_count[64] = {0};
int device_sm_count(int device) {
  if (device < 0 || device >= 64) return 132;
  if (g_sm_count[device] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || v <= 0) v = 132;
    g_sm_count[device] = v;
  }
  return g_sm_count[device];
}

// Launch policies (Policy3, traverse3.cuh), chosen by sweeps on the GPU this library was first written for and not
// re-swept on H100 (DESIGN.md section 10): 10 CTAs per SM (48 registers).  Coherent launches (camera rays,
// caller-supplied rays) read the 128-byte PairNode (no selects: they are issue bound); incoherent launches (AO, shadow
// and bounce rays) and trees whose PairNode array would not stay L2-resident read the 64-byte WideNode (they are bound
// by the L1 data pipe and by cache capacity, and the ALU pipe has room for the 12 selects).
// Leaf batching: after the first leaf round of an outer iteration another one runs only while >= 8 (coherent) / >= 12
// (incoherent) lanes hold a leaf -- a lane's second leaf otherwise costs a round of its own at ~5 active lanes; the
// camera-ray launch, whose retire step spawns the AO ray (630 instructions), also waits with the retire step until
// retired + empty lanes reach the refill threshold.
// Two node steps per evaluation of the node phase's exit conditions (+1.8 ... +2.8 %).
// Refill threshold: with deferred retire the camera launch does best when a warp takes a whole new 8x4-pixel packet
// only after ALL its lanes have finished (32) -- its rays have similar lengths, and the AO rays it spawns then reach
// the AO queue in packets of neighbouring pixels, which speeds the AO launch up too; caller-supplied rays 24;
// incoherent launches 20 (28 and more lose 10-50 % there).
//                 MINB REFILL PAIR128 LEAF_AGAIN DEFER NODE_UNROLL
typedef Policy3<10, 24, true, 8, false, 2> DefaultPolicy;
// The camera launch over the accel's own arrays runs 9 CTAs per SM (56 registers: its AO-spawn retire step spills at
// 48) and, like the incoherent launches, three node steps per exit check.  Re-swept on H100 (80GB HBM3, 700 W) over the camera-relative layout and
// the precomputed face normals: MINB 9/10 x NODE_UNROLL 2/3 all lie within 1 % of each other on the bench headline
// (10 spills 32 B at 48 registers), so this row stays (DESIGN.md section 10).
typedef Policy3<9, 32, true, 12, true, 3> CameraPolicy;
// The packet walk of the camera launch over the camera-relative copies (traverse_packet_kernel): two samples per lane,
// 7 CTAs per SM (72 registers, 28 B spilled).  Swept on H100 (80GB HBM3, 700 W; DESIGN.md section 10): one sample per
// lane at 9 CTAs (56 registers) is 5 % slower on the bench headline; two samples at 6 CTAs (80 registers, no spills)
// 2 %; at 8 and 9 CTAs they spill 92 B and more.
typedef PacketPolicy<7, 2> CameraPacketPolicy;
typedef Policy3<10, 20, false, 12, false, 3> IncoherentPolicy;
typedef Policy3<9, 32, false, 12, true, 3> IncoherentCameraPolicy;
// The path tracer's radiance launch: its retire step IS the shading block, which needs more registers than the plain
// traversal (8 CTAs per SM, 64 registers) and runs deferred (with more lanes).
typedef Policy3<8, 24, false, 8, true, 2> PathRadiancePolicy;
// PairNode arrays above this size are not used (50 MB L2; the triangles want their share)
constexpr size_t kPair128MaxBytes = (size_t)38 << 20;
// The camera launch reads camera-relative copies of the PairNode and TriCM arrays (traverse3.cuh, from_origin) only
// while the originals plus the copies fit in this: the AO launch that follows reads the originals, and the copies must
// not evict them (the H100's L2 is two partitions of 25 MB)
constexpr size_t kCameraRelMaxBytes = (size_t)24 << 20;

template <class Rays, int DEPTH, bool COUNT, class P, class Epi>
static cudaError_t launch_fast3(const Accel *a, Rays rays, size_t n, Epi epi, const TraceOptions16 &opt,
                                uint32_t flags, unsigned long long *cursor, unsigned long long *d_counts,
                                const unsigned long long *n_ptr, cudaStream_t s) {
  const int sms = device_sm_count(a->device);
  const size_t warps_per_block = kTraverseBlock / 32;
  size_t grid = (size_t)sms * P::kMinBlocks;  // persistent: every SM holds its full complement of CTAs
  const size_t need_blocks = ((n + 31) / 32 + warps_per_block - 1) / warps_per_block;
  if (grid > need_blocks) grid = need_blocks;
  if (grid == 0) grid = 1;
  const void *nodes = Rays::kSharedOrigin ? static_cast<const void *>(a->d_pair_rel)
                     : P::kPair128        ? static_cast<const void *>(a->d_pair)
                                          : static_cast<const void *>(a->d_wide);
  const TriCM *tris = Rays::kSharedOrigin ? a->d_tris_rel : a->d_tris_cm;
  traverse_fast3_kernel<Rays, DEPTH, COUNT, P, Epi><<<(unsigned)grid, kTraverseBlock, 0, s>>>(
      nodes, tris, rays, n, epi, opt, flags, cursor, d_counts, n_ptr);
  return cudaGetLastError();
}

// a child pair pushes at most one entry and descends one level: the stack never holds more entries than the tree
// has levels.  Two instantiations: 64 entries (every tree the production builder emits) and 512 (the reference's
// kNANORT_MAX_STACK_DEPTH, for adopted trees; nrt_build / nrt_adopt reject deeper ones).
static bool needs_deep_stack(const Accel *a) { return a->stats.max_tree_depth + 2 > 64u; }

template <class Rays, bool COUNT, class P, class Epi>
static int launch_fast3_cursor(const Accel *a, Rays rays, size_t n, Epi epi, const TraceOptions16 &opt, uint32_t flags,
                               unsigned long long *d_counts, const unsigned long long *n_ptr, cudaStream_t s,
                               unsigned long long *cursor) {
  NRT_CUDA(cudaMemsetAsync(cursor, 0, sizeof(unsigned long long), s));
  cudaError_t e;
  if (needs_deep_stack(a))
    e = launch_fast3<Rays, 512, COUNT, P>(a, rays, n, epi, opt, flags, cursor, d_counts, n_ptr, s);
  else
    e = launch_fast3<Rays, 64, COUNT, P>(a, rays, n, epi, opt, flags, cursor, d_counts, n_ptr, s);
  NRT_CUDA(e);
  return NRT_OK;
}

// `cursor`: a cursor the caller owns (the small-call slots: held until their launch has finished), or nullptr for the
// next one of the accel's ring (Accel::ring)
template <class Rays, bool COUNT, class P, class Epi>
static int launch_fast3_any(const Accel *a, Rays rays, size_t n, Epi epi, const TraceOptions16 &opt, uint32_t flags,
                            unsigned long long *d_counts, const unsigned long long *n_ptr, cudaStream_t s,
                            unsigned long long *cursor = nullptr) {
  if (!a->d_pair || !a->d_tris_cm) {
    set_error("traverse: this accel has no triangle traversal layout");
    return NRT_ERR_INVALID;
  }
  if (cursor) return launch_fast3_cursor<Rays, COUNT, P>(a, rays, n, epi, opt, flags, d_counts, n_ptr, s, cursor);
  return a->ring.run(s, [&](uint32_t k) {
    return launch_fast3_cursor<Rays, COUNT, P>(a, rays, n, epi, opt, flags, d_counts, n_ptr, s,
                                               reinterpret_cast<unsigned long long *>(a->d_counters) + 16 + k);
  });
}

// the default for coherent launches, with the size cut-off
template <class Rays, bool COUNT, class Epi>
static int launch_fast3_coherent(const Accel *a, Rays rays, size_t n, Epi epi, const TraceOptions16 &opt, uint32_t flags,
                                 unsigned long long *d_counts, const unsigned long long *n_ptr, cudaStream_t s,
                                 unsigned long long *cursor = nullptr) {
  if (a->n_wide * sizeof(PairNode) > kPair128MaxBytes)
    return launch_fast3_any<Rays, COUNT, IncoherentPolicy>(a, rays, n, epi, opt, flags, d_counts, n_ptr, s, cursor);
  return launch_fast3_any<Rays, COUNT, DefaultPolicy>(a, rays, n, epi, opt, flags, d_counts, n_ptr, s, cursor);
}

template <class Rays, bool COUNT>
static int launch_fast(const Accel *a, Rays rays, size_t n, Hit16 *d_hits, uint8_t *d_mask,
                       const TraceOptions16 &opt, uint32_t flags, unsigned long long *d_counts, cudaStream_t s,
                       const unsigned long long *n_ptr = nullptr, unsigned long long *cursor = nullptr) {
  if (!COUNT && ((flags >> 8) & 0xFFu) != 0) {  // the counting walk ignores them
    set_error("nrt_traverse: flags bits 8..15 are reserved");
    return NRT_ERR_INVALID;
  }
  const StoreHitsEpilogue epi{d_hits, d_mask};
  return launch_fast3_coherent<Rays, COUNT>(a, rays, n, epi, opt, flags, d_counts, n_ptr, s, cursor);
}

template <class Rays, bool COUNT>
static int launch_conf(const Accel *a, Rays rays, size_t n, Hit16 *d_hits, uint8_t *d_mask,
                       const TraceOptions16 &opt, uint32_t flags, unsigned long long *d_counts, cudaStream_t s,
                       const unsigned long long *n_ptr = nullptr) {
  size_t grid = (n + 127) / 128;
  if (grid == 0) return NRT_OK;
  traverse_conformance_kernel<Rays, COUNT><<<(unsigned)grid, 128, 0, s>>>(a->d_nodes, a->d_tris, rays, n, d_hits,
                                                                       d_mask, opt, flags, d_counts, n_ptr);
  NRT_CUDA(cudaGetLastError());
  return NRT_OK;
}

int launch_traverse(const Accel *a, const Ray36 *d_rays, size_t n, Hit16 *d_hits, uint8_t *d_mask,
                    const TraceOptions16 &opt, uint32_t flags, cudaStream_t s, unsigned long long *cursor) {
  if (n == 0) return NRT_OK;
  if (flags & NRT_TRAVERSE_RAY32) {  // compact records: default policy only
    if (a->prim_kind != 0 || (reinterpret_cast<uintptr_t>(d_rays) & 15u) != 0) {
      set_error("nrt_traverse: NRT_TRAVERSE_RAY32 needs a triangle accel and 16-byte aligned rays");
      return NRT_ERR_INVALID;
    }
    Aos32Rays r32{reinterpret_cast<const float4 *>(d_rays)};
    if (flags & NRT_TRAVERSE_CONFORMANCE)
      return launch_conf<Aos32Rays, false>(a, r32, n, d_hits, d_mask, opt, flags, nullptr, s);
    const StoreHitsEpilogue epi{d_hits, d_mask};
    if (flags & NRT_TRAVERSE_ANY_HIT)
      return launch_fast3_coherent<Aos32Rays, false>(a, r32, n, AnyHit<StoreHitsEpilogue>(epi), opt, flags, nullptr, nullptr, s,
                                                     cursor);
    return launch_fast3_coherent<Aos32Rays, false>(a, r32, n, epi, opt, flags, nullptr, nullptr, s, cursor);
  }
  if (a->prim_kind != 0) return launch_traverse_prims(a, d_rays, n, d_hits, d_mask, opt, flags, s);  // spheres ...
  AosRays r{d_rays};
  if (flags & NRT_TRAVERSE_CONFORMANCE) return launch_conf<AosRays, false>(a, r, n, d_hits, d_mask, opt, flags, nullptr, s);
  if (flags & NRT_TRAVERSE_ANY_HIT)  // occlusion query: default policy only
    return launch_fast3_coherent<AosRays, false>(a, r, n, AnyHit<StoreHitsEpilogue>(StoreHitsEpilogue{d_hits, d_mask}), opt,
                                                 flags, nullptr, nullptr, s, cursor);
  return launch_fast<AosRays, false>(a, r, n, d_hits, d_mask, opt, flags, nullptr, s, nullptr, cursor);
}

int launch_traverse_soa(const Accel *a, const float4 *d_org_tmin, const float4 *d_dir_tmax, size_t n,
                        Hit16 *d_hits, const TraceOptions16 &opt, uint32_t flags, cudaStream_t s) {
  if (n == 0) return NRT_OK;
  SoaRays r{d_org_tmin, d_dir_tmax};
  if (flags & NRT_TRAVERSE_CONFORMANCE) return launch_conf<SoaRays, false>(a, r, n, d_hits, nullptr, opt, flags, nullptr, s);
  return launch_fast<SoaRays, false>(a, r, n, d_hits, nullptr, opt, flags, nullptr, s);
}

// `capacity` bounds the count stored at d_count (grid sizing only).
int launch_traverse_soa_devcount(const Accel *a, const float4 *d_org_tmin, const float4 *d_dir_tmax,
                                 const unsigned long long *d_count, size_t capacity, Hit16 *d_hits,
                                 const TraceOptions16 &opt, uint32_t flags, cudaStream_t s) {
  if (capacity == 0) return NRT_OK;
  SoaRays r{d_org_tmin, d_dir_tmax};
  if (flags & NRT_TRAVERSE_CONFORMANCE)
    return launch_conf<SoaRays, false>(a, r, capacity, d_hits, nullptr, opt, flags, nullptr, s, d_count);
  return launch_fast<SoaRays, false>(a, r, capacity, d_hits, nullptr, opt, flags, nullptr, s, d_count);
}

// Fused wavefront launches (render.cu): the retire step spawns the AO ray / accumulates visibility.
template <class Epi, class P = DefaultPolicy, class Rays = SoaRays>
static int launch_fused(const Accel *a, Rays rays, size_t n, const unsigned long long *n_ptr, Epi epi,
                        const TraceOptions16 &opt, uint32_t flags, cudaStream_t s) {
  if (n == 0) return NRT_OK;
  return launch_fast3_any<Rays, false, P>(a, rays, n, epi, opt, flags, nullptr, n_ptr, s);
}

template <int DEPTH>
static cudaError_t launch_packet(const Accel *a, CameraRays rays, size_t n, const PrimaryToAoEpilogue &epi,
                                 const TraceOptions16 &opt, uint32_t flags, unsigned long long *cursor, cudaStream_t s) {
  typedef CameraUnits<CameraPacketPolicy::kRays> Units;
  const Units units(epi.p);
  const size_t n_units = units.count(n);  // one warp each
  const size_t warps_per_block = kTraverseBlock / 32;
  size_t grid = (size_t)device_sm_count(a->device) * CameraPacketPolicy::kMinBlocks;
  const size_t need_blocks = (n_units + warps_per_block - 1) / warps_per_block;
  if (grid > need_blocks) grid = need_blocks;
  traverse_packet_kernel<CameraRays, Units, DEPTH, CameraPacketPolicy, PrimaryToAoEpilogue>
      <<<(unsigned)grid, kTraverseBlock, 0, s>>>(a->d_pair_rel, a->d_tris_rel, rays, units, n_units, n, epi, opt, flags,
                                                 cursor);
  return cudaGetLastError();
}

// the packet walk, with a cursor of the accel's ring (as launch_fast3_any); the caller has made the camera-relative copies
static int launch_packet_any(const Accel *a, CameraRays rays, size_t n, const PrimaryToAoEpilogue &epi,
                             const TraceOptions16 &opt, uint32_t flags, cudaStream_t s) {
  if (!a->d_pair_rel || !a->d_tris_rel) {
    set_error("traverse: this accel has no camera-relative traversal layout");
    return NRT_ERR_INVALID;
  }
  return a->ring.run(s, [&](uint32_t k) {
    unsigned long long *cursor = reinterpret_cast<unsigned long long *>(a->d_counters) + 16 + k;
    NRT_CUDA(cudaMemsetAsync(cursor, 0, sizeof(unsigned long long), s));
    const cudaError_t e = needs_deep_stack(a) ? launch_packet<512>(a, rays, n, epi, opt, flags, cursor, s)
                                              : launch_packet<64>(a, rays, n, epi, opt, flags, cursor, s);
    NRT_CUDA(e);
    return NRT_OK;
  });
}

// Camera rays, generated inside the kernel (no generator kernel, no primary queue).  On the PairNode path they read
// camera-relative copies of the nodes and triangles while the originals and the copies together stay well inside one
// half of the L2 (kCameraRelMaxBytes); the caller orders `s` after every earlier pass that may still read the copies.
// Over the copies, each 8x4-pixel packet walks the tree as one warp (traverse_packet_kernel).  The launches over the
// accel's own arrays keep the per-lane walk: their trees are the ones too big for the copies, and on the 1 M terrain
// (PairNodes, 86 MB of nodes and triangles against the 50 MB L2) the pass took 26 % longer with the packet walk.
int launch_traverse_camera_fused(Accel *a, const Wave &w, const nrt_ao_params &p, unsigned long long slot0, size_t count,
                                 const float4 *d_face_n, float *d_accum, unsigned long long *d_wave_counters,
                                 const TraceOptions16 &opt, uint32_t flags, cudaStream_t s) {
  PrimaryToAoEpilogue epi{p, w, d_face_n, d_accum, d_wave_counters};
  if (count == 0) return NRT_OK;
  if (a->n_wide * sizeof(PairNode) > kPair128MaxBytes)
    return launch_fast3_any<CameraRaysAbs, false, IncoherentCameraPolicy>(a, CameraRaysAbs(p, slot0), count, epi, opt, flags,
                                                                          nullptr, nullptr, s);
  if (2 * (a->n_wide * sizeof(PairNode) + (size_t)a->n_prims * sizeof(TriCM)) > kCameraRelMaxBytes)
    return launch_fast3_any<CameraRaysAbs, false, CameraPolicy>(a, CameraRaysAbs(p, slot0), count, epi, opt, flags, nullptr,
                                                                nullptr, s);
  const int rc = camera_relative_layout(a, p.cam, s);
  if (rc != NRT_OK) return rc;
  return launch_packet_any(a, CameraRays(p, slot0), count, epi, opt, flags, s);
}

int launch_traverse_ao_fused(const Accel *a, const Wave &w, const unsigned long long *d_count, size_t capacity,
                             float *d_accum, unsigned long long *d_totals, const TraceOptions16 &opt, uint32_t flags,
                             cudaStream_t s) {
  AoAccumulateEpilogue epi{w.ao_pix, d_accum, d_totals};
  if (flags & NRT_TRAVERSE_ANY_HIT)
    return launch_fused<AnyHit<AoAccumulateEpilogue>, IncoherentPolicy>(a, SoaRays{w.ao_org_tmin, w.ao_dir_tmax}, capacity, d_count,
                                                                        AnyHit<AoAccumulateEpilogue>(epi), opt, flags, s);
  return launch_fused<AoAccumulateEpilogue, IncoherentPolicy>(a, SoaRays{w.ao_org_tmin, w.ao_dir_tmax}, capacity, d_count, epi,
                                                              opt, flags, s);
}

int launch_traverse_path_radiance(const Accel *a, const PathShadeEpilogue &epi, const unsigned long long *d_count,
                                  size_t capacity, const TraceOptions16 &opt, uint32_t flags, cudaStream_t s) {
  return launch_fused<PathShadeEpilogue, PathRadiancePolicy>(
      a, SoaRays{epi.q.org_tmin[epi.in], epi.q.dir_tmax[epi.in]}, capacity, d_count, epi, opt, flags, s);
}

// the lightmap bake's bounces 1 and up (lightmap.cu): the path radiance launch with the texel slot map
int launch_traverse_lightmap_radiance(const Accel *a, const LightmapShadeEpilogue &epi, const unsigned long long *d_count,
                                      size_t capacity, const TraceOptions16 &opt, uint32_t flags, cudaStream_t s) {
  return launch_fused<LightmapShadeEpilogue, PathRadiancePolicy>(
      a, SoaRays{epi.q.org_tmin[epi.in], epi.q.dir_tmax[epi.in]}, capacity, d_count, epi, opt, flags, s);
}

int launch_traverse_path_shadow(const Accel *a, const PathQueues &q, const unsigned long long *d_count,
                                size_t capacity, float *d_accum, const TraceOptions16 &opt, uint32_t flags,
                                cudaStream_t s) {
  ShadowAccumulateEpilogue epi{q.sh_contrib_pix, d_accum};
  if (flags & NRT_TRAVERSE_ANY_HIT)
    return launch_fused<AnyHit<ShadowAccumulateEpilogue>, IncoherentPolicy>(a, SoaRays{q.sh_org_tmin, q.sh_dir_tmax}, capacity,
                                                                            d_count, AnyHit<ShadowAccumulateEpilogue>(epi), opt,
                                                                            flags, s);
  return launch_fused<ShadowAccumulateEpilogue, IncoherentPolicy>(a, SoaRays{q.sh_org_tmin, q.sh_dir_tmax}, capacity, d_count,
                                                                  epi, opt, flags, s);
}

// Texel cast (bake.cu): the production walk stores each texel's record through its payload; the conformance walk
// writes records by ray index to d_by_ray, which the caller scatters to the flipped texels.
int launch_traverse_texels(const Accel *a, const TexelRays &rays, size_t n, const TexelStore &store, Hit16 *d_by_ray,
                           uint32_t flags, cudaStream_t s) {
  if (n == 0) return NRT_OK;
  const TraceOptions16 opt = default_trace_options();
  if (flags & NRT_TRAVERSE_CONFORMANCE)
    return launch_conf<TexelRays, false>(a, rays, n, d_by_ray, nullptr, opt, flags, nullptr, s);
  return launch_fast3_coherent<TexelRays, false>(a, rays, n, TexelStoreEpilogue{store}, opt, flags, nullptr, nullptr, s);
}

// AO rays of the bake, generated at fetch
int launch_traverse_bake(const Accel *a, const BakeAoRays &rays, size_t n, float *d_accum, unsigned long long *d_occluded,
                         uint32_t flags, cudaStream_t s) {
  if (n == 0) return NRT_OK;
  const TraceOptions16 opt = default_trace_options();
  const BakeAccumulateEpilogue epi{d_accum, d_occluded};
  if (flags & NRT_TRAVERSE_ANY_HIT)
    return launch_fast3_any<BakeAoRays, false, IncoherentPolicy>(a, rays, n, AnyHit<BakeAccumulateEpilogue>(epi), opt,
                                                                 flags, nullptr, nullptr, s);
  return launch_fast3_any<BakeAoRays, false, IncoherentPolicy>(a, rays, n, epi, opt, flags, nullptr, nullptr, s);
}

// The conformance walk with a retire step: the reference-order walk of traverse_conformance_kernel, then the
// epilogue, called by every lane of the block (lanes past n retire nothing).
template <class Rays, class Epi>
__global__ void __launch_bounds__(128)
    traverse_conformance_epi_kernel(const Node40 *__restrict__ nodes, const PackedTri *__restrict__ tris, Rays rays,
                                    size_t n, Epi epi, TraceOptions16 opt, uint32_t flags,
                                    const unsigned long long *n_ptr) {
  if (n_ptr) n = (size_t)*n_ptr;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  Best best;
  best.t = 0.0f;
  best.u = 0.0f;
  best.v = 0.0f;
  best.prim = 0xFFFFFFFFu;
  float max_t = 0.0f;
  if (i < n) {
    float ox, oy, oz, dx, dy, dz, min_t;
    rays.load(i, ox, oy, oz, dx, dy, dz, min_t, max_t);
    RayCtx c;
    setup_ray(c, ox, oy, oz, dx, dy, dz, min_t, (flags & NRT_TRAVERSE_CPP03_INVERSE) != 0);
    best.t = max_t;
    reference_walk(nodes, c, min_t, max_t, PackedTriLeaf{tris, c, opt, best});
  }
  epi(i < n, i, best.t, best.u, best.v, best.prim, max_t, nullptr);
}

template <class Rays, class Epi, class P>
static int launch_bdpt(const Accel *a, const Rays &rays, const Epi &epi, const unsigned long long *d_count,
                       size_t capacity, uint32_t flags, cudaStream_t s) {
  if (capacity == 0) return NRT_OK;
  const TraceOptions16 opt = default_trace_options();
  if (flags & NRT_TRAVERSE_CONFORMANCE) {
    traverse_conformance_epi_kernel<Rays, Epi><<<(unsigned)((capacity + 127) / 128), 128, 0, s>>>(
        a->d_nodes, a->d_tris, rays, capacity, epi, opt, flags, d_count);
    NRT_CUDA(cudaGetLastError());
    return NRT_OK;
  }
  return launch_fused<Epi, P, Rays>(a, rays, capacity, d_count, epi, opt, flags, s);
}

// Bidirectional path tracer (bdpt.cu): subpath bounces, whose retire step is raytrace's per-hit block (the path
// radiance launch's policy: a shading retire step), and the connection rays, whose retire step is calcG's test
// (incoherent rays, a light retire step).
int launch_traverse_bdpt_bounce(const Accel *a, const bd::BounceRays &rays, const bd::BounceEpilogue &epi,
                                const unsigned long long *d_count, size_t capacity, uint32_t flags, cudaStream_t s) {
  return launch_bdpt<bd::BounceRays, bd::BounceEpilogue, PathRadiancePolicy>(a, rays, epi, d_count, capacity, flags, s);
}

int launch_traverse_bdpt_connect(const Accel *a, const bd::ConnRays &rays, const bd::ConnEpilogue &epi,
                                 const unsigned long long *d_count, size_t capacity, uint32_t flags, cudaStream_t s) {
  return launch_bdpt<bd::ConnRays, bd::ConnEpilogue, IncoherentPolicy>(a, rays, epi, d_count, capacity, flags, s);
}

int launch_traverse_count(const Accel *a, const Ray36 *d_rays, size_t n, const TraceOptions16 &opt,
                          uint32_t flags, uint64_t *d_counts2, cudaStream_t s) {
  if (a->prim_kind != 0) {  // both counting walks test triangles: their counts would mean nothing on other kinds
    set_error("nrt_traverse_count_device / nrt_traverse_lane_stats_device: counting walks need a triangle accel");
    return NRT_ERR_INVALID;
  }
  NRT_CUDA(cudaMemsetAsync(d_counts2, 0, 16 * sizeof(uint64_t), s));  // [0] boxes, [1] prims, [2..15] lane statistics
  if (n == 0) return NRT_OK;
  AosRays r{d_rays};
  unsigned long long *cnt = reinterpret_cast<unsigned long long *>(d_counts2);
  flags = (flags & ~kCountRootIsLeaf) | (a->root_is_leaf ? kCountRootIsLeaf : 0u);
  if (flags & NRT_TRAVERSE_CONFORMANCE) return launch_conf<AosRays, true>(a, r, n, nullptr, nullptr, opt, flags, cnt, s);
  return launch_fast<AosRays, true>(a, r, n, nullptr, nullptr, opt, flags, cnt, s);
}

}  // namespace nrt
