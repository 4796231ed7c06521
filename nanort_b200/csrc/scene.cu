// Two-level scene: instances of bottom-level accels under a top-level tree (sm_90a, --fmad=false).
//
// Replaces (file:line in the reference tree):
//   nanosg::Node::Update                      examples/nanosg/nanosg.h:400-445   instance_setup_kernel
//   Matrix::Inverse / Mult / MultV            examples/nanosg/nanosg.h:92-222    mat_inverse / multv
//   XformBoundingBox                          examples/nanosg/nanosg.h:241-299   instance_setup_kernel
//   nanosg::Scene::Commit (top-level Build)   examples/nanosg/nanosg.h:706-755   nrt_scene_commit (build.cu / build_ref.cu
//                                                                                 over box primitives)
//   BVHAccel::ListNodeIntersections +
//   TestLeafNodeIntersections                 nanort.h:2558-2692                 scene_list_kernel
//   NodeBBoxIntersector::Intersect            examples/nanosg/nanosg.h:597-637   raw_box() (nodehits.cuh)
//   nanosg::Scene::Traverse                   examples/nanosg/nanosg.h:779-875   scene_list_kernel / scene_unified_kernel
//
// Two kernels.  scene_list_kernel is the reference's algorithm verbatim, one thread per ray: collect the (at most 64)
// nearest instance boxes in a max-heap that follows libstdc++'s push_heap / pop_heap sift rules, visit them nearest
// first, walk each instance's nanort-layout tree in the reference's order.  scene_unified_kernel is the production
// path: persistent warps, one pass over the top-level tree (sub-trees that start behind the current nearest hit are
// skipped), each candidate instance traversed with the 64-byte child-pair WideNodes (common.cuh).
// Both compute the local ray, the world hit point and the world distance with the reference's operation order, so a
// hit record is bit-identical to the reference's whenever both pick the same (instance, triangle); the pick itself
// can differ only between candidates at exactly the same world distance.  A ray that pierces more than 64 instance
// boxes (the reference then drops the farthest boxes) or whose direction is not unit length (the reference's answer
// then depends on its visiting order) is re-run by the list kernel.
#include <float.h>
#include <math_constants.h>

#include <algorithm>
#include <cstring>
#include <new>
#include <vector>

#include "../../include/nanort_b200_scene_path.h"
#include "common.cuh"
#include "scene.cuh"
#include "trav_common.cuh"
#include "nodehits.cuh"

namespace nrt {

namespace {

constexpr int kNoLeaf = kEmptyLeaf;

// ---- instance setup ------------------------------------------------------------------------------------------
// Cramer's-rule inverse in the reference's operation order.  Pair products, then for every element
// (p0 s0 + p1 s1 + p2 s2) - (q0 s0' + q1 s1' + q2 s2'); the tables hold {pair index, source index}.  The very last
// term of element 15 reads source 0 where the rule has source 10 -- the reference does (nanosg.h:173); only m[3][3]
// depends on it and MultV never reads that entry.
__constant__ uint8_t kPairs[2][12][2] = {
    {{10, 15}, {11, 14}, {9, 15}, {11, 13}, {9, 14}, {10, 13}, {8, 15}, {11, 12}, {8, 14}, {10, 12}, {8, 13}, {9, 12}},
    {{2, 7}, {3, 6}, {1, 7}, {3, 5}, {1, 6}, {2, 5}, {0, 7}, {3, 4}, {0, 6}, {2, 4}, {0, 5}, {1, 4}}};
__constant__ uint8_t kCof[16][2][3][2] = {
    {{{0, 5}, {3, 6}, {4, 7}}, {{1, 5}, {2, 6}, {5, 7}}},
    {{{1, 4}, {6, 6}, {9, 7}}, {{0, 4}, {7, 6}, {8, 7}}},
    {{{2, 4}, {7, 5}, {10, 7}}, {{3, 4}, {6, 5}, {11, 7}}},
    {{{5, 4}, {8, 5}, {11, 6}}, {{4, 4}, {9, 5}, {10, 6}}},
    {{{1, 1}, {2, 2}, {5, 3}}, {{0, 1}, {3, 2}, {4, 3}}},
    {{{0, 0}, {7, 2}, {8, 3}}, {{1, 0}, {6, 2}, {9, 3}}},
    {{{3, 0}, {6, 1}, {11, 3}}, {{2, 0}, {7, 1}, {10, 3}}},
    {{{4, 0}, {9, 1}, {10, 2}}, {{5, 0}, {8, 1}, {11, 2}}},
    {{{0, 13}, {3, 14}, {4, 15}}, {{1, 13}, {2, 14}, {5, 15}}},
    {{{1, 12}, {6, 14}, {9, 15}}, {{0, 12}, {7, 14}, {8, 15}}},
    {{{2, 12}, {7, 13}, {10, 15}}, {{3, 12}, {6, 13}, {11, 15}}},
    {{{5, 12}, {8, 13}, {11, 14}}, {{4, 12}, {9, 13}, {10, 14}}},
    {{{2, 10}, {5, 11}, {1, 9}}, {{4, 11}, {0, 9}, {3, 10}}},
    {{{8, 11}, {0, 8}, {7, 10}}, {{6, 10}, {9, 11}, {1, 8}}},
    {{{6, 9}, {11, 11}, {3, 8}}, {{10, 11}, {2, 8}, {7, 9}}},
    {{{10, 10}, {4, 8}, {9, 9}}, {{8, 9}, {11, 0}, {5, 8}}}};

__device__ void mat_inverse(float m[16]) {  // m[4 r + c], in place
  float src[16], pr[12], out[16];
  for (int i = 0; i < 4; i++)
    for (int c = 0; c < 4; c++) src[i + 4 * c] = m[4 * i + c];
  for (int half = 0; half < 2; half++) {
    for (int k = 0; k < 12; k++) pr[k] = src[kPairs[half][k][0]] * src[kPairs[half][k][1]];
    for (int e = 8 * half; e < 8 * half + 8; e++) {
      float acc[2];
      for (int sgn = 0; sgn < 2; sgn++) {
        const uint8_t(*t)[2] = kCof[e][sgn];
        acc[sgn] = (pr[t[0][0]] * src[t[0][1]] + pr[t[1][0]] * src[t[1][1]]) + pr[t[2][0]] * src[t[2][1]];
      }
      out[e] = acc[0] - acc[1];
    }
  }
  float det = ((src[0] * out[0] + src[1] * out[1]) + src[2] * out[2]) + src[3] * out[3];
  det = 1.0f / det;
  for (int e = 0; e < 16; e++) m[e] = out[e] * det;
}

__device__ __forceinline__ Mat43 to_mat43(const float m[16]) {
  Mat43 r;
  r.a = make_float4(m[0], m[1], m[2], m[4]);
  r.b = make_float4(m[5], m[6], m[8], m[9]);
  r.c = make_float4(m[10], m[12], m[13], m[14]);
  return r;
}

// (b < a) ? b : a  and  (a < b) ? b : a : std::min / std::max as XformBoundingBox calls them
__device__ __forceinline__ float std_min(float a, float b) { return (b < a) ? b : a; }
__device__ __forceinline__ float std_max(float a, float b) { return (a < b) ? b : a; }

struct InstanceIn {  // host -> device
  float xform[16];
  float lbmin[3], lbmax[3];
  const float *verts;
  const WideNode *wide;
  const PackedTri *tris;
  const Node40 *nodes;
  const uint32_t *faces;
};

// Node::Update for scene roots: xform = identity x local; world box; inverse; inverse of the 3x3 part.
// state76 (optional): the reference's member layout, see nrt_scene_instance_state.
__global__ void instance_setup_kernel(const InstanceIn *__restrict__ in, uint32_t n, InstanceDev *__restrict__ out,
                                      float *__restrict__ boxes6, float *__restrict__ state76) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const InstanceIn I = in[i];
  float xf[16];
  // Matrix::Mult(xform, identity, local): dst[i][j] = sum_k parent[k][j] * local[i][k], accumulated from 0
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) {
      float acc = 0.0f;
      for (int k = 0; k < 4; k++) acc += (k == c ? 1.0f : 0.0f) * I.xform[4 * r + k];
      xf[4 * r + c] = acc;
    }
  const Mat43 X = to_mat43(xf);
  float bmin[3], bmax[3];
  for (int c = 0; c < 8; c++) {
    float x, y, z;
    multv(X, (c & 1) ? I.lbmax[0] : I.lbmin[0], (c & 2) ? I.lbmax[1] : I.lbmin[1], (c & 4) ? I.lbmax[2] : I.lbmin[2],
          x, y, z);
    if (c == 0) {
      bmin[0] = bmax[0] = x;
      bmin[1] = bmax[1] = y;
      bmin[2] = bmax[2] = z;
    } else {
      bmin[0] = std_min(x, bmin[0]);
      bmin[1] = std_min(y, bmin[1]);
      bmin[2] = std_min(z, bmin[2]);
      bmax[0] = std_max(x, bmax[0]);
      bmax[1] = std_max(y, bmax[1]);
      bmax[2] = std_max(z, bmax[2]);
    }
  }
  float inv[16], inv33[16];
  for (int e = 0; e < 16; e++) inv[e] = inv33[e] = xf[e];
  mat_inverse(inv);
  inv33[12] = inv33[13] = inv33[14] = 0.0f;
  mat_inverse(inv33);
  InstanceDev o;
  o.inv = to_mat43(inv);
  o.inv33 = to_mat43(inv33);
  o.xf = X;
  for (int k = 0; k < 3; k++) {
    o.bmin[k] = bmin[k];
    o.bmax[k] = bmax[k];
    boxes6[6 * (size_t)i + k] = bmin[k];
    boxes6[6 * (size_t)i + 3 + k] = bmax[k];
  }
  o.verts = I.verts;
  o.wide = I.wide;
  o.tris = I.tris;
  o.nodes = I.nodes;
  o.faces = I.faces;
  out[i] = o;
  if (state76) {
    float *s = state76 + 76 * (size_t)i;
    for (int e = 0; e < 16; e++) {
      s[e] = xf[e];
      s[16 + e] = inv[e];
      s[32 + e] = inv33[e];
      s[48 + 4 * (e % 4) + e / 4] = inv33[e];  // transpose
    }
    for (int k = 0; k < 3; k++) {
      s[64 + k] = I.lbmin[k];
      s[67 + k] = I.lbmax[k];
      s[70 + k] = bmin[k];
      s[73 + k] = bmax[k];
    }
  }
}

// ---- shared per-ray pieces ------------------------------------------------------------------------------------
// world distance of a local hit: P_local = o + t d; P = P_local . xform; t_world = |P - org|  (nanosg.h:832-848)
__device__ __forceinline__ float world_hit(const Mat43 &xf, const WorldRay &w, float lox, float loy, float loz,
                                           float ldx, float ldy, float ldz, float t, float &px, float &py, float &pz) {
  const float lx = lox + t * ldx, ly = loy + t * ldy, lz = loz + t * ldz;
  multv(xf, lx, ly, lz, px, py, pz);
  const float ax = px - w.ox, ay = py - w.oy, az = pz - w.oz;
  return sqrtf((ax * ax + ay * ay) + az * az);
}

struct SceneBest {
  float t, u, v, px, py, pz;
  uint32_t prim, node;
};

__device__ __forceinline__ void store_scene_hit(SceneHit32 *hits, uint8_t *mask, size_t i, const SceneBest &b,
                                                bool hit, float max_t) {
  float4 r0, r1;
  if (hit) {
    r0 = make_float4(b.u, b.v, b.t, __uint_as_float(b.prim));
    r1 = make_float4(__uint_as_float(b.node), b.px, b.py, b.pz);
  } else {
    r0 = make_float4(0.0f, 0.0f, max_t, __uint_as_float(0xFFFFFFFFu));
    r1 = make_float4(__uint_as_float(0xFFFFFFFFu), 0.0f, 0.0f, 0.0f);
  }
  float4 *o = reinterpret_cast<float4 *>(hits + i);
  o[0] = r0;
  o[1] = r1;
  if (mask) mask[i] = hit ? 1 : 0;
}

// Scene::Traverse never forwards its cull_back_face flag (nanosg.h:800-829): both kernels trace the instances with
// default_trace_options().
__global__ void __launch_bounds__(128)
    scene_list_kernel(SceneDev sc, const Ray36 *__restrict__ rays, size_t n, const uint32_t *__restrict__ subset,
                      const unsigned long long *__restrict__ n_subset, SceneHit32 *__restrict__ hits,
                      uint8_t *__restrict__ mask, uint32_t flags) {
  if (n_subset) n = (size_t)*n_subset;
  const bool cpp03 = (flags & NRT_TRAVERSE_CPP03_INVERSE) != 0;
  const TraceOptions16 opt = default_trace_options();
  for (size_t job = (size_t)blockIdx.x * blockDim.x + threadIdx.x; job < n; job += (size_t)gridDim.x * blockDim.x) {
    const size_t i = subset ? (size_t)subset[job] : job;
    const WorldRay w = load_world(rays, i);
    RayCtx c;
    setup_ray(c, w.ox, w.oy, w.oz, w.dx, w.dy, w.dz, w.min_t, cpp03);
    NodeHitHeap heap;
    collect_node_hits(sc.top_nodes, sc.top_idx, [&](uint32_t id) { return sc.inst[id].bmin; }, w, c, kMaxNodeHits,
                      heap);

    SceneBest best;
    best.t = FLT_MAX;
    best.node = 0xFFFFFFFFu;
    bool has_hit = false;
    for (int k = 0; k < heap.n; k++) {
      if (best.t < heap.t[k]) continue;  // early cull (nanosg.h:803-807)
      const uint32_t id = heap.id[k];
      const InstanceDev *I = sc.inst + id;
      const Mat43 minv = load_mat(&I->inv), minv33 = load_mat(&I->inv33);
      float lox, loy, loz, ldx, ldy, ldz;
      multv(minv, w.ox, w.oy, w.oz, lox, loy, loz);
      multv(minv33, w.dx, w.dy, w.dz, ldx, ldy, ldz);
      RayCtx lc;
      setup_ray(lc, lox, loy, loz, ldx, ldy, ldz, 0.0f, cpp03);
      Best lb;
      lb.t = FLT_MAX;
      lb.u = 0.0f;
      lb.v = 0.0f;
      lb.prim = 0xFFFFFFFFu;
      reference_walk(I->nodes, lc, 0.0f, FLT_MAX, PackedTriLeaf{I->tris, lc, opt, lb});
      if (!(lb.t < FLT_MAX)) continue;
      const Mat43 mxf = load_mat(&I->xf);
      float px, py, pz;
      const float tw = world_hit(mxf, w, lox, loy, loz, ldx, ldy, ldz, lb.t, px, py, pz);
      if (tw < best.t) {
        best.t = tw;
        best.u = lb.u;
        best.v = lb.v;
        best.prim = lb.prim;
        best.node = id;
        best.px = px;
        best.py = py;
        best.pz = pz;
        has_hit = true;
      }
    }
    store_scene_hit(hits, mask, i, best, has_hit, w.max_t);
  }
}

constexpr int kSceneBlock = 128;

// ---- production kernel, unified walk ------------------------------------------------------------------------------
// The top-level tree is laid out as the same 64-byte child-pair nodes as every instance tree, so that ONE node step
// serves lanes that walk the top level and lanes that are inside an instance: the per-lane ray constants `c` are the
// world ray's or the local ray's, the per-lane base pointers select the tree, and a single per-lane stack holds the
// top-level entries, a sentinel, and the instance's entries above it.  A top-level leaf is an instance slot: the
// reference's box test decides whether the lane enters (transform the ray, push the sentinel, start at the
// instance's root); popping the sentinel ends the visit (world distance of the local hit, restore the world
// constants from shared memory).  Lanes never wait for each other's instance visits.
//   top-level step: pass iff the widened slab test over [min_t, max_t] passes (nanort.h:2284-2325) and the
//                   unclamped entry distance is not behind the nearest hit (every instance box below starts later)
//   instance step:  pass iff the slab test over [0, best.t] passes; stack entries are culled against best.t
constexpr int kUnifiedMinBlocks = 8;  // 64 registers
constexpr int kUnifiedRefillMin = 16;  // lanes that must have retired before the warp fetches new rays
constexpr int kUnifiedNodeExit = 8;    // leave the node phase when fewer lanes than this descend
constexpr int kSentinel = (int)0x80000001;  // ~kSentinel = 0x7FFFFFFE is never a slot

__device__ __forceinline__ bool is_leaf_ref(int r) { return r < 0 && r != kNoLeaf && r != kSentinel; }

// slab test that also returns the entry distance before the clamp to lo_clip
__device__ __forceinline__ bool slab_e(const RayCtx &c, float lox, float loy, float loz, float hix, float hiy,
                                       float hiz, float lo_clip, float hi_clip, float &te) {
  const float nx = c.sx ? hix : lox, fx = c.sx ? lox : hix;
  const float ny = c.sy ? hiy : loy, fy = c.sy ? loy : hiy;
  const float nz = c.sz ? hiz : loz, fz = c.sz ? loz : hiz;
  const float tnx = (nx - c.ox) * c.ix;
  const float tny = (ny - c.oy) * c.iy;
  const float tnz = (nz - c.oz) * c.iz;
  const float tfx = ((fx - c.ox) * c.ix) * 1.00000024f;
  const float tfy = ((fy - c.oy) * c.iy) * 1.00000024f;
  const float tfz = ((fz - c.oz) * c.iz) * 1.00000024f;
  te = fmaxf(tnz, fmaxf(tny, tnx));  // NaN operands drop out like in slab(); all-NaN stays NaN
  const float tmin = fmaxf(te, lo_clip);
  const float tmax = fminf(tfz, fminf(tfy, fminf(tfx, hi_clip)));
  return tmin <= tmax;
}

template <int LOCAL_DEPTH, int MINB>
__global__ void __launch_bounds__(kSceneBlock, MINB)
    scene_unified_kernel(SceneDev sc, const Ray36 *__restrict__ rays, size_t n, SceneHit32 *__restrict__ hits,
                         uint8_t *__restrict__ mask, uint32_t flags, unsigned long long *cursor,
                         uint32_t *__restrict__ overflow, unsigned long long *overflow_count) {
  __shared__ float wsave[16 * kSceneBlock];  // world-ray constants of lanes that are inside an instance
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const unsigned lt_mask = (1u << lane) - 1u;
  const bool cpp03 = (flags & NRT_TRAVERSE_CPP03_INVERSE) != 0;
  const TraceOptions16 opt = default_trace_options();

  long long ray_idx = -1;
  bool exhausted = false;
  WorldRay w;
  SceneBest nearest;
  uint32_t n_boxes = 0;
  int inst = -1;
  RayCtx c;
  Best best;
  const WideNode *wide = sc.top_wide;
  const PackedTri *tris = sc.top_slots;
  uint2 lstk[LOCAL_DEPTH];
  int sp = 0, cur = kNoLeaf, leaf = kNoLeaf;

  auto push = [&](int ref, float t) {
    if (sp < LOCAL_DEPTH) lstk[sp] = make_uint2((uint32_t)ref, __float_as_uint(t));
    sp++;
  };
  // next entry that does not start behind the current bound (instance: best.t, top level: nearest.t); the sentinel
  // is stored with -inf and always comes back
  auto pop = [&]() -> int {
    const float bound = inst >= 0 ? best.t : nearest.t;
    while (sp > 0) {
      --sp;
      if (sp >= LOCAL_DEPTH) continue;
      const uint2 e = lstk[sp];
      if (!(__uint_as_float(e.y) > bound)) return (int)e.x;
    }
    return kNoLeaf;
  };
  auto save_world = [&]() {
    float *q = wsave + tid;
    q[0 * kSceneBlock] = c.ox, q[1 * kSceneBlock] = c.oy, q[2 * kSceneBlock] = c.oz;
    q[3 * kSceneBlock] = c.ix, q[4 * kSceneBlock] = c.iy, q[5 * kSceneBlock] = c.iz;
    q[6 * kSceneBlock] = c.Sx, q[7 * kSceneBlock] = c.Sy, q[8 * kSceneBlock] = c.Sz;
    q[9 * kSceneBlock] = c.t_min;
    q[10 * kSceneBlock] = __int_as_float(c.sx | (c.sy << 1) | (c.sz << 2) | (c.kx << 4) | (c.ky << 6) | (c.kz << 8));
  };
  auto restore_world = [&]() {
    const float *q = wsave + tid;
    c.ox = q[0 * kSceneBlock], c.oy = q[1 * kSceneBlock], c.oz = q[2 * kSceneBlock];
    c.ix = q[3 * kSceneBlock], c.iy = q[4 * kSceneBlock], c.iz = q[5 * kSceneBlock];
    c.Sx = q[6 * kSceneBlock], c.Sy = q[7 * kSceneBlock], c.Sz = q[8 * kSceneBlock];
    c.t_min = q[9 * kSceneBlock];
    const int b = __float_as_int(q[10 * kSceneBlock]);
    c.sx = b & 1, c.sy = (b >> 1) & 1, c.sz = (b >> 2) & 1;
    c.kx = (b >> 4) & 3, c.ky = (b >> 6) & 3, c.kz = (b >> 8) & 3;
  };

  for (;;) {
    // ---- replace retired rays
    const unsigned dead = __ballot_sync(FULL_MASK, ray_idx < 0);
    if (dead != 0u && !exhausted && (dead == FULL_MASK || __popc(dead) >= kUnifiedRefillMin)) {
      const int cnt = __popc(dead);
      const int leader = __ffs(dead) - 1;
      unsigned long long base = 0;
      if (lane == leader) base = atomicAdd(cursor, (unsigned long long)cnt);
      base = __shfl_sync(FULL_MASK, base, leader);
      if (base + (unsigned long long)cnt >= (unsigned long long)n) exhausted = true;
      if (ray_idx < 0) {
        const unsigned long long mine = base + (unsigned long long)__popc(dead & lt_mask);
        if (mine < (unsigned long long)n) {
          w = load_world(rays, (size_t)mine);
          setup_ray(c, w.ox, w.oy, w.oz, w.dx, w.dy, w.dz, w.min_t, cpp03);
          nearest.t = FLT_MAX;
          nearest.node = 0xFFFFFFFFu;
          best.t = FLT_MAX;
          ray_idx = (long long)mine;
          n_boxes = 0;
          inst = -1;
          wide = sc.top_wide;
          tris = sc.top_slots;
          sp = 0;
          cur = range_has_nan(w.min_t, w.max_t) ? kNoLeaf : 0;
          leaf = kNoLeaf;
          // Scene::Traverse compares world DISTANCES of hits with ray PARAMETERS of box entries (nanosg.h:803, 848):
          // for a direction that is not unit length its answer depends on the visiting order, which only the list
          // kernel reproduces; such a ray is handed over like a > 64-box ray
          const float len2 = (w.dx * w.dx + w.dy * w.dy) + w.dz * w.dz;
          if (!(fabsf(len2 - 1.0f) <= 1e-5f)) {
            cur = kNoLeaf;
            n_boxes = (uint32_t)kMaxNodeHits + 1u;
          }
        }
      }
    }
    if (__all_sync(FULL_MASK, ray_idx < 0)) {
      if (exhausted) break;
      continue;
    }

    // ---- node steps (top level and instances alike)
    for (;;) {
      const unsigned desc = __ballot_sync(FULL_MASK, cur >= 0);
      if (desc == 0u) break;
      if (__popc(desc) < kUnifiedNodeExit && __any_sync(FULL_MASK, leaf != kNoLeaf || cur == kSentinel)) break;
      if (cur >= 0) {
        const float4 *p = reinterpret_cast<const float4 *>(wide + cur);
        const float4 q0 = __ldg(p), q1 = __ldg(p + 1), q2 = __ldg(p + 2);
        const int4 q3 = __ldg(reinterpret_cast<const int4 *>(p + 3));
        const bool in_inst = inst >= 0;
        const float lo_clip = in_inst ? 0.0f : w.min_t;
        const float hi_clip = in_inst ? best.t : w.max_t;
        const float bound = in_inst ? best.t : nearest.t;
        float t0, t1;
        bool h0 = slab_e(c, q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, lo_clip, hi_clip, t0);
        bool h1 = slab_e(c, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, lo_clip, hi_clip, t1);
        // an empty child (the second child of a root that is a leaf) never passes: its inverted box does pass when
        // the ray's origin is NaN, because slab_e drops NaN operands, and kNoLeaf as the next node inside an
        // instance would leave the lane there for ever
        h0 &= !(t0 > bound) && q3.x != kNoLeaf;
        h1 &= !(t1 > bound) && q3.y != kNoLeaf;
        const bool both = h0 & h1;
        const bool swap = t1 < t0;
        const int nearr = swap ? q3.y : q3.x;
        const int farr = swap ? q3.x : q3.y;
        if (both) push(farr, swap ? t0 : t1);
        int next = both ? nearr : (h0 ? q3.x : q3.y);
        if (!(h0 | h1)) next = pop();
        if (is_leaf_ref(next) && leaf == kNoLeaf) {  // postpone the first leaf, keep descending
          leaf = next;
          next = pop();
        }
        cur = next;
      }
    }

    // ---- leaves: triangles inside an instance, instance slots at the top level; then instance exits
    for (;;) {
      if (!__any_sync(FULL_MASK, leaf != kNoLeaf || cur == kSentinel)) break;
      if (leaf != kNoLeaf) {
        const float4 *t = reinterpret_cast<const float4 *>(tris + (size_t)(~leaf));
        if (inst >= 0) {
          for (;;) {
            const float4 a = __ldg(t), b = __ldg(t + 1), cc = __ldg(t + 2);
            tri_test2(c, opt, a, b, cc, best);
            if (__float_as_uint(b.w) != 0u) break;
            t += 3;
          }
          leaf = kNoLeaf;
        } else {
          const float4 a = __ldg(t), b = __ldg(t + 1);
          const int slot = ~leaf;
          leaf = kNoLeaf;
          if (__float_as_uint(b.w) == 0u) {  // more instances in this top-level leaf (depth-limit leaves only)
            if (cur != kNoLeaf) push(cur, -CUDART_INF_F);
            cur = ~(slot + 1);
          }
          // NodeBBoxIntersector::Intersect on the world box (nanosg.h:597-637)
          const float rix = 1.0f / w.dx, riy = 1.0f / w.dy, riz = 1.0f / w.dz;
          const bool sx = w.dx < 0.0f, sy = w.dy < 0.0f, sz = w.dz < 0.0f;
          const float tnx = ((sx ? b.x : a.x) - w.ox) * rix, tfx = ((sx ? a.x : b.x) - w.ox) * rix;
          const float tny = ((sy ? b.y : a.y) - w.oy) * riy, tfy = ((sy ? a.y : b.y) - w.oy) * riy;
          const float tnz = ((sz ? b.z : a.z) - w.oz) * riz, tfz = ((sz ? a.z : b.z) - w.oz) * riz;
          const float tmin = smax(tnz, smax(tny, tnx));
          const float tmax = smin(tfz, smin(tfy, tfx));
          if (tmin <= tmax) {
            n_boxes++;
            if (!(nearest.t < tmin)) {  // early cull (nanosg.h:803-807)
              const uint32_t id = __float_as_uint(a.w);
              const InstanceDev *I = sc.inst + id;
              const Mat43 minv = load_mat(&I->inv), minv33 = load_mat(&I->inv33);
              float lox, loy, loz, ldx, ldy, ldz;
              multv(minv, w.ox, w.oy, w.oz, lox, loy, loz);
              multv(minv33, w.dx, w.dy, w.dz, ldx, ldy, ldz);
              if (cur != kNoLeaf) push(cur, -CUDART_INF_F);  // what this lane was about to do at the top level
              push(kSentinel, -CUDART_INF_F);
              save_world();
              setup_ray(c, lox, loy, loz, ldx, ldy, ldz, 0.0f, cpp03);
              best.t = FLT_MAX;
              best.u = 0.0f;
              best.v = 0.0f;
              best.prim = 0xFFFFFFFFu;
              wide = I->wide;
              tris = I->tris;
              inst = (int)id;
              cur = 0;
            }
          }
        }
        if (leaf == kNoLeaf && is_leaf_ref(cur)) {
          leaf = cur;
          cur = pop();
        }
      } else if (cur == kSentinel) {
        // instance exit: world distance of the local hit (nanosg.h:832-870), back to the top-level walk
        if (best.t < FLT_MAX) {
          const InstanceDev *I = sc.inst + inst;
          const Mat43 minv33 = load_mat(&I->inv33), mxf = load_mat(&I->xf);
          float ldx, ldy, ldz, px, py, pz;
          multv(minv33, w.dx, w.dy, w.dz, ldx, ldy, ldz);
          const float tw = world_hit(mxf, w, c.ox, c.oy, c.oz, ldx, ldy, ldz, best.t, px, py, pz);
          if (tw < nearest.t) {
            nearest.t = tw;
            nearest.u = best.u;
            nearest.v = best.v;
            nearest.prim = best.prim;
            nearest.node = (uint32_t)inst;
            nearest.px = px;
            nearest.py = py;
            nearest.pz = pz;
          }
        }
        restore_world();
        inst = -1;
        wide = sc.top_wide;
        tris = sc.top_slots;
        cur = pop();
        if (is_leaf_ref(cur)) {
          leaf = cur;
          cur = pop();
        }
      }
    }

    // ---- retire
    if (ray_idx >= 0 && inst < 0 && cur == kNoLeaf && leaf == kNoLeaf) {
      store_scene_hit(hits, mask, (size_t)ray_idx, nearest, nearest.node != 0xFFFFFFFFu, w.max_t);
      if (n_boxes > (uint32_t)kMaxNodeHits) {
        const unsigned long long slot = atomicAdd(overflow_count, 1ull);
        overflow[slot] = (uint32_t)ray_idx;
      }
      ray_idx = -1;
    }
  }
}

}  // namespace

// ---- scene object -------------------------------------------------------------------------------------------------
struct Scene {
  int device = 0;
  uint32_t n = 0;
  Accel *top = nullptr;  // box-primitive accel: d_nodes / d_indices / d_prim_boxes
  InstanceDev *d_inst = nullptr;
  float *d_state = nullptr;  // 76 floats per instance
  uint32_t max_blas_depth = 0;
  std::vector<uint32_t> n_faces;  // per instance: triangles of its accel
  // per-launch scratch of the ring's slot k: the ray cursor d_counters[k], the overflow count d_counters[4 + k] and its
  // own overflow list
  static constexpr int kSlots = 4;
  uint32_t *d_overflow[kSlots] = {nullptr, nullptr, nullptr, nullptr};
  size_t overflow_cap[kSlots] = {0, 0, 0, 0};
  unsigned long long *d_counters = nullptr;
  LaunchRing<kSlots> ring;
  cudaStream_t stream = nullptr;  // commit
  StagingPipeline staging;        // nrt_scene_traverse
};

static void scene_destroy(Scene *s) {
  if (!s) return;
  DeviceGuard dg(s->device);
  if (s->top) {
    cudaFree(s->top->d_nodes);
    cudaFree(s->top->d_indices);
    cudaFree(s->top->d_prim_boxes);
    cudaFree(s->top->d_wide);
    cudaFree(s->top->d_tris);
    delete s->top;
  }
  cudaFree(s->d_inst);
  cudaFree(s->d_state);
  for (int k = 0; k < Scene::kSlots; k++) cudaFree(s->d_overflow[k]);
  cudaFree(s->d_counters);
  if (s->stream) cudaStreamDestroy(s->stream);
  delete s;
}

static int scene_launch(Scene *sc, const Ray36 *d_rays, size_t n, SceneHit32 *d_hits, uint8_t *d_mask, uint32_t flags,
                        cudaStream_t s) {
  if (n == 0) return NRT_OK;
  if (n > 0xFFFFFFFFull) {
    set_error("nrt_scene_traverse: more than 2^32-1 rays in one call");
    return NRT_ERR_INVALID;
  }
  const SceneDev dev{sc->top->d_nodes, sc->top->d_indices, sc->d_inst, sc->top->d_wide, sc->top->d_tris};
  const uint32_t stack_need = sc->top->stats.max_tree_depth + sc->max_blas_depth + 6;
  const bool list_only = (flags & NRT_TRAVERSE_CONFORMANCE) != 0 || stack_need > 1024;
  const int sms = device_sm_count(sc->device);
  if (list_only) {
    const size_t blocks = std::min<size_t>((n + 127) / 128, (size_t)sms * 32);
    scene_list_kernel<<<(unsigned)blocks, 128, 0, s>>>(dev, d_rays, n, nullptr, nullptr, d_hits, d_mask, flags);
    NRT_CUDA(cudaGetLastError());
    return NRT_OK;
  }
  if (stack_need <= 64 && ((flags >> 8) & 0xFFu) != 0) {  // the list-only and deep-stack walks ignore them
    set_error("nrt_scene_traverse: flags bits 8..15 are reserved");
    return NRT_ERR_INVALID;
  }
  return sc->ring.run(s, [&](uint32_t slot) {
    if (sc->overflow_cap[slot] < n) {  // grows rarely; the launch that last used the old list must be done with it
      const int rc = sc->ring.wait_host(slot);
      if (rc != NRT_OK) return rc;
      cudaFree(sc->d_overflow[slot]);
      sc->d_overflow[slot] = nullptr;
      sc->overflow_cap[slot] = 0;
      NRT_CUDA(cudaMalloc(&sc->d_overflow[slot], sizeof(uint32_t) * n));
      sc->overflow_cap[slot] = n;
    }
    uint32_t *d_overflow = sc->d_overflow[slot];
    unsigned long long *cursor = sc->d_counters + slot;
    unsigned long long *ovf = sc->d_counters + Scene::kSlots + slot;
    NRT_CUDA(cudaMemsetAsync(cursor, 0, sizeof(unsigned long long), s));
    NRT_CUDA(cudaMemsetAsync(ovf, 0, sizeof(unsigned long long), s));
    const size_t need = ((n + 31) / 32 + 3) / 4;
    size_t grid = (size_t)sms * (stack_need > 64 ? 2 : kUnifiedMinBlocks);
    if (grid > need) grid = need;
    if (stack_need > 64)
      scene_unified_kernel<1024, 2><<<(unsigned)grid, kSceneBlock, 0, s>>>(dev, d_rays, n, d_hits, d_mask, flags, cursor,
                                                                        d_overflow, ovf);
    else
      scene_unified_kernel<64, kUnifiedMinBlocks><<<(unsigned)grid, kSceneBlock, 0, s>>>(
          dev, d_rays, n, d_hits, d_mask, flags, cursor, d_overflow, ovf);
    NRT_CUDA(cudaGetLastError());
    scene_list_kernel<<<(unsigned)std::min<size_t>((n + 127) / 128, (size_t)sms * 4), 128, 0, s>>>(
        dev, d_rays, n, d_overflow, ovf, d_hits, d_mask, flags);
    NRT_CUDA(cudaGetLastError());
    return NRT_OK;
  });
}

SceneView scene_view(const nrt_scene *s) {
  const Scene *sc = reinterpret_cast<const Scene *>(s);
  return SceneView{sc->device, sc->n, sc->n_faces.data(), sc->d_inst, sc->d_state};
}

int scene_walk(const nrt_scene *s, const Ray36 *d_rays, size_t n, void *d_hits, uint8_t *d_mask, uint32_t flags,
               cudaStream_t st) {
  return scene_launch(const_cast<Scene *>(reinterpret_cast<const Scene *>(s)), d_rays, n, static_cast<SceneHit32 *>(d_hits),
                      d_mask, flags, st);
}

}  // namespace nrt

using namespace nrt;

extern "C" {

int nrt_scene_commit(const nrt_instance *instances, uint32_t n_instances, uint32_t flags, nrt_scene **out) {
  if (!out) {
    set_error("nrt_scene_commit: out is NULL");
    return NRT_ERR_INVALID;
  }
  *out = nullptr;
  if (!instances || n_instances == 0) {  // Scene::Commit refuses an empty scene (nanosg.h:708-711)
    set_error("nrt_scene_commit: empty scene");
    return NRT_ERR_INVALID;
  }
  for (uint32_t i = 0; i < n_instances; i++) {
    const Accel *a = reinterpret_cast<const Accel *>(instances[i].accel);
    if (!a || !a->d_wide || !a->d_nodes) {
      set_error("nrt_scene_commit: instance without a built accel");
      return NRT_ERR_INVALID;
    }
    if (a->device != reinterpret_cast<const Accel *>(instances[0].accel)->device) {
      set_error("nrt_scene_commit: instances live on different devices");
      return NRT_ERR_INVALID;
    }
  }
  Scene *sc = new (std::nothrow) Scene();
  if (!sc) return NRT_ERR_NOMEM;
  sc->device = reinterpret_cast<const Accel *>(instances[0].accel)->device;
  sc->n = n_instances;
  int rc = NRT_OK;
  InstanceIn *d_in = nullptr;
  auto fail = [&](int code) {
    cudaFree(d_in);
    scene_destroy(sc);
    return code;
  };
  DeviceGuard dg(sc->device);
  cudaError_t e = dg.err;
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&sc->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMalloc(&sc->d_counters, 32 * sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaMemset(sc->d_counters, 0, 32 * sizeof(unsigned long long));
  if (e == cudaSuccess) e = cudaMalloc(&sc->d_inst, sizeof(InstanceDev) * (size_t)n_instances);
  if (e == cudaSuccess) e = cudaMalloc(&sc->d_state, sizeof(float) * 76 * (size_t)n_instances);
  if (e == cudaSuccess) e = cudaMalloc(&d_in, sizeof(InstanceIn) * (size_t)n_instances);
  if (e != cudaSuccess) return fail(cuda_fail(e, "nrt_scene_commit allocations", __FILE__, __LINE__));
  sc->top = new (std::nothrow) Accel();
  if (!sc->top) return fail(NRT_ERR_NOMEM);
  sc->top->device = sc->device;
  sc->top->n_prims = n_instances;
  sc->top->options = default_build_options();
  sc->top->options.min_leaf_primitives = 1;  // nanosg.h:731-732
  e = cudaMalloc(&sc->top->d_prim_boxes, sizeof(float) * 6 * (size_t)n_instances);
  if (e != cudaSuccess) return fail(cuda_fail(e, "nrt_scene_commit boxes", __FILE__, __LINE__));
  {
    std::vector<InstanceIn> h(n_instances);
    for (uint32_t i = 0; i < n_instances; i++) {
      const Accel *a = reinterpret_cast<const Accel *>(instances[i].accel);
      memset(&h[i], 0, sizeof(InstanceIn));
      memcpy(h[i].xform, instances[i].xform, sizeof(float) * 16);
      for (int k = 0; k < 3; k++) {  // BVHAccel::BoundingBox = the root node's box (nanort.h:792-804)
        h[i].lbmin[k] = a->root_bmin[k];
        h[i].lbmax[k] = a->root_bmax[k];
      }
      h[i].wide = a->d_wide;
      h[i].tris = a->d_tris;
      h[i].nodes = a->d_nodes;
      h[i].verts = a->d_verts;
      h[i].faces = a->d_faces;
      sc->max_blas_depth = std::max(sc->max_blas_depth, a->stats.max_tree_depth);
      sc->n_faces.push_back(a->d_faces ? (uint32_t)a->n_prims : 0u);  // 0: not a triangle accel
    }
    e = cudaMemcpyAsync(d_in, h.data(), sizeof(InstanceIn) * (size_t)n_instances, cudaMemcpyHostToDevice, sc->stream);
    if (e == cudaSuccess) {
      instance_setup_kernel<<<(n_instances + 127) / 128, 128, 0, sc->stream>>>(d_in, n_instances, sc->d_inst,
                                                                              sc->top->d_prim_boxes, sc->d_state);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(sc->stream);
    if (e != cudaSuccess) return fail(cuda_fail(e, "nrt_scene_commit instance setup", __FILE__, __LINE__));
  }
  rc = (flags & NRT_BUILD_REFERENCE_TREE)
           ? build_reference_tree_on_device(sc->top, !(flags & NRT_BUILD_REFERENCE_CPP03_ORDER), sc->stream)
           : build_on_device(sc->top, sc->stream);
  if (rc == NRT_OK) rc = derive_private_layout(sc->top, sc->stream);
  if (rc == NRT_OK) {
    e = cudaStreamSynchronize(sc->stream);
    if (e != cudaSuccess) rc = cuda_fail(e, "nrt_scene_commit build", __FILE__, __LINE__);
  }
  if (rc != NRT_OK) return fail(rc);
  cudaFree(d_in);
  *out = reinterpret_cast<nrt_scene *>(sc);
  return NRT_OK;
}

void nrt_scene_free(nrt_scene *s) { scene_destroy(reinterpret_cast<Scene *>(s)); }

int nrt_scene_bounding_box(const nrt_scene *s, float bmin[3], float bmax[3]) {
  if (!s || !bmin || !bmax) {
    set_error("nrt_scene_bounding_box: NULL argument");
    return NRT_ERR_INVALID;
  }
  const Scene *sc = reinterpret_cast<const Scene *>(s);
  for (int k = 0; k < 3; k++) {
    bmin[k] = sc->top->root_bmin[k];
    bmax[k] = sc->top->root_bmax[k];
  }
  return NRT_OK;
}

int nrt_scene_nodes(nrt_scene *s, const void **nodes_40B, size_t *n_nodes, const uint32_t **indices,
                    size_t *n_indices) {
  if (!s) {
    set_error("nrt_scene_nodes: NULL scene");
    return NRT_ERR_INVALID;
  }
  Accel *a = reinterpret_cast<Scene *>(s)->top;
  return a->mirror.get(a->device, a->d_nodes, a->n_nodes, a->d_indices, a->n_prims, nodes_40B, n_nodes, indices,
                       n_indices);
}

int nrt_scene_instance_state(const nrt_scene *s, uint32_t instance, float out76[76]) {
  const Scene *sc = reinterpret_cast<const Scene *>(s);
  if (!sc || !out76 || instance >= sc->n) {
    set_error("nrt_scene_instance_state: bad argument");
    return NRT_ERR_INVALID;
  }
  NRT_DEVICE(sc->device);
  NRT_CUDA(cudaMemcpy(out76, sc->d_state + 76 * (size_t)instance, sizeof(float) * 76, cudaMemcpyDeviceToHost));
  return NRT_OK;
}

// Asynchronous on `stream`.  Any number of calls (and scene AO passes) on one scene may be in flight on any streams at
// once: scene_launch orders a call on the device after the earlier call that used the same scratch slot.
int nrt_scene_traverse_device(const nrt_scene *s, const void *d_rays_36B, size_t n_rays, void *d_hits_32B,
                              uint8_t *d_hit_mask, uint32_t flags, void *stream) {
  if (!s || (n_rays && (!d_rays_36B || !d_hits_32B))) {
    set_error("nrt_scene_traverse_device: NULL argument");
    return NRT_ERR_INVALID;
  }
  Scene *sc = const_cast<Scene *>(reinterpret_cast<const Scene *>(s));
  NRT_DEVICE(sc->device);
  return scene_launch(sc, static_cast<const Ray36 *>(d_rays_36B), n_rays, static_cast<SceneHit32 *>(d_hits_32B),
                      d_hit_mask, flags, static_cast<cudaStream_t>(stream));
}

int nrt_scene_traverse(const nrt_scene *s, const void *rays_36B, size_t n_rays, void *hits_32B, uint8_t *hit_mask,
                       uint32_t flags) {
  if (!s || (n_rays && (!rays_36B || !hits_32B))) {
    set_error("nrt_scene_traverse: NULL argument");
    return NRT_ERR_INVALID;
  }
  if (n_rays == 0) return NRT_OK;
  Scene *sc = const_cast<Scene *>(reinterpret_cast<const Scene *>(s));
  NRT_DEVICE(sc->device);
  return sc->staging.run(rays_36B, n_rays, sizeof(Ray36), hits_32B, sizeof(SceneHit32), hit_mask,
                         [&](const void *d_rays, size_t m, void *d_hits, uint8_t *d_mask, cudaStream_t st) {
                           return scene_launch(sc, static_cast<const Ray36 *>(d_rays), m, static_cast<SceneHit32 *>(d_hits),
                                               d_mask, flags, st);
                         });
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------------
// Primary + 1-bounce AO over a two-level scene (nrt_scene_render_ao_device): the wavefront pass of render.cu with
// nrt_scene_traverse_device as its traversal step.  Same composition from the reference's pieces (render.cu header):
// camera ray main.cc:809-817, hit point = the scene record's P (nanosg.h:846-850), geometric normal of the hit triangle
// in WORLD space (its vertices moved by the instance's local->world matrix, then main.cc:306-312) flipped towards the
// viewer, cosine direction main.cc:216-250, occlusion query = a closest-hit Scene::Traverse from the hit point lifted by
// ao_min_t along the normal, occluded iff the reported distance is below ao_max_t (see scene_gen_ao_kernel).
// Stand-alone stage kernels (the scene walk has no retire-step functor); one host read of the AO count per wave.
#include "wavefront.cuh"
#include "pass_host.cuh"

namespace nrt {
namespace {

__global__ void __launch_bounds__(256)
    scene_gen_primary_kernel(nrt_ao_params p, unsigned long long slot0, uint32_t count, Ray36 *__restrict__ rays,
                             uint32_t *__restrict__ pix_out, unsigned long long *counters /* [1] valid primaries */) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false;
  if (i < count) {
    uint32_t pix, smp;
    Ray36 r;
    r.org[0] = p.cam[0], r.org[1] = p.cam[1], r.org[2] = p.cam[2];
    r.type = 0;
    if (!slot_to_pixel(p, slot0 + i, pix, smp)) {
      pix = 0xFFFFFFFFu;
      r.dir[0] = 0.0f, r.dir[1] = 0.0f, r.dir[2] = -1.0f;
      r.min_t = 0.0f, r.max_t = -1.0f;  // max_t < min_t: misses at the root
    } else {
      valid = true;
      camera_ray(p.cam, p.width, p.height, p.seed, pix, smp + p.sample0, r.dir[0], r.dir[1], r.dir[2]);
      r.min_t = p.ray_min_t, r.max_t = p.ray_max_t;
    }
    rays[i] = r;
    pix_out[i] = pix;
  }
  const unsigned m = __ballot_sync(0xFFFFFFFFu, valid);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(counters + 1, (unsigned long long)__popc(m));
}

// one AO ray per primary hit, compacted with one atomic per warp; primary misses count as unoccluded
__global__ void __launch_bounds__(256)
    scene_gen_ao_kernel(nrt_ao_params p, unsigned long long slot0, uint32_t count, const Ray36 *__restrict__ rays,
                        const uint32_t *__restrict__ pix_in, const SceneHit32 *__restrict__ hits,
                        const uint8_t *__restrict__ mask, const InstanceDev *__restrict__ inst, Ray36 *__restrict__ ao_rays,
                        uint32_t *__restrict__ ao_pix, float *__restrict__ accum, unsigned long long *counters /* [0] */) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  bool make = false;
  Ray36 ao;
  uint32_t pix = 0xFFFFFFFFu;
  if (i < count) {
    pix = pix_in[i];
    if (pix != 0xFFFFFFFFu) {
      if (!mask[i]) {
        atomicAdd(accum + pix, 1.0f);
      } else {
        const SceneHit32 h = hits[i];
        const InstanceDev *I = inst + h.node_id;
        const Mat43 xf = load_mat(&I->xf);
        const uint32_t *f = I->faces + 3 * (size_t)h.prim_id;
        const float *v0 = I->verts + 3 * (size_t)f[0], *v1 = I->verts + 3 * (size_t)f[1], *v2 = I->verts + 3 * (size_t)f[2];
        float ax, ay, az, bx, by, bz, cx, cy, cz;
        multv(xf, v0[0], v0[1], v0[2], ax, ay, az);
        multv(xf, v1[0], v1[1], v1[2], bx, by, bz);
        multv(xf, v2[0], v2[1], v2[2], cx, cy, cz);
        const float e1x = bx - ax, e1y = by - ay, e1z = bz - az;
        const float e2x = cx - ax, e2y = cy - ay, e2z = cz - az;
        float nx = e1y * e2z - e1z * e2y, ny = e1z * e2x - e1x * e2z, nz = e1x * e2y - e1y * e2x;
        float ln = sqrtf(nx * nx + ny * ny + nz * nz);
        ln = ln > 0.0f ? 1.0f / ln : 0.0f;
        nx *= ln, ny *= ln, nz *= ln;
        const Ray36 r = rays[i];
        if (nx * r.dir[0] + ny * r.dir[1] + nz * r.dir[2] > 0.0f) nx = -nx, ny = -ny, nz = -nz;
        // orthonormal basis around n + cosine-weighted direction: make_ao_ray() of wavefront.cuh, same arithmetic
        const uint32_t smp = slot_sample(p, slot0 + i);
        const float sg = nz >= 0.0f ? 1.0f : -1.0f;
        const float a = -1.0f / (sg + nz), b = nx * ny * a;
        const float t1x = 1.0f + sg * nx * nx * a, t1y = sg * b, t1z = -sg * nx;
        const float t2x = b, t2y = sg + ny * ny * a, t2z = -ny;
        const float u1 = rand_ps(pix, smp, 2, p.seed), u2 = rand_ps(pix, smp, 3, p.seed);
        const float rr = sqrtf(u1), ph = 6.28318530718f * u2;
        float sn, cs;
        sincosf(ph, &sn, &cs);
        const float lx = rr * cs, ly = rr * sn, lz = sqrtf(fmaxf(0.0f, 1.0f - u1));
        const float wx = t1x * lx + t2x * ly + nx * lz, wy = t1y * lx + t2y * ly + ny * lz, wz = t1z * lx + t2z * ly + nz * lz;
        const float il = 1.0f / sqrtf(wx * wx + wy * wy + wz * wz);
        // Scene::Traverse walks an instance with the LOCAL range {0, FLT_MAX} (nanosg.h:831-836): min_t cannot keep the
        // ray off the surface it starts on, so the origin is lifted by ao_min_t along the (viewer-facing) normal, and
        // max_t only gates the top-level walk -- the accumulate step applies the radius to the reported distance
        ao.org[0] = h.P[0] + nx * p.ao_min_t, ao.org[1] = h.P[1] + ny * p.ao_min_t, ao.org[2] = h.P[2] + nz * p.ao_min_t;
        ao.dir[0] = wx * il, ao.dir[1] = wy * il, ao.dir[2] = wz * il;
        ao.min_t = 0.0f, ao.max_t = p.ao_max_t;
        ao.type = 0;
        make = true;
      }
    }
  }
  const unsigned m = __ballot_sync(0xFFFFFFFFu, make);
  if (m == 0u) return;
  unsigned long long base = 0;
  if (lane == 0) base = atomicAdd(counters + 0, (unsigned long long)__popc(m));
  base = __shfl_sync(0xFFFFFFFFu, base, 0);
  if (make) {
    const unsigned long long j = base + __popc(m & ((1u << lane) - 1u));
    ao_rays[j] = ao;
    ao_pix[j] = pix;
  }
}

__global__ void __launch_bounds__(256)
    scene_accumulate_ao_kernel(const uint8_t *__restrict__ ao_mask, const SceneHit32 *__restrict__ ao_hits,
                               const uint32_t *__restrict__ ao_pix, unsigned long long n, float max_t,
                               float *__restrict__ accum, unsigned long long *totals /* [1] occluded AO rays */) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  bool occluded = false;
  if (i < n) {
    occluded = ao_mask[i] != 0 && ao_hits[i].t < max_t;
    if (!occluded) atomicAdd(accum + ao_pix[i], 1.0f);
  }
  const unsigned m = __ballot_sync(0xFFFFFFFFu, occluded);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(totals + 1, (unsigned long long)__popc(m));
}

}  // namespace
}  // namespace nrt

extern "C" int nrt_scene_render_ao_device(const nrt_scene *s, const nrt_ao_params *params, float *d_accum, nrt_ao_result *res,
                                          void *stream) {
  if (!s || !params || !d_accum) {
    set_error("nrt_scene_render_ao_device: NULL argument");
    return NRT_ERR_INVALID;
  }
  const nrt_ao_params p = *params;
  if (p.width == 0 || p.height == 0 || p.spp == 0 || p.tile_w == 0 || p.tile_h == 0 || (p.tile_w % 8) || (p.tile_h % 4) ||
      p.n_shards == 0 || p.shard >= p.n_shards || (p.flags & NRT_AO_PACKED_TILES)) {
    set_error("nrt_scene_render_ao_device: bad parameters (tiles are multiples of 8x4 pixels; no packed tiles)");
    return NRT_ERR_INVALID;
  }
  Scene *sc = const_cast<Scene *>(reinterpret_cast<const Scene *>(s));
  NRT_DEVICE(sc->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint32_t trav_flags = p.flags & 0xFFFFu;
  // this shard's ray slots: whole tiles, dealt round-robin (render.cu: run_ao_pass)
  const ShardSlots sh = shard_slots(p.width, p.height, p.tile_w, p.tile_h, p.spp, p.shard, p.n_shards);
  const unsigned long long slots = sh.total, wave = sh.wave(1ull << 22);
  if (wave > 0xFFFFFFF0ull) {
    set_error("nrt_scene_render_ao_device: a tile holds too many ray slots");
    return NRT_ERR_INVALID;
  }
  CallMemory mem(st);
  Ray36 *rays = nullptr, *ao_rays = nullptr;
  uint32_t *pix = nullptr, *ao_pix = nullptr;
  SceneHit32 *hits = nullptr;
  uint8_t *mask = nullptr;
  unsigned long long *counters = nullptr;  // [0] AO rays of the wave, [1] valid primaries; [4..6] totals
  unsigned long long h_tot[3] = {0, 0, 0};
  uint32_t launches = 0, trav_launches = 0;
  PassClock clock(res != nullptr);
  if (slots > 0) {
    if (const int rc = mem.alloc([&](Carver &c) {
          rays = c.take<Ray36>(wave);
          ao_rays = c.take<Ray36>(wave);
          pix = c.take<uint32_t>(wave);
          ao_pix = c.take<uint32_t>(wave);
          hits = c.take<SceneHit32>(wave);
          mask = c.take<uint8_t>(wave);
          counters = c.take<unsigned long long>(8);
        }))
      return rc;
    NRT_CUDA(cudaMemsetAsync(counters, 0, sizeof(unsigned long long) * 8, st));
    if (const int rc = clock.start(st)) return rc;
  }
  for (unsigned long long slot0 = 0; slot0 < slots; slot0 += wave) {
    const uint32_t count = (uint32_t)std::min(wave, slots - slot0);
    const unsigned blocks = (count + 255) / 256;
    NRT_CUDA(cudaMemsetAsync(counters, 0, sizeof(unsigned long long) * 2, st));
    scene_gen_primary_kernel<<<blocks, 256, 0, st>>>(p, slot0, count, rays, pix, counters);
    if (const int rc = scene_launch(sc, rays, count, hits, mask, trav_flags, st)) return rc;
    scene_gen_ao_kernel<<<blocks, 256, 0, st>>>(p, slot0, count, rays, pix, hits, mask, sc->d_inst, ao_rays, ao_pix,
                                                d_accum, counters);
    unsigned long long h_cnt[2] = {0, 0};
    NRT_CUDA(cudaMemcpyAsync(h_cnt, counters, sizeof(h_cnt), cudaMemcpyDeviceToHost, st));
    NRT_CUDA(cudaStreamSynchronize(st));  // the scene walk takes its ray count from the host
    launches += 3;
    trav_launches += 1;
    h_tot[0] += h_cnt[0];
    h_tot[2] += h_cnt[1];
    if (h_cnt[0] > 0) {
      if (const int rc = scene_launch(sc, ao_rays, (size_t)h_cnt[0], hits, mask, trav_flags, st)) return rc;
      scene_accumulate_ao_kernel<<<(unsigned)((h_cnt[0] + 255) / 256), 256, 0, st>>>(mask, hits, ao_pix, h_cnt[0],
                                                                                       p.ao_max_t, d_accum, counters + 4);
      launches += 2;
      trav_launches += 1;
    }
    NRT_CUDA(cudaGetLastError());
  }
  if (slots > 0) {
    if (const int rc = clock.stop(st)) return rc;
    NRT_CUDA(cudaMemcpyAsync(&h_tot[1], counters + 5, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    NRT_CUDA(cudaStreamSynchronize(st));
  }
  if (res) {
    float total_ms = 0.0f, span[2];
    if (const int rc = clock.read(&total_ms, span)) return rc;
    res->primary_rays = h_tot[2];
    res->ao_rays = h_tot[0];
    res->ao_hits = h_tot[1];
    res->total_ms = total_ms;
    res->traverse_ms = 0.0f;  // not split: the scene walk is timed as part of the pass
    res->primary_traverse_ms = res->ao_traverse_ms = 0.0f;
    res->launches = launches;
    res->traverse_launches = trav_launches;
  }
  return mem.drain();
}

// ------------------------------------------------------------------------------------------------------------------
// Path tracing over a two-level scene (nrt_scene_render_path_device, nrt_scene_path_bounce_device): path.cu's wavefront
// loop with nrt_scene_traverse_device as its traversal step, as stand-alone stage kernels.  The shading of a hit is
// path_shade_hit (wavefront.cuh), the block the flat pass runs in its retire step, fed with world-space geometry:
// P = org + t dir from the world ray and world distance, the hit triangle moved to world space by the instance's
// matrix, its face-varying normals by the instance's inverse_transpose33, the lights from world-space records.
// Spawned rays are lifted off the surface like the AO pass's (nanosg walks an instance with the local range
// {0, FLT_MAX}, so min_t cannot keep a ray off the surface it starts on).
namespace nrt {

void launch_path_camera(const nrt_path_params &p, unsigned long long slot0, uint32_t count, const PathQueues &q,
                        unsigned long long *counters, cudaStream_t s);

namespace {

__global__ void __launch_bounds__(128)
    scene_light_setup_kernel(const uint32_t *__restrict__ pairs, uint32_t n, const InstanceDev *__restrict__ inst,
                             const SceneShadingDev *__restrict__ shading, const PathMaterial *__restrict__ mats,
                             float4 *__restrict__ rec) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t node = pairs[2 * (size_t)k], prim = pairs[2 * (size_t)k + 1];
  float w[9], nx, ny, nz, a2;
  world_triangle(inst + node, prim, w);
  world_normal(w, nx, ny, nz, a2);
  const uint32_t *ids = shading[node].mat_ids;
  const PathMaterial &m = mats[ids ? ids[prim] : 0u];
  rec[4 * (size_t)k + 0] = make_float4(w[0], w[1], w[2], w[3]);
  rec[4 * (size_t)k + 1] = make_float4(w[4], w[5], w[6], w[7]);
  rec[4 * (size_t)k + 2] = make_float4(w[8], nx, ny, nz);
  rec[4 * (size_t)k + 3] = make_float4(0.5f * a2, m.emission[0], m.emission[1], m.emission[2]);
}

__global__ void __launch_bounds__(256)
    scene_pack_rays_kernel(const float4 *__restrict__ org_tmin, const float4 *__restrict__ dir_tmax, uint32_t n,
                           Ray36 *__restrict__ rays) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 o = org_tmin[i], d = dir_tmax[i];
  Ray36 r;
  r.org[0] = o.x, r.org[1] = o.y, r.org[2] = o.z;
  r.dir[0] = d.x, r.dir[1] = d.y, r.dir[2] = d.z;
  r.min_t = o.w, r.max_t = d.w;
  r.type = 0;
  rays[i] = r;
}

// the shading of the n radiance rays of queue `in` from their scene hit records; Slots maps a path id to its (pixel
// or texel, sample): TileSlots for the path pass, TexelSlots for the lightmap bake's bounces 1 and up (scene_bake.cu)
template <class Slots>
__global__ void __launch_bounds__(256)
    scene_path_shade_kernel(nrt_path_params p, Slots slots, uint32_t bounce, uint32_t n, PathQueues q, int in,
                            const SceneHit32 *__restrict__ hits, const uint8_t *__restrict__ mask,
                            const InstanceDev *__restrict__ inst, const float *__restrict__ state76,
                            const SceneShadingDev *__restrict__ shading, const float4 *__restrict__ lights,
                            float *accum, unsigned long long *counters) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool cont = false, shadow = false;
  float4 co = make_float4(0, 0, 0, 0), cd = co, so = co, sd = co, sc = co;
  uint32_t pid = 0, pix, smp;
  if (i < n && mask[i]) {
    pid = q.path_id[in][i];
    if (slots(p, pid, pix, smp)) {
      const float4 o = q.org_tmin[in][i], d = q.dir_tmax[in][i];
      const SceneHit32 h = hits[i];
      const SceneShadingDev sh = shading[h.node_id];
      float w[9], gx, gy, gz, a2;
      world_triangle(inst + h.node_id, h.prim_id, w);
      world_normal(w, gx, gy, gz, a2);
      float nx, ny, nz;
      if (sh.fvn) {  // vertex normals to world space (nanosg.h:866-867), then main.cc:862-875
        const float *T = state76 + 76 * (size_t)h.node_id + 48;  // inverse_transpose33
        const float *n0 = sh.fvn + 9 * (size_t)h.prim_id;
        float wn[9];
        for (int k = 0; k < 3; k++) multv16(T, n0[3 * k], n0[3 * k + 1], n0[3 * k + 2], wn[3 * k], wn[3 * k + 1], wn[3 * k + 2]);
        const float b0 = 1.0f - h.u - h.v;
        nx = b0 * wn[0] + h.u * wn[3] + h.v * wn[6];
        ny = b0 * wn[1] + h.u * wn[4] + h.v * wn[7];
        nz = b0 * wn[2] + h.u * wn[5] + h.v * wn[8];
        const float l = sqrtf(nx * nx + ny * ny + nz * nz);
        if (fabsf(l) > 1.0e-6f) {
          const float il = 1.0f / l;
          nx *= il;
          ny *= il;
          nz *= il;
        }
      } else {  // calcNormal's orientation, -cross(e1, e2), as the flat pass
        nx = -gx;
        ny = -gy;
        nz = -gz;
      }
      const PathMaterial *mats = reinterpret_cast<const PathMaterial *>(p.d_materials);
      path_shade_hit(p, bounce, pix, smp, o, d, h.t, nx, ny, nz, mats + (sh.mat_ids ? sh.mat_ids[h.prim_id] : 0u),
                     SceneLights{lights}, SceneSpawn{gx, gy, gz}, q.weight[pid], q.weight + pid, accum, cont, shadow, co,
                     cd, so, sd, sc);
    }
  }
  path_append(q, in ^ 1, counters, cont, shadow, pid, co, cd, so, sd, sc);
}

// shadow rays: occluded iff the scene walk reports a hit nearer than max_t (SceneSpawn::shadow)
__global__ void __launch_bounds__(256)
    scene_path_shadow_kernel(const SceneHit32 *__restrict__ hits, const uint8_t *__restrict__ mask,
                             const float4 *__restrict__ sh_dir_tmax, const float4 *__restrict__ contrib_pix, uint32_t n,
                             float *accum) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (mask[i] && hits[i].t < sh_dir_tmax[i].w) return;
  const float4 c = contrib_pix[i];
  const size_t pix = __float_as_uint(c.w);
  atomicAdd(accum + 3 * pix + 0, c.x);
  atomicAdd(accum + 3 * pix + 1, c.y);
  atomicAdd(accum + 3 * pix + 2, c.z);
}

}  // namespace

int scene_path_setup(const char *name, const nrt_scene *s, const nrt_path_params &p, const nrt_scene_shading *shading,
                     size_t cap, cudaStream_t st, CallMemory &mem, ScenePathCall &c) {
  if (!shading) return refuse(name, "NULL shading array (one nrt_scene_shading per instance)");
  if (p.d_material_ids || p.d_facevarying_normals)
    return refuse(name,
                  "material ids and face-varying normals are given per instance (nrt_scene_shading), not in the params");
  if (p.flags & NRT_TRAVERSE_ANY_HIT) return refuse(name, "NRT_TRAVERSE_ANY_HIT is not supported by the scene walk");
  Scene *sc = const_cast<Scene *>(reinterpret_cast<const Scene *>(s));
  for (uint32_t i = 0; i < sc->n; i++)
    if (sc->n_faces[i] == 0) return refuse(name, "triangle instances only");
  c.s = s;
  c.p = p;
  c.trav_flags = p.flags & 0xFFFFu;
  std::vector<uint32_t> pairs(2 * (size_t)p.n_emissive);
  if (p.n_emissive) {
    NRT_CUDA(cudaMemcpyAsync(pairs.data(), p.d_emissive_faces, sizeof(uint32_t) * pairs.size(), cudaMemcpyDeviceToHost,
                             st));
    NRT_CUDA(cudaStreamSynchronize(st));
    for (uint32_t k = 0; k < p.n_emissive; k++)
      if (pairs[2 * k] >= sc->n || pairs[2 * k + 1] >= sc->n_faces[pairs[2 * k]])
        return refuse(name, ("emissive pair " + std::to_string(k) + " is not an {instance, face} of the scene").c_str());
  }
  const bool lights = p.n_emissive && cap > 0;
  if (const int rc = mem.alloc([&](Carver &k) {
        c.shading = k.take<SceneShadingDev>(sc->n);
        c.ctr = k.take<unsigned long long>(4);
        if (lights) c.lights = k.take<float4>(4 * (size_t)p.n_emissive);
        c.rays = k.take<Ray36>(cap);
        c.hits = k.take<SceneHit32>(cap);
        c.mask = k.take<uint8_t>(cap);
      }))
    return rc;
  NRT_CUDA(cudaMemcpyAsync(c.shading, shading, sizeof(SceneShadingDev) * sc->n, cudaMemcpyHostToDevice, st));
  if (lights) {
    scene_light_setup_kernel<<<(p.n_emissive + 127) / 128, 128, 0, st>>>(
        static_cast<const uint32_t *>(p.d_emissive_faces), p.n_emissive, sc->d_inst,
        c.shading, static_cast<const PathMaterial *>(p.d_materials),
        c.lights);
    NRT_CUDA(cudaGetLastError());
    c.launches++;
  }
  return NRT_OK;
}

// The shadow walk of a bounce: walk the ns rays of the shadow queue and add the visible light samples.
int scene_shadow_pass(ScenePathCall &c, const PathQueues &q, uint32_t ns, float *accum, cudaStream_t st) {
  if (ns == 0) return NRT_OK;
  Scene *sc = const_cast<Scene *>(reinterpret_cast<const Scene *>(c.s));
  const unsigned sb = (ns + 255) / 256;
  SceneHit32 *hits = c.hits;
  scene_pack_rays_kernel<<<sb, 256, 0, st>>>(q.sh_org_tmin, q.sh_dir_tmax, ns, c.rays);
  if (const int rc = scene_launch(sc, c.rays, ns, hits, c.mask, c.trav_flags, st)) return rc;
  scene_path_shadow_kernel<<<sb, 256, 0, st>>>(hits, c.mask, q.sh_dir_tmax, q.sh_contrib_pix, ns, accum);
  NRT_CUDA(cudaGetLastError());
  c.launches += 3;
  c.trav_launches += 1;
  return NRT_OK;
}

namespace {

// The path pass's own rules on its parameters, before scene_path_setup's (nothing is launched when they are refused)
int scene_path_check(const char *name, const nrt_path_params &p) {
  if (const int rc = check_path_params(p, name)) return rc;
  if (p.flags & NRT_AO_PACKED_TILES) return refuse(name, "NRT_AO_PACKED_TILES is not supported");
  return NRT_OK;
}

// One bounce: walk the n rays of queue `in`, shade them (Slots: TileSlots or TexelSlots), read the counts;
// then, with shadow_pass, walk the shadow rays and add the visible light samples.  out[0] continuation rays, out[1]
// shadow rays, out[2] camera rays (ctr[2]).
template <class Slots>
int scene_bounce(ScenePathCall &c, const Slots &slots, uint32_t bounce, uint32_t n, const PathQueues &q, int in,
                 float *accum, bool shadow_pass, unsigned long long out[3], cudaStream_t st) {
  Scene *sc = const_cast<Scene *>(reinterpret_cast<const Scene *>(c.s));
  const unsigned blocks = (n + 255) / 256;
  SceneHit32 *hits = c.hits;
  NRT_CUDA(cudaMemsetAsync(c.ctr, 0, 2 * sizeof(unsigned long long), st));
  scene_pack_rays_kernel<<<blocks, 256, 0, st>>>(q.org_tmin[in], q.dir_tmax[in], n, c.rays);
  if (const int rc = scene_launch(sc, c.rays, n, hits, c.mask, c.trav_flags, st)) return rc;
  scene_path_shade_kernel<<<blocks, 256, 0, st>>>(c.p, slots, bounce, n, q, in, hits, c.mask, sc->d_inst,
                                                  sc->d_state, c.shading,
                                                  c.lights, accum, c.ctr);
  NRT_CUDA(cudaGetLastError());
  NRT_CUDA(cudaMemcpyAsync(out, c.ctr, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  NRT_CUDA(cudaStreamSynchronize(st));  // the scene walk takes its ray count from the host
  c.launches += 3;
  c.trav_launches += 1;
  return shadow_pass ? scene_shadow_pass(c, q, (uint32_t)out[1], accum, st) : NRT_OK;
}

int scene_path_bounce(ScenePathCall &c, unsigned long long slot0, uint32_t bounce, uint32_t n, const PathQueues &q,
                      int in, float *accum, bool shadow_pass, unsigned long long out[3], cudaStream_t st) {
  return scene_bounce(c, TileSlots{slot0}, bounce, n, q, in, accum, shadow_pass, out, st);
}

}  // namespace

// Bounces 1 and up of the scene lightmap bake (scene_bake.cu): scene_bounce with the texel slot map.
int scene_texel_bounce(ScenePathCall &c, const TexelSlots &slots, uint32_t bounce, uint32_t n, const PathQueues &q,
                       int in, float *accum, bool shadow_pass, unsigned long long out[3], cudaStream_t st) {
  return scene_bounce(c, slots, bounce, n, q, in, accum, shadow_pass, out, st);
}

}  // namespace nrt

extern "C" int nrt_scene_render_path_device(const nrt_scene *s, const nrt_path_params *pp,
                                            const nrt_scene_shading *shading, float *d_accum_rgb, nrt_path_result *res,
                                            void *stream) {
  static const char *who = "nrt_scene_render_path_device";
  if (!s || !pp || !d_accum_rgb) return refuse(who, "NULL argument");
  const nrt_path_params p = *pp;
  if (const int rc = scene_path_check(who, p)) return rc;
  const Scene *sc = reinterpret_cast<const Scene *>(s);
  NRT_DEVICE(sc->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // this shard's ray slots: whole tiles, dealt round-robin, in waves of whole tiles (nrt_scene_render_ao_device)
  const ShardSlots sh = shard_slots(p.width, p.height, p.tile_w, p.tile_h, p.spp, p.shard, p.n_shards);
  const unsigned long long slots = sh.total, wave = sh.wave(1ull << 22);
  if (wave > 0xFFFFFFF0ull) return refuse(who, "a tile holds too many ray slots");
  CallMemory mem(st);
  ScenePathCall c;
  if (const int rc = scene_path_setup(who, s, p, shading, (size_t)wave, st, mem, c)) return rc;
  PathQueues q;
  if (const int rc = mem.alloc([&](Carver &k) { q = carve_path_queues(k, wave); })) return rc;
  PassClock clock(res != nullptr);
  if (const int rc = clock.start(st)) return rc;
  unsigned long long camera = 0, radiance = 0, shadow = 0;
  for (unsigned long long slot0 = 0; slot0 < slots; slot0 += wave) {
    const uint32_t count = (uint32_t)std::min(wave, slots - slot0);
    NRT_CUDA(cudaMemsetAsync(c.ctr, 0, 4 * sizeof(unsigned long long), st));
    launch_path_camera(p, slot0, count, q, c.ctr, st);
    c.launches++;
    uint32_t n = count;
    int in = 0;
    for (uint32_t b = 0; b < p.max_bounces && n > 0; b++) {
      unsigned long long out[3];
      if (const int rc = scene_path_bounce(c, slot0, b, n, q, in, d_accum_rgb, true, out, st)) return rc;
      if (b == 0) camera += out[2];
      radiance += b == 0 ? out[2] : n;  // slots outside the image are no Traverse calls
      shadow += out[1];
      n = (uint32_t)out[0];
      in ^= 1;
    }
    NRT_CUDA(cudaGetLastError());
  }
  if (const int rc = clock.stop(st)) return rc;
  if (const int rc = mem.drain()) return rc;
  if (res) {
    float total_ms = 0.0f, span[2];
    if (const int rc = clock.read(&total_ms, span)) return rc;
    res->camera_rays = camera;
    res->radiance_rays = radiance;
    res->shadow_rays = shadow;
    res->traverse_ms = 0.0f;  // not split: the scene walk is timed as part of the pass
    res->total_ms = total_ms;
    res->launches = c.launches;
    res->traverse_launches = c.trav_launches;
  }
  return NRT_OK;
}

extern "C" int nrt_scene_path_bounce_device(const nrt_scene *s, const nrt_path_params *pp,
                                            const nrt_scene_shading *shading, uint32_t bounce, uint64_t n_rays,
                                            const void *d_org_tmin, const void *d_dir_tmax, const uint32_t *d_path_id,
                                            void *d_weight, void *d_out_org_tmin, void *d_out_dir_tmax,
                                            uint32_t *d_out_path_id, void *d_sh_org_tmin, void *d_sh_dir_tmax,
                                            void *d_sh_contrib_pix, float *d_accum_rgb, uint64_t *n_continue,
                                            uint64_t *n_shadow, int skip_shadow_pass, void *stream) {
  static const char *who = "nrt_scene_path_bounce_device";
  if (!s || !pp || !d_org_tmin || !d_dir_tmax || !d_path_id || !d_weight || !d_out_org_tmin || !d_out_dir_tmax ||
      !d_out_path_id || !d_sh_org_tmin || !d_sh_dir_tmax || !d_sh_contrib_pix || !d_accum_rgb)
    return refuse(who, "NULL argument");
  if (n_continue) *n_continue = 0;
  if (n_shadow) *n_shadow = 0;
  if (n_rays > 0xFFFFFFF0ull) return refuse(who, "more than 2^32 - 16 rays");
  const nrt_path_params p = *pp;
  if (const int rc = scene_path_check(who, p)) return rc;
  const Scene *sc = reinterpret_cast<const Scene *>(s);
  NRT_DEVICE(sc->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallMemory mem(st);
  ScenePathCall c;
  if (const int rc = scene_path_setup(who, s, p, shading, (size_t)n_rays, st, mem, c)) return rc;
  if (n_rays == 0) return mem.drain();
  const PathQueues q = caller_path_queues(d_org_tmin, d_dir_tmax, d_path_id, d_weight, d_out_org_tmin, d_out_dir_tmax,
                                         d_out_path_id, d_sh_org_tmin, d_sh_dir_tmax, d_sh_contrib_pix);
  unsigned long long out[3] = {0, 0, 0};
  if (const int rc = scene_path_bounce(c, 0ull, bounce, (uint32_t)n_rays, q, 0, d_accum_rgb, !skip_shadow_pass, out, st))
    return rc;
  return finish_bounce(nullptr, out, n_continue, n_shadow, st);
}
