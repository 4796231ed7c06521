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
//   NodeBBoxIntersector::Intersect            examples/nanosg/nanosg.h:597-637   raw_box()
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

#include "common.cuh"
#include "trav_common.cuh"
#include "nodehits.cuh"

namespace nrt {

namespace {

constexpr int kMaxNodeHits = 64;  // kMaxIntersections, nanosg.h:787
constexpr int kNoLeaf = kEmptyLeaf;

// m[r][k] for r = 0..3, k = 0..2 (the only entries MultV reads), flat index 3 r + k, as three float4
struct Mat43 {
  float4 a, b, c;
};

struct InstanceDev {
  Mat43 inv;    // world -> local, points
  Mat43 inv33;  // world -> local, directions
  Mat43 xf;     // local -> world
  float bmin[3], bmax[3];  // world box
  const float *verts;      // the instance accel's packed float3 vertices / faces (the AO pass needs the hit triangle)
  const WideNode *wide;
  const PackedTri *tris;
  const Node40 *nodes;
  const uint32_t *faces;
};
static_assert(sizeof(InstanceDev) == 208, "InstanceDev");

struct SceneDev {
  const Node40 *top_nodes;
  const uint32_t *top_idx;
  const InstanceDev *inst;
  const WideNode *top_wide;    // top-level tree as child-pair nodes
  const PackedTri *top_slots;  // its leaves: {world bmin, instance id | world bmax, last flag | -}
};

struct SceneHit32 {
  float u, v, t;
  uint32_t prim_id, node_id;
  float P[3];
};
static_assert(sizeof(SceneHit32) == 32, "nrt_scene_hit");

// t[k] = ((m[0][k] v0 + m[1][k] v1) + m[2][k] v2) + m[3][k]   (Matrix::MultV, nanosg.h:214-222)
__device__ __forceinline__ void multv(const Mat43 &m, float x, float y, float z, float &ox, float &oy, float &oz) {
  ox = ((m.a.x * x + m.a.w * y) + m.b.z * z) + m.c.y;
  oy = ((m.a.y * x + m.b.x * y) + m.b.w * z) + m.c.z;
  oz = ((m.a.z * x + m.b.y * y) + m.c.x * z) + m.c.w;
}

__device__ __forceinline__ Mat43 load_mat(const Mat43 *p) {
  Mat43 m;
  const float4 *q = reinterpret_cast<const float4 *>(p);
  m.a = __ldg(q);
  m.b = __ldg(q + 1);
  m.c = __ldg(q + 2);
  return m;
}

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

__device__ __forceinline__ TraceOptions16 local_trace_options() {
  TraceOptions16 o;
  o.prim_ids_range[0] = 0;
  o.prim_ids_range[1] = 0x7FFFFFFFu;
  o.skip_prim_id = 0xFFFFFFFFu;
  o.cull_back_face = 0;  // Scene::Traverse never forwards its flag (nanosg.h:800-829)
  o.pad[0] = o.pad[1] = o.pad[2] = 0;
  return o;
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

constexpr int kListStack = 512;  // kMaxStackDepth (nanort.h:2613) == kNANORT_MAX_STACK_DEPTH

__global__ void __launch_bounds__(128)
    scene_list_kernel(SceneDev sc, const Ray36 *__restrict__ rays, size_t n, const uint32_t *__restrict__ subset,
                      const unsigned long long *__restrict__ n_subset, SceneHit32 *__restrict__ hits,
                      uint8_t *__restrict__ mask, uint32_t flags) {
  if (n_subset) n = (size_t)*n_subset;
  const bool cpp03 = (flags & NRT_TRAVERSE_CPP03_INVERSE) != 0;
  const TraceOptions16 opt = local_trace_options();
  for (size_t job = (size_t)blockIdx.x * blockDim.x + threadIdx.x; job < n; job += (size_t)gridDim.x * blockDim.x) {
    const size_t i = subset ? (size_t)subset[job] : job;
    const WorldRay w = load_world(rays, i);
    RayCtx c;
    setup_ray(c, w.ox, w.oy, w.oz, w.dx, w.dy, w.dz, w.min_t, cpp03);
    const float rix = 1.0f / w.dx, riy = 1.0f / w.dy, riz = 1.0f / w.dz;
    NodeHitHeap heap;
    heap.n = 0;
    uint32_t stack[kListStack];
    int sp = range_has_nan(w.min_t, w.max_t) ? -1 : 0;
    stack[0] = 0;
    while (sp >= 0) {  // ListNodeIntersections: hit_t stays at ray.max_t
      const Node40 *nd = sc.top_nodes + stack[sp];
      sp--;
      const float *f = reinterpret_cast<const float *>(nd);
      float tn;
      if (!slab(c, __ldg(f + 0), __ldg(f + 1), __ldg(f + 2), __ldg(f + 3), __ldg(f + 4), __ldg(f + 5), w.min_t, w.max_t,
                tn))
        continue;
      const uint32_t d0 = __ldg(&nd->data[0]), d1 = __ldg(&nd->data[1]);
      if (__ldg(&nd->flag) == 0) {
        const int axis = __ldg(&nd->axis);
        const int sgn = axis == 0 ? c.sx : (axis == 1 ? c.sy : c.sz);
        if (sp + 2 < kListStack) {
          stack[++sp] = sgn ? d0 : d1;
          stack[++sp] = sgn ? d1 : d0;
        }
        continue;
      }
      for (uint32_t k = 0; k < d0; k++) {
        const uint32_t id = __ldg(sc.top_idx + d1 + k);
        float tmin;
        if (!raw_box(w, rix, riy, riz, sc.inst[id].bmin, sc.inst[id].bmax, tmin)) continue;
        if (heap.n < kMaxNodeHits) {
          heap.push(tmin, id);
        } else if (tmin < heap.t[0]) {
          heap.pop();
          heap.push(tmin, id);
        }
      }
    }
    const int n_hits = heap.n;
    for (int k = 0; k < n_hits; k++) heap.pop();  // in-place heap sort: slots 0..n_hits-1 now run nearest first

    SceneBest best;
    best.t = FLT_MAX;
    best.node = 0xFFFFFFFFu;
    bool has_hit = false;
    for (int k = 0; k < n_hits; k++) {
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
      float hit_t = FLT_MAX;
      const Node40 *nodes = I->nodes;
      const PackedTri *tris = I->tris;
      sp = 0;
      stack[0] = 0;
      while (sp >= 0) {  // BVHAccel::Traverse in the reference's order (nanort.h:2526-2547)
        const Node40 *nd = nodes + stack[sp];
        sp--;
        const float *f = reinterpret_cast<const float *>(nd);
        float tn;
        if (!slab(lc, __ldg(f + 0), __ldg(f + 1), __ldg(f + 2), __ldg(f + 3), __ldg(f + 4), __ldg(f + 5), 0.0f, hit_t,
                  tn))
          continue;
        const uint32_t d0 = __ldg(&nd->data[0]), d1 = __ldg(&nd->data[1]);
        if (__ldg(&nd->flag) == 0) {
          const int axis = __ldg(&nd->axis);
          const int sgn = axis == 0 ? lc.sx : (axis == 1 ? lc.sy : lc.sz);
          if (sp + 2 < kListStack) {
            stack[++sp] = sgn ? d0 : d1;
            stack[++sp] = sgn ? d1 : d0;
          }
        } else {
          bool any = false;
          for (uint32_t q = 0; q < d0; q++) {
            const float4 *t = reinterpret_cast<const float4 *>(tris + (size_t)d1 + q);
            if (tri_test(lc, opt, __ldg(t), __ldg(t + 1), __ldg(t + 2), lb)) any = true;
          }
          if (any) hit_t = lb.t;
        }
      }
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
  const TraceOptions16 opt = local_trace_options();

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
  // per-launch scratch, handed out round-robin: slot k owns the ray cursor d_counters[k], the overflow count
  // d_counters[4 + k] and its own overflow list.  slot_done[k] is recorded after the last launch that used slot k,
  // and the next launch on slot k makes its stream wait for it, so launches in flight on any number of streams never
  // share a cursor or an overflow list.  next_slot and the events are guarded by mu.
  static constexpr int kSlots = 4;
  uint32_t *d_overflow[kSlots] = {nullptr, nullptr, nullptr, nullptr};
  size_t overflow_cap[kSlots] = {0, 0, 0, 0};
  cudaEvent_t slot_done[kSlots] = {nullptr, nullptr, nullptr, nullptr};
  unsigned long long *d_counters = nullptr;
  uint32_t next_slot = 0;
  cudaStream_t stream = nullptr;
  void *d_rays = nullptr, *d_hits = nullptr, *d_mask = nullptr;
  size_t stage = 0;
  std::mutex mu;
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
  for (int k = 0; k < Scene::kSlots; k++) {
    cudaFree(s->d_overflow[k]);
    if (s->slot_done[k]) cudaEventDestroy(s->slot_done[k]);
  }
  cudaFree(s->d_counters);
  cudaFree(s->d_rays);
  cudaFree(s->d_hits);
  cudaFree(s->d_mask);
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
  // the whole launch sequence under the lock: taking the slot, waiting for its previous user, enqueueing the kernels
  // and recording slot_done happen in the same order on the host and on the device
  std::lock_guard<std::mutex> lock(sc->mu);
  const int slot = (int)sc->next_slot;
  sc->next_slot = (sc->next_slot + 1) % (uint32_t)Scene::kSlots;
  if (sc->overflow_cap[slot] < n) {  // grows rarely; the launch that last used the old list must be done with it
    NRT_CUDA(cudaEventSynchronize(sc->slot_done[slot]));
    cudaFree(sc->d_overflow[slot]);
    sc->d_overflow[slot] = nullptr;
    sc->overflow_cap[slot] = 0;
    NRT_CUDA(cudaMalloc(&sc->d_overflow[slot], sizeof(uint32_t) * n));
    sc->overflow_cap[slot] = n;
  }
  uint32_t *d_overflow = sc->d_overflow[slot];
  NRT_CUDA(cudaStreamWaitEvent(s, sc->slot_done[slot], 0));
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
  NRT_CUDA(cudaEventRecord(sc->slot_done[slot], s));
  return NRT_OK;
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
  for (int k = 0; k < Scene::kSlots && e == cudaSuccess; k++)
    e = cudaEventCreateWithFlags(&sc->slot_done[k], cudaEventDisableTiming);
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
  Scene *sc = reinterpret_cast<Scene *>(s);
  Accel *a = sc->top;
  std::lock_guard<std::mutex> lock(sc->mu);
  if (!a->mirrors_valid) {
    NRT_DEVICE(sc->device);
    a->h_nodes.resize(a->n_nodes);
    a->h_indices.resize(a->n_prims);
    NRT_CUDA(cudaMemcpy(a->h_nodes.data(), a->d_nodes, sizeof(Node40) * a->n_nodes, cudaMemcpyDeviceToHost));
    NRT_CUDA(cudaMemcpy(a->h_indices.data(), a->d_indices, sizeof(uint32_t) * a->n_prims, cudaMemcpyDeviceToHost));
    a->mirrors_valid = true;
  }
  if (nodes_40B) *nodes_40B = a->h_nodes.data();
  if (n_nodes) *n_nodes = a->h_nodes.size();
  if (indices) *indices = a->h_indices.data();
  if (n_indices) *n_indices = a->h_indices.size();
  return NRT_OK;
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
  const size_t kChunk = (size_t)1 << 20;
  const size_t chunk = std::min(n_rays, kChunk);
  // one caller at a time on the staging buffers (Scene::Traverse is const and thread-safe in the reference)
  static std::mutex host_mu;
  std::lock_guard<std::mutex> lock(host_mu);
  if (sc->stage < chunk) {
    cudaFree(sc->d_rays);
    cudaFree(sc->d_hits);
    cudaFree(sc->d_mask);
    sc->d_rays = sc->d_hits = sc->d_mask = nullptr;
    sc->stage = 0;
    NRT_CUDA(cudaMalloc(&sc->d_rays, chunk * sizeof(Ray36)));
    NRT_CUDA(cudaMalloc(&sc->d_hits, chunk * sizeof(SceneHit32)));
    NRT_CUDA(cudaMalloc(&sc->d_mask, chunk));
    sc->stage = chunk;
  }
  const char *src = static_cast<const char *>(rays_36B);
  char *dst = static_cast<char *>(hits_32B);
  for (size_t done = 0; done < n_rays; done += chunk) {
    const size_t m = std::min(chunk, n_rays - done);
    NRT_CUDA(cudaMemcpyAsync(sc->d_rays, src + done * sizeof(Ray36), m * sizeof(Ray36), cudaMemcpyHostToDevice,
                             sc->stream));
    int rc = scene_launch(sc, static_cast<const Ray36 *>(sc->d_rays), m, static_cast<SceneHit32 *>(sc->d_hits),
                          static_cast<uint8_t *>(sc->d_mask), flags, sc->stream);
    if (rc != NRT_OK) return rc;
    NRT_CUDA(cudaMemcpyAsync(dst + done * sizeof(SceneHit32), sc->d_hits, m * sizeof(SceneHit32),
                             cudaMemcpyDeviceToHost, sc->stream));
    if (hit_mask) NRT_CUDA(cudaMemcpyAsync(hit_mask + done, sc->d_mask, m, cudaMemcpyDeviceToHost, sc->stream));
    NRT_CUDA(cudaStreamSynchronize(sc->stream));
  }
  return NRT_OK;
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

struct SceneWave {
  Ray36 *rays = nullptr, *ao_rays = nullptr;
  uint32_t *pix = nullptr, *ao_pix = nullptr;
  SceneHit32 *hits = nullptr;
  uint8_t *mask = nullptr;
  unsigned long long *counters = nullptr;  // [0] AO rays of the wave, [1] valid primaries; [4..6] totals
  void release() {
    cudaFree(rays), cudaFree(ao_rays), cudaFree(pix), cudaFree(ao_pix), cudaFree(hits), cudaFree(mask), cudaFree(counters);
  }
};

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
  const unsigned long long tiles_x = (p.width + p.tile_w - 1) / p.tile_w, tiles_y = (p.height + p.tile_h - 1) / p.tile_h;
  const unsigned long long n_tiles = tiles_x * tiles_y;
  const unsigned long long my_tiles = n_tiles > p.shard ? (n_tiles - p.shard + p.n_shards - 1) / p.n_shards : 0;
  const unsigned long long per_tile = (unsigned long long)p.tile_w * p.tile_h * p.spp;
  const unsigned long long slots = my_tiles * per_tile;
  unsigned long long wave = std::max<unsigned long long>(per_tile, (((unsigned long long)1 << 22) / per_tile) * per_tile);
  if (wave > slots) wave = slots;
  if (wave > 0xFFFFFFF0ull) {
    set_error("nrt_scene_render_ao_device: a tile holds too many ray slots");
    return NRT_ERR_INVALID;
  }
  SceneWave w;
  unsigned long long h_tot[3] = {0, 0, 0};
  uint32_t launches = 0, trav_launches = 0;
  int rc = NRT_OK;
  cudaError_t e = cudaSuccess;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  if (slots > 0) {
    e = cudaMalloc(&w.rays, sizeof(Ray36) * wave);
    if (e == cudaSuccess) e = cudaMalloc(&w.ao_rays, sizeof(Ray36) * wave);
    if (e == cudaSuccess) e = cudaMalloc(&w.pix, sizeof(uint32_t) * wave);
    if (e == cudaSuccess) e = cudaMalloc(&w.ao_pix, sizeof(uint32_t) * wave);
    if (e == cudaSuccess) e = cudaMalloc(&w.hits, sizeof(SceneHit32) * wave);
    if (e == cudaSuccess) e = cudaMalloc(&w.mask, wave);
    if (e == cudaSuccess) e = cudaMalloc(&w.counters, sizeof(unsigned long long) * 8);
    if (e == cudaSuccess) e = cudaMemsetAsync(w.counters, 0, sizeof(unsigned long long) * 8, st);
    if (e == cudaSuccess) e = cudaEventCreate(&ev0);
    if (e == cudaSuccess) e = cudaEventCreate(&ev1);
    if (e == cudaSuccess) e = cudaEventRecord(ev0, st);
  }
  for (unsigned long long slot0 = 0; slot0 < slots && e == cudaSuccess && rc == NRT_OK; slot0 += wave) {
    const uint32_t count = (uint32_t)std::min(wave, slots - slot0);
    const unsigned blocks = (count + 255) / 256;
    e = cudaMemsetAsync(w.counters, 0, sizeof(unsigned long long) * 2, st);
    if (e != cudaSuccess) break;
    scene_gen_primary_kernel<<<blocks, 256, 0, st>>>(p, slot0, count, w.rays, w.pix, w.counters);
    rc = scene_launch(sc, w.rays, count, w.hits, w.mask, trav_flags, st);
    if (rc != NRT_OK) break;
    scene_gen_ao_kernel<<<blocks, 256, 0, st>>>(p, slot0, count, w.rays, w.pix, w.hits, w.mask, sc->d_inst, w.ao_rays, w.ao_pix,
                                                d_accum, w.counters);
    unsigned long long h_cnt[2] = {0, 0};
    e = cudaMemcpyAsync(h_cnt, w.counters, sizeof(h_cnt), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);  // the scene walk takes its ray count from the host
    if (e != cudaSuccess) break;
    launches += 3;
    trav_launches += 1;
    h_tot[0] += h_cnt[0];
    h_tot[2] += h_cnt[1];
    if (h_cnt[0] > 0) {
      rc = scene_launch(sc, w.ao_rays, (size_t)h_cnt[0], w.hits, w.mask, trav_flags, st);
      if (rc != NRT_OK) break;
      scene_accumulate_ao_kernel<<<(unsigned)((h_cnt[0] + 255) / 256), 256, 0, st>>>(w.mask, w.hits, w.ao_pix, h_cnt[0], p.ao_max_t,
                                                                                       d_accum, w.counters + 4);
      launches += 2;
      trav_launches += 1;
    }
    e = cudaGetLastError();
  }
  float total_ms = 0.0f;
  if (slots > 0 && e == cudaSuccess && rc == NRT_OK) {
    e = cudaEventRecord(ev1, st);
    unsigned long long h_occ = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&h_occ, w.counters + 5, sizeof(h_occ), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e == cudaSuccess) e = cudaEventElapsedTime(&total_ms, ev0, ev1);
    h_tot[1] = h_occ;
  } else if (slots > 0) {
    cudaStreamSynchronize(st);  // nothing of a failed pass may still be running on the buffers freed below
  }
  if (ev0) cudaEventDestroy(ev0);
  if (ev1) cudaEventDestroy(ev1);
  w.release();
  if (rc != NRT_OK) return rc;
  NRT_CUDA(e);
  if (res) {
    res->primary_rays = h_tot[2];
    res->ao_rays = h_tot[0];
    res->ao_hits = h_tot[1];
    res->total_ms = total_ms;
    res->traverse_ms = 0.0f;  // not split: the scene walk is timed as part of the pass
    res->primary_traverse_ms = res->ao_traverse_ms = 0.0f;
    res->launches = launches;
    res->traverse_launches = trav_launches;
  }
  return NRT_OK;
}
