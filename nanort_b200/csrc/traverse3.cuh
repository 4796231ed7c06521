// Production traversal kernel (sm_90a).  Persistent warps pull rays from a global cursor and replace finished rays
// with new ones once enough lanes of the warp have retired (warp-ballot compaction of the ray pool).  Traversal is
// while-while with one postponed leaf per lane over child-pair nodes; the per-lane stack keeps (ref, entry distance)
// so that a popped subtree that now lies behind the current best is skipped without touching memory -- the same visit
// set the reference obtains by re-testing the box when it is popped (nanort.h:2532).
//
// Its first version was issue bound, with ~29 % of the issued instructions being control flow, hence: a triangle test
// without early returns (one predicate at the end; only the fp64 fallback branches), empty children that carry an
// inverted box (no reference checks in the node step), child selection by selects and one predicated push.  The
// profiles of that version further showed:
//
//   * 12 of the 54 instructions of a child-pair slab test were FSELs picking bmin/bmax by ray_dir_sign
//     (nanort.h:2291-2302) and they sit on the half-rate ALU pipe (60 % busy)  -> PairNode: the selection is an
//     address computed once per ray, the planes arrive as {near0 near1 far0 far1}.
//   * the (kx, ky, kz) permutation of the watertight test (nanort.h:1073-1081) compiled to eight small branches per
//     triangle (48 of 169 instructions)                                      -> TriCM: component-major triangles,
//     the permutation is the load address, the ray carries its origin already permuted.
//   * the far-plane widening `* 1.00000024f` (nanort.h:2303-2305) was applied per axis; rounding is monotonic, so
//     min(a*w, b*w, c*w) == min(a, b, c)*w bit for bit (w > 0): one multiply per box instead of three.
//   * three inlined copies of the pop loop ran at 3-16 active lanes           -> one pop site per iteration.
//
// Replaces (file:line in the reference tree): BVHAccel<float>::Traverse nanort.h:2487-2556, TestLeafNode :2372-2407,
// IntersectRayAABB<float> :2284-2325, TriangleIntersector::Intersect :1054-1150, PrepareTraversal :1163-1201.
#pragma once
#include "common.cuh"
#include "trav_common.cuh"

namespace nrt {

struct RayCtx3 {
  float ox, oy, oz;     // origin
  float ix, iy, iz;     // vsafe_inverse(dir)
  float Sx, Sy, Sz;     // watertight shear constants
  float okx, oky, okz;  // origin permuted by (kx, ky, kz)
  float t_min;
  // which float4 (16-byte unit) of a PairNode holds {near0 near1 far0 far1} of each axis: 0/1, 2/3, 4/5
  uint32_t nx, ny, nz;
  uint32_t tx, ty, tz;  // which float4 of a TriCM holds component kx / ky / kz: 0..2
};

__device__ __forceinline__ void setup_ray3(RayCtx3 &c, float ox, float oy, float oz, float dx, float dy, float dz,
                                           float min_t, bool cpp03) {
  RayCtx r;
  setup_ray(r, ox, oy, oz, dx, dy, dz, min_t, cpp03);  // the one definition of the reference's per-ray constants
  c.ox = ox;
  c.oy = oy;
  c.oz = oz;
  c.ix = r.ix;
  c.iy = r.iy;
  c.iz = r.iz;
  c.Sx = r.Sx;
  c.Sy = r.Sy;
  c.Sz = r.Sz;
  c.okx = sel3(r.kx, ox, oy, oz);
  c.oky = sel3(r.ky, ox, oy, oz);
  c.okz = sel3(r.kz, ox, oy, oz);
  c.t_min = min_t;
  c.nx = r.sx ? 1u : 0u;
  c.ny = r.sy ? 3u : 2u;
  c.nz = r.sz ? 5u : 4u;
  c.tx = (uint32_t)r.kx;
  c.ty = (uint32_t)r.ky;
  c.tz = (uint32_t)r.kz;
}

// v - o, or v itself when the layout already holds v - o (REL: camera-relative nodes and triangles, whose rays all
// start at the origin that was subtracted -- the same IEEE subtraction, done once per node instead of once per ray)
template <bool REL>
__device__ __forceinline__ float from_origin(float v, float o) {
  return REL ? v : v - o;
}

// Both child boxes of a PairNode (nanort.h:2284-2325, twice).  X = {near0 near1 far0 far1} of the x planes, etc.
// NaN handling as in slab(): fmaxf / fminf drop a NaN plane value, the range values are never NaN.
template <bool REL = false>
__device__ __forceinline__ void slab_pair(const RayCtx3 &c, const float4 X, const float4 Y, const float4 Z, float min_t,
                                          float best_t, bool &h0, bool &h1, float &t0, float &t1) {
  const float n0x = from_origin<REL>(X.x, c.ox) * c.ix, n1x = from_origin<REL>(X.y, c.ox) * c.ix;
  const float f0x = from_origin<REL>(X.z, c.ox) * c.ix, f1x = from_origin<REL>(X.w, c.ox) * c.ix;
  const float n0y = from_origin<REL>(Y.x, c.oy) * c.iy, n1y = from_origin<REL>(Y.y, c.oy) * c.iy;
  const float f0y = from_origin<REL>(Y.z, c.oy) * c.iy, f1y = from_origin<REL>(Y.w, c.oy) * c.iy;
  const float n0z = from_origin<REL>(Z.x, c.oz) * c.iz, n1z = from_origin<REL>(Z.y, c.oz) * c.iz;
  const float f0z = from_origin<REL>(Z.z, c.oz) * c.iz, f1z = from_origin<REL>(Z.w, c.oz) * c.iz;
  t0 = fmaxf(fmaxf(fmaxf(n0x, n0y), n0z), min_t);
  t1 = fmaxf(fmaxf(fmaxf(n1x, n1y), n1z), min_t);
  // min over the axes first, widen once: identical to widening each axis (monotonic rounding, factor > 0)
  const float e0 = fminf(fminf(fminf(f0x, f0y), f0z) * 1.00000024f, best_t);
  const float e1 = fminf(fminf(fminf(f1x, f1y), f1z) * 1.00000024f, best_t);
  h0 = t0 <= e0;
  h1 = t1 <= e1;
}

// The planes of a 64-byte WideNode (q0 = c0.lo.xyz, c0.hi.x | q1 = c0.hi.yz, c1.lo.xy | q2 = c1.lo.z, c1.hi.xyz) in
// the PairNode order {near0 near1 far0 far1}, picked by the ray's direction signs with selects.
__device__ __forceinline__ void wide_planes(const RayCtx3 &c, const float4 q0, const float4 q1, const float4 q2, float4 &X,
                                            float4 &Y, float4 &Z) {
  const bool sx = (c.nx & 1u) != 0u, sy = (c.ny & 1u) != 0u, sz = (c.nz & 1u) != 0u;
  X = make_float4(sx ? q0.w : q0.x, sx ? q2.y : q1.z, sx ? q0.x : q0.w, sx ? q1.z : q2.y);
  Y = make_float4(sy ? q1.x : q0.y, sy ? q2.z : q1.w, sy ? q0.y : q1.x, sy ? q1.w : q2.z);
  Z = make_float4(sz ? q1.y : q0.z, sz ? q2.w : q2.x, sz ? q0.z : q1.y, sz ? q2.x : q2.w);
}

// slab_pair on the WideNode
__device__ __forceinline__ void slab_pair_sel(const RayCtx3 &c, const float4 q0, const float4 q1, const float4 q2,
                                              float min_t, float best_t, bool &h0, bool &h1, float &t0, float &t1) {
  float4 X, Y, Z;
  wide_planes(c, q0, q1, q2, X, Y, Z);
  slab_pair(c, X, Y, Z, min_t, best_t, h0, h1, t0, t1);
}

// Slab test of the union of a pair's two child boxes, in the arithmetic of slab() (trav_common.cuh): the union's near
// plane is the nearer of the two near planes, its far plane the farther of the two far planes.  Every tree our builders
// or the reference emit has exact-union boxes, so on the root pair this is the reference's test of the root box
// (nanort.h:2527-2530).  An empty child's inverted box never wins either choice.  Used by the visit counters only.
__device__ __forceinline__ bool slab_union(const RayCtx3 &c, const float4 X, const float4 Y, const float4 Z, float min_t,
                                           float max_t) {
  const bool sx = (c.nx & 1u) != 0u, sy = (c.ny & 1u) != 0u, sz = (c.nz & 1u) != 0u;
  const float nx = sx ? fmaxf(X.x, X.y) : fminf(X.x, X.y), fx = sx ? fminf(X.z, X.w) : fmaxf(X.z, X.w);
  const float ny = sy ? fmaxf(Y.x, Y.y) : fminf(Y.x, Y.y), fy = sy ? fminf(Y.z, Y.w) : fmaxf(Y.z, Y.w);
  const float nz = sz ? fmaxf(Z.x, Z.y) : fminf(Z.x, Z.y), fz = sz ? fminf(Z.z, Z.w) : fmaxf(Z.z, Z.w);
  const float tnx = (nx - c.ox) * c.ix, tny = (ny - c.oy) * c.iy, tnz = (nz - c.oz) * c.iz;
  const float tfx = ((fx - c.ox) * c.ix) * 1.00000024f;
  const float tfy = ((fy - c.oy) * c.iy) * 1.00000024f;
  const float tfz = ((fz - c.oz) * c.iz) * 1.00000024f;
  const float tmin = fmaxf(tnz, fmaxf(tny, fmaxf(tnx, min_t)));
  const float tmax = fminf(tfz, fminf(tfy, fminf(tfx, max_t)));
  return tmin <= tmax;
}

// Watertight test on a component-major triangle: VX = {A[kx] B[kx] C[kx] w} etc.  Arithmetic order of
// nanort.h:1073-1147 (tri_test2 with the permutation already applied by the loads).  REL: as slab_pair.
template <bool REL = false>
__device__ __forceinline__ void tri_test3(const RayCtx3 &c, const TraceOptions16 &opt, bool filtered, const float4 VX,
                                          const float4 VY, const float4 VZ, Best &best) {
  const uint32_t prim = __float_as_uint(VX.w) & 0x7FFFFFFFu;
  bool rej = false;
  if (filtered)  // warp-uniform: the options are kernel parameters
    rej = (prim < opt.prim_ids_range[0]) | (prim >= opt.prim_ids_range[1]) | (prim == opt.skip_prim_id);
  const float Akx = from_origin<REL>(VX.x, c.okx), Bkx = from_origin<REL>(VX.y, c.okx), Ckx = from_origin<REL>(VX.z, c.okx);
  const float Aky = from_origin<REL>(VY.x, c.oky), Bky = from_origin<REL>(VY.y, c.oky), Cky = from_origin<REL>(VY.z, c.oky);
  const float Akz = from_origin<REL>(VZ.x, c.okz), Bkz = from_origin<REL>(VZ.y, c.okz), Ckz = from_origin<REL>(VZ.z, c.okz);
  const float Ax = Akx - c.Sx * Akz, Ay = Aky - c.Sy * Akz;
  const float Bx = Bkx - c.Sx * Bkz, By = Bky - c.Sy * Bkz;
  const float Cx = Ckx - c.Sx * Ckz, Cy = Cky - c.Sy * Ckz;
  float U = Cx * By - Cy * Bx;
  float V = Ax * Cy - Ay * Cx;
  float W = Bx * Ay - By * Ax;
  if (U == 0.0f || V == 0.0f || W == 0.0f) {  // rare: exact edge / vertex hits (nanort.h:1095-1107)
    U = (float)((double)Cx * (double)By - (double)Cy * (double)Bx);
    V = (float)((double)Ax * (double)Cy - (double)Ay * (double)Cx);
    W = (float)((double)Bx * (double)Ay - (double)By * (double)Ax);
  }
  const bool neg = (U < 0.0f) | (V < 0.0f) | (W < 0.0f);
  const bool pos = (U > 0.0f) | (V > 0.0f) | (W > 0.0f);
  rej |= neg & ((opt.cull_back_face != 0) | pos);
  const float det = (U + V) + W;
  rej |= (det == 0.0f);
  const float Az = c.Sz * Akz, Bz = c.Sz * Bkz, Cz = c.Sz * Ckz;
  const float D = (U * Az + V * Bz) + W * Cz;
  const float rcp = 1.0f / det;
  const float tt = D * rcp;
  rej |= (tt > best.t) | (tt < c.t_min);
  if (!rej) {
    best.t = tt;
    best.u = V * rcp;
    best.v = W * rcp;
    best.prim = prim;
  }
}

constexpr int kNone3 = kEmptyLeaf;  // "no node": finished, or (with a non-empty stack) waiting for a pop

constexpr int kTraverseBlock = 128;  // threads per CTA
constexpr int kNodeExit = 8;         // leave the node phase when fewer lanes than this want node work
// flags bit that only the counting launch sets (it clears the caller's): the tree is one leaf, and its root pair is the
// leaf plus an empty phantom child that the reference never visits
constexpr uint32_t kCountRootIsLeaf = 1u << 31;

// Launch policy of traverse_fast3_kernel (the values and why: traverse.cu)
template <int MINB_, int REFILL_MIN_, bool PAIR128_, int LEAF_AGAIN_MIN_, bool DEFER_RETIRE_, int NODE_UNROLL_>
struct Policy3 {
  static constexpr int kMinBlocks = MINB_;        // CTAs per SM (the register budget) and of the persistent grid
  static constexpr int kRefillMin = REFILL_MIN_;  // lanes that must have retired before the warp fetches new rays
  // true: 128-byte PairNode (sign-addressed planes, no selects); false: the 64-byte WideNode with 12 selects per pair
  // (half the cache footprint per node)
  static constexpr bool kPair128 = PAIR128_;
  // after the first leaf round of an outer iteration, another one runs only while at least this many lanes hold a
  // leaf (1: until none is left; 33: one round) -- a lane's second leaf (found while the first was postponed) is
  // otherwise tested in a round of its own with the few lanes that have one; carried over, it joins the next phase's
  static constexpr int kLeafAgainMin = LEAF_AGAIN_MIN_;
  // true: finished rays wait for the retire step until retired + empty lanes reach kRefillMin (or nothing else is
  // left to do), so that the epilogue and the refill that follows run with more lanes
  static constexpr bool kDeferRetire = DEFER_RETIRE_;
  // node steps per evaluation of the node phase's exit conditions (two ballots + a population count per check)
  static constexpr int kNodeUnroll = NODE_UNROLL_;
};

// DEPTH: capacity of the per-lane stack (entries); chosen by the launcher from the tree depth, so a push can
// never overflow (a child pair pushes one entry and descends one level).
template <class Rays, int DEPTH, bool COUNT, class P, class Epi>
__global__ void __launch_bounds__(kTraverseBlock, P::kMinBlocks)
    traverse_fast3_kernel(const void *__restrict__ pair, const TriCM *__restrict__ tris, Rays rays, size_t n, Epi epi,
                          TraceOptions16 opt, uint32_t flags, unsigned long long *cursor, unsigned long long *counts,
                          const unsigned long long *n_ptr) {
  // the launcher passes camera-relative nodes and triangles (Accel::d_pair_rel / d_tris_rel) to loaders whose rays
  // all start at one origin; the counting walk's root test (slab_union) and the WideNode planes stay absolute
  constexpr bool kRel = Rays::kSharedOrigin;
  static_assert(!kRel || (P::kPair128 && !COUNT), "camera-relative layout: PairNode, no counting");
  if (n_ptr) n = (size_t)*n_ptr;
  const int lane = threadIdx.x & 31;
  const unsigned lt_mask = (1u << lane) - 1u;
  const bool cpp03 = (flags & NRT_TRAVERSE_CPP03_INVERSE) != 0;
  const bool filtered = opt.prim_ids_range[0] != 0u || opt.prim_ids_range[1] < 0x7FFFFFFFu ||
                        opt.skip_prim_id < 0x7FFFFFFFu;
  const float4 *const pair4 = reinterpret_cast<const float4 *>(pair);  // 8 float4 per PairNode
  const float4 *const tris4 = reinterpret_cast<const float4 *>(tris);  // 3 float4 per TriCM

  // per-lane stack; the two extra entries keep what only the retire step reads (ray index, max_t) out of the
  // register file (thread-local memory, L1-resident)
  constexpr int PW = Rays::kPayloadWords;  // words a ray loader hands to the retire step (parked next to the stack)
  uint2 lstk[DEPTH + 2 + (PW + 1) / 2];
  int sp = 0;
  RayCtx3 c;
  Best best;
  float min_t = 0.0f;
  bool alive = false;
  int cur = kNone3, leaf = kNone3;
  bool exhausted = false;
  unsigned long long n_boxes = 0, n_prims = 0;
  const bool root_is_leaf = COUNT && (flags & kCountRootIsLeaf) != 0u;
  // COUNT only: lane-state histogram of the warp's iterations (nrt_traverse_lane_stats_device; lane 0 accumulates)
  unsigned long long st[14] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};

  for (;;) {
    // ---- replace retired rays (warp-ballot compaction of the ray pool)
    const unsigned dead = __ballot_sync(FULL_MASK, !alive);
    if (dead != 0u && !exhausted && (dead == FULL_MASK || __popc(dead) >= P::kRefillMin)) {
      const int cnt = __popc(dead);
      const int leader = __ffs(dead) - 1;
      if (COUNT) {
        st[0] += 1;    // refill events
        st[1] += cnt;  // lanes refilled (incl. lanes past the end of the ray set)
      }
      unsigned long long base = 0;
      if (lane == leader) base = atomicAdd(cursor, (unsigned long long)cnt);
      base = __shfl_sync(FULL_MASK, base, leader);
      if (base + (unsigned long long)cnt >= (unsigned long long)n) exhausted = true;
      if (!alive) {
        const unsigned long long mine = base + (unsigned long long)__popc(dead & lt_mask);
        if (mine < (unsigned long long)n) {
          float ox, oy, oz, dx, dy, dz, max_t;
          uint32_t payload[PW > 0 ? PW : 1];
          rays.load((size_t)mine, ox, oy, oz, dx, dy, dz, min_t, max_t, payload);
#pragma unroll
          for (int w = 0; w + 1 < PW; w += 2) lstk[DEPTH + 2 + w / 2] = make_uint2(payload[w], payload[w + 1]);
          if (PW & 1) lstk[DEPTH + 2 + PW / 2].x = payload[PW - 1];
          setup_ray3(c, ox, oy, oz, dx, dy, dz, min_t, cpp03);
          best.t = max_t;
          best.u = 0.0f;
          best.v = 0.0f;
          best.prim = 0xFFFFFFFFu;
          alive = true;
          lstk[DEPTH] = make_uint2((uint32_t)mine, (uint32_t)(mine >> 32));
          lstk[DEPTH + 1].x = __float_as_uint(max_t);
          sp = 0;
          cur = range_has_nan(min_t, max_t) ? kNone3 : 0;
          leaf = kNone3;
          if (COUNT) {
            // the reference's first pop, the root box; a ray that misses it visits nothing else
            n_boxes += 1;
            float4 X, Y, Z;
            if (P::kPair128) {
              X = __ldg(pair4 + c.nx);
              Y = __ldg(pair4 + c.ny);
              Z = __ldg(pair4 + c.nz);
            } else {
              wide_planes(c, __ldg(pair4), __ldg(pair4 + 1), __ldg(pair4 + 2), X, Y, Z);
            }
            if (cur == 0 && !slab_union(c, X, Y, Z, min_t, max_t)) cur = kNone3;
          }
        }
      }
    }
    if (__all_sync(FULL_MASK, !alive)) {
      if (exhausted) break;
      continue;
    }

    // ---- inner nodes.  A lane wants node work when it stands on a node, or stands nowhere but has stack entries.
    for (;;) {
      bool want = cur >= 0 || (cur == kNone3 && sp > 0);
      const unsigned desc = __ballot_sync(FULL_MASK, want);
      if (desc == 0u) break;
      if (__popc(desc) < kNodeExit && __any_sync(FULL_MASK, leaf != kNone3)) break;
#pragma unroll
      for (int rep = 0; rep < P::kNodeUnroll; ++rep) {
        if (rep > 0) want = cur >= 0 || (cur == kNone3 && sp > 0);
        if (want) {
          // The one pop site.  Pops until the lane stands on a node again: entries that start behind the current best
          // are dropped without touching memory (same visit set as the reference's re-test at pop, nanort.h:2532), a
          // popped leaf goes into the free leaf slot and the popping continues -- so that every lane that still has
          // inner nodes to visit takes a node step in THIS iteration (a lane that only pops is a wasted warp step).
          while (cur == kNone3 && sp > 0) {
            --sp;
            const uint2 e = lstk[sp];
            if (__uint_as_float(e.y) <= best.t) {
              cur = (int)e.x;
              if (cur < 0 && leaf == kNone3) {
                leaf = cur;
                cur = kNone3;
              }
            }
          }
        }
        if (COUNT) {  // who does what in this warp step
          const bool fin = alive && cur == kNone3 && leaf == kNone3 && sp == 0;
          st[2] += 1;                                                  // node-phase warp steps
          st[3] += __popc(__ballot_sync(FULL_MASK, cur >= 0));          // lanes testing a child pair
          st[4] += __popc(__ballot_sync(FULL_MASK, !alive));            // lanes without a ray
          st[5] += __popc(__ballot_sync(FULL_MASK, fin));               // lanes whose ray is finished (waits for the retire step)
          st[6] += __popc(__ballot_sync(FULL_MASK, alive && !fin && cur < 0));  // lanes parked on leaves
        }
        if (want) {
          if (cur >= 0) {
            bool h0, h1;
            float t0, t1;
            int2 R;
            if (P::kPair128) {
              const uint32_t n8 = (uint32_t)cur * 8u;
              const float4 X = __ldg(pair4 + (n8 + c.nx));
              const float4 Y = __ldg(pair4 + (n8 + c.ny));
              const float4 Z = __ldg(pair4 + (n8 + c.nz));
              R = __ldg(reinterpret_cast<const int2 *>(pair4 + (n8 + 6u)));
              slab_pair<kRel>(c, X, Y, Z, min_t, best.t, h0, h1, t0, t1);
            } else {
              const float4 *q = pair4 + (uint32_t)cur * 4u;
              const float4 q0 = __ldg(q), q1 = __ldg(q + 1), q2 = __ldg(q + 2);
              R = __ldg(reinterpret_cast<const int2 *>(q + 3));
              slab_pair_sel(c, q0, q1, q2, min_t, best.t, h0, h1, t0, t1);
            }
            if (COUNT) n_boxes += (root_is_leaf && cur == 0) ? 0 : 2;  // the one-leaf root was counted at load
            const bool swap = t1 < t0;
            const bool both = h0 & h1;
            if (both) {
              lstk[sp] = make_uint2((uint32_t)(swap ? R.x : R.y), __float_as_uint(swap ? t0 : t1));
              sp++;
            }
            cur = both ? (swap ? R.y : R.x) : (h0 ? R.x : (h1 ? R.y : kNone3));
            if (cur < 0 && cur != kNone3 && leaf == kNone3) {  // postpone the first leaf, keep descending
              leaf = cur;
              cur = kNone3;
            }
          }
        }
      }
    }

    // ---- leaves
    for (bool first_round = true;; first_round = false) {
      const unsigned with_leaf = __ballot_sync(FULL_MASK, leaf != kNone3);
      if (with_leaf == 0u) break;
      if (P::kLeafAgainMin > 1 && !first_round && __popc(with_leaf) < P::kLeafAgainMin) break;  // carried over
      if (COUNT) {
        st[7] += 1;                                                // leaf-phase rounds
        st[8] += __popc(with_leaf);  // lanes that enter a round with a leaf
      }
      if (leaf != kNone3) {
        uint32_t slot = (uint32_t)(~leaf);
        for (;;) {
          if (COUNT && lane == __ffs(__activemask()) - 1) st[9] += 1;  // triangle-test warp steps
          const uint32_t s3 = slot * 3u;
          const float4 VX = __ldg(tris4 + (s3 + c.tx));
          const float4 VY = __ldg(tris4 + (s3 + c.ty));
          const float4 VZ = __ldg(tris4 + (s3 + c.tz));
          if (COUNT) n_prims++;
          tri_test3<kRel>(c, opt, filtered, VX, VY, VZ, best);
          if ((int)__float_as_uint(VX.w) < 0) break;  // last triangle of the leaf
          slot++;
        }
        leaf = kNone3;
        if (cur < 0 && cur != kNone3) {  // a leaf was waiting in cur (the lane was parked)
          leaf = cur;
          cur = kNone3;
        }
        // occlusion query (NRT_TRAVERSE_ANY_HIT): a hit inside [min_t, max_t) ends the ray.  A record accepted AT
        // max_t is a miss (nanort.h:2552) and does not.
        if (Epi::kAnyHit && best.prim != 0xFFFFFFFFu && best.t < __uint_as_float(lstk[DEPTH + 1].x)) {
          sp = 0;
          cur = kNone3;
          leaf = kNone3;
        }
      }
    }

    // ---- retire: the epilogue (store the hit / spawn the AO ray / accumulate / shade) runs warp-wide
    const bool retiring = alive && cur == kNone3 && leaf == kNone3 && sp == 0;
    bool retire_now;
    if (P::kDeferRetire) {
      // wait until the retire step and the refill behind it have enough lanes -- unless the ray set is exhausted
      // (no refill will come) or no lane has anything else to do
      const unsigned rm = __ballot_sync(FULL_MASK, retiring);
      const unsigned idle = rm | __ballot_sync(FULL_MASK, !alive);
      retire_now = rm != 0u && (exhausted || idle == FULL_MASK || __popc(idle) >= P::kRefillMin);
    } else {
      retire_now = __any_sync(FULL_MASK, retiring);
    }
    if (COUNT) {
      st[12] += 1;  // outer iterations
      if (retire_now) {
        st[10] += 1;                                              // retire events
        st[11] += __popc(__ballot_sync(FULL_MASK, retiring));  // lanes retiring
      }
    }
    if (retire_now) {
      size_t ray_idx = 0;
      float max_t = 0.0f;
      uint32_t payload[PW > 0 ? PW : 1];
      if (retiring) {
        const uint2 id = lstk[DEPTH];
        ray_idx = (size_t)id.x | ((size_t)id.y << 32);
        max_t = __uint_as_float(lstk[DEPTH + 1].x);
#pragma unroll
        for (int w = 0; w + 1 < PW; w += 2) {
          const uint2 e = lstk[DEPTH + 2 + w / 2];
          payload[w] = e.x;
          payload[w + 1] = e.y;
        }
        if (PW & 1) payload[PW - 1] = lstk[DEPTH + 2 + PW / 2].x;
      }
      epi(retiring, ray_idx, best.t, best.u, best.v, best.prim, max_t, payload);
    }
    if (retiring && retire_now) alive = false;
  }

  if (COUNT) {
    for (int o = 16; o > 0; o >>= 1) {
      n_boxes += __shfl_down_sync(FULL_MASK, n_boxes, o);
      n_prims += __shfl_down_sync(FULL_MASK, n_prims, o);
    }
    // warp-uniform statistics were added by every lane alike: lane 0's copy is the warp's; st[9] is per lane
    for (int o = 16; o > 0; o >>= 1) st[9] += __shfl_down_sync(FULL_MASK, st[9], o);
    if (lane == 0) {
      atomicAdd(counts + 0, n_boxes);
      atomicAdd(counts + 1, n_prims);
#pragma unroll
      for (int k = 0; k < 14; ++k) atomicAdd(counts + 2 + k, st[k]);
    }
  }
}

// Launch policy of traverse_packet_kernel: a warp always takes a whole packet and retires it whole, so refill, deferred
// retire, leaf batching and node-step unrolling have nothing to tune
template <int MINB_, int K_>
struct PacketPolicy {
  static constexpr int kMinBlocks = MINB_;  // CTAs per SM (the register budget) and of the persistent grid
  static constexpr int kRays = K_;          // rays per lane: K samples of the lane's pixel walk as one
};

// A stack entry of the packet walk: the pushed child's ref, then each of the lane's K rays' entry distance (padded to
// one vector store and load)
template <int K>
struct PacketEntry;
template <>
struct PacketEntry<1> {
  typedef uint2 T;
};
template <>
struct PacketEntry<2> {
  typedef uint4 T;
};
__device__ __forceinline__ uint2 packet_entry(uint32_t ref, const uint32_t (&t)[1]) { return make_uint2(ref, t[0]); }
__device__ __forceinline__ uint4 packet_entry(uint32_t ref, const uint32_t (&t)[2]) {
  return make_uint4(ref, t[0], t[1], 0u);
}
__device__ __forceinline__ float packet_entry_t(const uint2 &e, int) { return __uint_as_float(e.y); }
__device__ __forceinline__ float packet_entry_t(const uint4 &e, int r) { return __uint_as_float(r == 0 ? e.y : e.z); }

// Packet traversal for camera rays: a warp takes one work unit (Units, wavefront.cuh: CameraUnits) -- one 8x4-pixel
// block at K consecutive samples, K rays per lane, the K samples of the lane's pixel -- and its K x 32 rays walk the
// tree together.  The samples of one block differ only by their sub-pixel jitter, so their walks are nearly the same,
// and the per-step work that is not per ray (the child refs, the ballots, the near-child vote, the stack pointer and
// the loop control) is shared by K x 32 rays.  The node the warp stands on is warp-uniform, and so is the stack
// pointer: every lane writes and reads its stack at the same index, so stack traffic is coalesced, and no lane
// postpones a leaf or waits in a vote on the others' phase.  Each ray still runs slab_pair / tri_test3 with its own
// best.t, enters a child only if its own test accepts it, and skips a popped entry that lies behind its own best
// (nanort.h:2532) -- only the order of the visits is the warp's (the near child is the one most rays that hit both
// children see nearer), the freedom the while-while kernel uses too.
//
// A ray that is not entering the current node ("inactive" there) only follows the warp: it runs the node step's loads
// and slab test with the others, but its hits are dropped (a ray that does not exist -- a sample past spp, a slot
// past the end of the ray set -- has a zeroed ray context whose plane offsets stay inside the node).  The entry
// distance a ray pushes for a child it did not hit is a NaN, which fails `entry <= best.t` at the pop: a real entry
// distance is never NaN, since slab_pair's fmaxf chain ends with min_t and fmaxf drops a NaN operand, and
// range_has_nan() rays never become active (their min_t / max_t are the only possible NaN there).
// DEPTH: capacity of the per-lane stack, as traverse_fast3_kernel (a pair pushes one entry and descends one level).
template <class Rays, class Units, int DEPTH, class P, class Epi>
__global__ void __launch_bounds__(kTraverseBlock, P::kMinBlocks)
    traverse_packet_kernel(const void *__restrict__ pair, const TriCM *__restrict__ tris, Rays rays, Units units,
                           size_t n_units, size_t n, Epi epi, TraceOptions16 opt, uint32_t flags,
                           unsigned long long *cursor) {
  constexpr bool kRel = Rays::kSharedOrigin;
  constexpr int K = P::kRays;
  static_assert(!Epi::kAnyHit, "packet walk: closest hit only");
  const int lane = threadIdx.x & 31;
  const bool cpp03 = (flags & NRT_TRAVERSE_CPP03_INVERSE) != 0;
  const bool filtered = opt.prim_ids_range[0] != 0u || opt.prim_ids_range[1] < 0x7FFFFFFFu ||
                        opt.skip_prim_id < 0x7FFFFFFFu;
  const float4 *const pair4 = reinterpret_cast<const float4 *>(pair);  // 8 float4 per PairNode
  const float4 *const tris4 = reinterpret_cast<const float4 *>(tris);  // 3 float4 per TriCM
  const uint32_t kNoEntry = 0x7FC00000u;                                // quiet NaN: never <= best.t

  // per-lane stack of (ref, K entry distances); the words past DEPTH park what only the retire step reads (each ray's
  // max_t and payload) in thread-local memory instead of the register file
  typedef typename PacketEntry<K>::T Entry;
  constexpr int PW = Rays::kPayloadWords;
  constexpr int kParkWords = K * (PW + 1);
  constexpr int kEntryWords = (int)(sizeof(Entry) / 4);
  Entry lstk[DEPTH + (kParkWords + kEntryWords - 1) / kEntryWords];
  uint32_t *const park = reinterpret_cast<uint32_t *>(lstk + DEPTH);  // ray r: park[r * (PW + 1) + 0 .. PW]

  for (;;) {
    unsigned long long unit = 0;
    if (lane == 0) unit = atomicAdd(cursor, 1ull);
    unit = __shfl_sync(FULL_MASK, unit, 0);
    if (unit >= (unsigned long long)n_units) break;

    RayCtx3 c[K];
    Best best[K];
    float min_t[K];
    bool active[K], valid[K];
    uint32_t slot[K];
#pragma unroll
    for (int r = 0; r < K; ++r) {
      c[r] = RayCtx3{};  // a ray that does not exist keeps these: in-range plane offsets for the node step's loads
      c[r].ny = 2u;
      c[r].nz = 4u;
      best[r].t = 0.0f;
      best[r].u = 0.0f;
      best[r].v = 0.0f;
      best[r].prim = 0xFFFFFFFFu;
      min_t[r] = 0.0f;
      active[r] = false;
      valid[r] = units.slot((uint32_t)unit, r, (uint32_t)lane, slot[r]) && (size_t)slot[r] < n;
      if (valid[r]) {
        float ox, oy, oz, dx, dy, dz, max_t;
        uint32_t payload[PW > 0 ? PW : 1];
        rays.load((size_t)slot[r], ox, oy, oz, dx, dy, dz, min_t[r], max_t, payload);
        uint32_t *const pk = park + r * (PW + 1);
        pk[0] = __float_as_uint(max_t);
#pragma unroll
        for (int w = 0; w < PW; ++w) pk[1 + w] = payload[w];
        setup_ray3(c[r], ox, oy, oz, dx, dy, dz, min_t[r], cpp03);
        best[r].t = max_t;
        active[r] = !range_has_nan(min_t[r], max_t);
      }
    }

    // The K rays of a lane leave one pixel a fraction of a pixel apart, so they almost always share their direction
    // signs and (kx, ky, kz): the sign-addressed plane offsets and the triangle component offsets.  When every ray of
    // the warp shares them with its lane's first ray, a node step or a triangle takes one set of loads for all K rays.
    // A ray that does not exist takes its lane's first ray's offsets (its hits are dropped; the loads stay inside the
    // node and the leaf).
    bool same = true;
#pragma unroll
    for (int r = 1; r < K; ++r) {
      if (!valid[r]) {
        c[r].nx = c[0].nx;
        c[r].ny = c[0].ny;
        c[r].nz = c[0].nz;
        c[r].tx = c[0].tx;
        c[r].ty = c[0].ty;
        c[r].tz = c[0].tz;
      }
      same &= c[r].nx == c[0].nx && c[r].ny == c[0].ny && c[r].nz == c[0].nz && c[r].tx == c[0].tx &&
              c[r].ty == c[0].ty && c[r].tz == c[0].tz;
    }
    const bool shared = K > 1 && __all_sync(FULL_MASK, same);  // warp-uniform

    bool any_active = false;
#pragma unroll
    for (int r = 0; r < K; ++r) any_active |= active[r];
    int cur = __any_sync(FULL_MASK, any_active) ? 0 : kNone3;  // warp-uniform from here on
    int sp = 0;
    while (cur != kNone3) {
      if (cur >= 0) {
        // every ray tests the pair (no branch around it: the step is issue bound), only active rays' hits count
        bool h0[K], h1[K];
        float t0[K], t1[K];
        bool any0 = false, any1 = false;
        const uint32_t n8 = (uint32_t)cur * 8u;
        const int2 R = __ldg(reinterpret_cast<const int2 *>(pair4 + (n8 + 6u)));
        if (shared) {
          const float4 X = __ldg(pair4 + (n8 + c[0].nx));
          const float4 Y = __ldg(pair4 + (n8 + c[0].ny));
          const float4 Z = __ldg(pair4 + (n8 + c[0].nz));
#pragma unroll
          for (int r = 0; r < K; ++r)
            slab_pair<kRel>(c[r], X, Y, Z, min_t[r], best[r].t, h0[r], h1[r], t0[r], t1[r]);
        } else {
#pragma unroll
          for (int r = 0; r < K; ++r) {
            const float4 X = __ldg(pair4 + (n8 + c[r].nx));
            const float4 Y = __ldg(pair4 + (n8 + c[r].ny));
            const float4 Z = __ldg(pair4 + (n8 + c[r].nz));
            slab_pair<kRel>(c[r], X, Y, Z, min_t[r], best[r].t, h0[r], h1[r], t0[r], t1[r]);
          }
        }
#pragma unroll
        for (int r = 0; r < K; ++r) {
          h0[r] &= active[r];
          h1[r] &= active[r];
          any0 |= h0[r];
          any1 |= h1[r];
        }
        const unsigned m0 = __ballot_sync(FULL_MASK, any0), m1 = __ballot_sync(FULL_MASK, any1);
        if (m0 != 0u && m1 != 0u) {
          // both children are wanted: the one that most rays hitting both see nearer goes first (the first child when
          // no ray hits both)
          int first1 = 0, both = 0;
#pragma unroll
          for (int r = 0; r < K; ++r) {
            first1 += (h0[r] & h1[r] & (t1[r] < t0[r])) ? 1 : 0;
            both += (h0[r] & h1[r]) ? 1 : 0;
          }
          const bool one = 2 * __reduce_add_sync(FULL_MASK, (unsigned)first1) > __reduce_add_sync(FULL_MASK, (unsigned)both);
          uint32_t te[K];
#pragma unroll
          for (int r = 0; r < K; ++r) {
            te[r] = (one ? h0[r] : h1[r]) ? __float_as_uint(one ? t0[r] : t1[r]) : kNoEntry;
            active[r] = one ? h1[r] : h0[r];
          }
          lstk[sp] = packet_entry((uint32_t)(one ? R.x : R.y), te);
          sp++;
          cur = one ? R.y : R.x;
        } else if (m0 != 0u) {
          cur = R.x;
#pragma unroll
          for (int r = 0; r < K; ++r) active[r] = h0[r];
        } else if (m1 != 0u) {
          cur = R.y;
#pragma unroll
          for (int r = 0; r < K; ++r) active[r] = h1[r];
        } else {
          cur = kNone3;
        }
      } else {
        bool any = false;
#pragma unroll
        for (int r = 0; r < K; ++r) any |= active[r];
        if (any) {
          uint32_t s = (uint32_t)(~cur);
          for (;;) {
            bool last = false;
            if (shared) {
              const uint32_t s3 = s * 3u;
              const float4 VX = __ldg(tris4 + (s3 + c[0].tx));
              const float4 VY = __ldg(tris4 + (s3 + c[0].ty));
              const float4 VZ = __ldg(tris4 + (s3 + c[0].tz));
#pragma unroll
              for (int r = 0; r < K; ++r)
                if (active[r]) tri_test3<kRel>(c[r], opt, filtered, VX, VY, VZ, best[r]);
              last = (int)__float_as_uint(VX.w) < 0;  // last triangle of the leaf
            } else {
#pragma unroll
              for (int r = 0; r < K; ++r) {
                if (active[r]) {
                  const uint32_t s3 = s * 3u;
                  const float4 VX = __ldg(tris4 + (s3 + c[r].tx));
                  const float4 VY = __ldg(tris4 + (s3 + c[r].ty));
                  const float4 VZ = __ldg(tris4 + (s3 + c[r].tz));
                  tri_test3<kRel>(c[r], opt, filtered, VX, VY, VZ, best[r]);
                  last = (int)__float_as_uint(VX.w) < 0;
                }
              }
            }
            if (last) break;
            s++;
          }
        }
        cur = kNone3;
      }
      // pop until some ray enters the popped entry
      while (cur == kNone3 && sp > 0) {
        --sp;
        const Entry e = lstk[sp];
        bool any = false;
#pragma unroll
        for (int r = 0; r < K; ++r) {
          active[r] = packet_entry_t(e, r) <= best[r].t;
          any |= active[r];
        }
        if (__any_sync(FULL_MASK, any)) cur = (int)e.x;
      }
    }

    // retire the whole unit: the epilogue runs with all 32 lanes, once per sample of the unit
#pragma unroll
    for (int r = 0; r < K; ++r) {
      uint32_t payload[PW > 0 ? PW : 1];
      float max_t = 0.0f;
      if (valid[r]) {
        const uint32_t *const pk = park + r * (PW + 1);
        max_t = __uint_as_float(pk[0]);
#pragma unroll
        for (int w = 0; w < PW; ++w) payload[w] = pk[1 + w];
      }
      epi(valid[r], (size_t)slot[r], best[r].t, best[r].u, best[r].v, best[r].prim, max_t, payload);
    }
  }
}

}  // namespace nrt
