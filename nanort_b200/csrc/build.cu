// Device-wide binned-SAH BVH builder (sm_90a), emitting nanort's own arrays.
//
// Replaces (file:line in the reference tree):
//   BVHAccel<float>::Build / BuildTree / BuildShallowTree  nanort.h:1892-2149, 1759-1890, 1600-1757
//   ContributeBinBuffer / FindCutFromBinBuffer             nanort.h:1314-1367, 1381-1430
//   CalculateSurfaceArea                                    nanort.h:1278-1283
//   TriangleMesh::BoundingBoxAndCenter                      nanort.h:958-971
//   TriangleSAHPred + std::partition                        nanort.h:897-911, 1841
//   ComputeBoundingBox*                                     nanort.h:1432-1594
//
// Semantics kept (SURVEY.md B.7): leaf iff n <= min_leaf_primitives || depth >= max_tree_depth; root
// depth 0; node boxes are the exact min/max of the member triangles; `bin_size` centroid bins per axis
// over the NODE's box, centroid = (p0+p1+p2)*(1/3); candidate planes are bin boundaries; cost =
// N_L*area(L) + N_R*area(R), area = 2*(dx*dy + dy*dz + dz*dx); strict `<` argmin along an axis, ties
// between axes go to the lower axis; data[0] is the child on the lower side; when no plane separates the
// centroids the range is cut at the median index; nodes come out in depth-first pre-order (the order of
// the reference's serial BuildTree), indices_ holds original primitive ids.
// Deliberate differences, both documented in DESIGN.md: all three axes are binned (the pinned commit
// bins only x because of the guard at nanort.h:1357, SURVEY.md F1), and a primitive goes left iff its
// centroid's BIN is below the chosen boundary (the reference re-evaluates p0+p1+p2 < 3*pos, which can
// differ from its own binning by one rounding).
//
// Structure: (A) level-synchronous passes over all primitives for nodes with more than kSubtree
// primitives -- block-private shared-memory bins flushed with atomics, one warp per node for the sweep,
// a device-wide scan + stable scatter for the partition; (B) one WARP per remaining subtree builds it to
// the leaves entirely in shared memory; (C) pre-order indices are computed in closed form from
// (leaves to the left, depth, right turns) and the 40-byte nodes are emitted in one pass.
#include <float.h>

#include <utility>

#include "build_common.cuh"
#include "common.cuh"
#include "radix_sort.cuh"
#include "scan.cuh"

namespace nrt {

namespace {

constexpr int kSubtree = 128;     // phase B handles nodes with at most this many primitives (one warp each)
constexpr int kMid = 2048;        // the middle phase (one CTA per node) takes nodes of kSubtree+1 .. kMid primitives
constexpr int kMidThreads = 256;
constexpr int kSubWarps = 4;      // warps (= subtrees) per phase-B CTA
constexpr int kSubStack = 8;      // log2(kSubtree) + 1 parked nodes per subtree
constexpr uint32_t kDeadNode = 0xFFFFFFFFu;  // BNode.depth of a reserved but unused pool slot

// ------------------------------------------------------------------ primitives
// plo = (bmin.xyz, c.x), phi = (bmax.xyz, c.y), pcz = c.z
__global__ void prim_setup_kernel(const float *__restrict__ verts, const uint32_t *__restrict__ faces, uint32_t n,
                                  float4 *__restrict__ plo, float4 *__restrict__ phi, float *__restrict__ pcz,
                                  uint32_t *__restrict__ scene_keys /*6*/) {
  __shared__ float s_box[8][6];  // per-warp partial scene box (256-thread CTAs)
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  if (i < n) {
    uint32_t f0 = faces[3 * (size_t)i], f1 = faces[3 * (size_t)i + 1], f2 = faces[3 * (size_t)i + 2];
    const float *p0 = verts + 3 * (size_t)f0, *p1 = verts + 3 * (size_t)f1, *p2 = verts + 3 * (size_t)f2;
    float c[3];
    const float third = 1.0f / 3.0f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      float a = p0[k], b = p1[k], cc = p2[k];
      lo[k] = fminf(a, fminf(b, cc));
      hi[k] = fmaxf(a, fmaxf(b, cc));
      c[k] = ((a + b) + cc) * third;
    }
    plo[i] = make_float4(lo[0], lo[1], lo[2], c[0]);
    phi[i] = make_float4(hi[0], hi[1], hi[2], c[1]);
    pcz[i] = c[2];
  }
  // scene box: warp reduce, then one atomic per warp and component
#pragma unroll
  for (int k = 0; k < 3; k++) {
    float a = lo[k], b = hi[k];
    for (int o = 16; o > 0; o >>= 1) {
      a = fminf(a, __shfl_xor_sync(0xFFFFFFFFu, a, o));
      b = fmaxf(b, __shfl_xor_sync(0xFFFFFFFFu, b, o));
    }
    if ((threadIdx.x & 31) == 0) {
      s_box[threadIdx.x >> 5][k] = a;
      s_box[threadIdx.x >> 5][3 + k] = b;
    }
  }
  __syncthreads();
  if (threadIdx.x < 6) {  // one atomic per CTA and component
    const int k = threadIdx.x;
    float v = s_box[0][k];
    for (int w = 1; w < (int)(blockDim.x >> 5); w++) v = k < 3 ? fminf(v, s_box[w][k]) : fmaxf(v, s_box[w][k]);
    if (k < 3)
      atomicMin(scene_keys + k, fkey(v));
    else
      atomicMax(scene_keys + k, fkey(v));
  }
}

// Same records for axis-aligned boxes as primitives (the two-level scene's top-level build,
// NodeBBoxGeometry::BoundingBoxAndCenter, examples/nanosg/nanosg.h:560-573): centre = (bmax + bmin) / 2.
__global__ void box_setup_kernel(const float *__restrict__ boxes6, uint32_t n, float4 *__restrict__ plo,
                                 float4 *__restrict__ phi, float *__restrict__ pcz,
                                 uint32_t *__restrict__ scene_keys /*6*/) {
  __shared__ float s_box[8][6];  // per-warp partial scene box (256-thread CTAs)
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  if (i < n) {
    float c[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
      lo[k] = boxes6[6 * (size_t)i + k];
      hi[k] = boxes6[6 * (size_t)i + 3 + k];
      c[k] = (hi[k] + lo[k]) / 2.0f;
    }
    plo[i] = make_float4(lo[0], lo[1], lo[2], c[0]);
    phi[i] = make_float4(hi[0], hi[1], hi[2], c[1]);
    pcz[i] = c[2];
  }
#pragma unroll
  for (int k = 0; k < 3; k++) {
    float a = lo[k], b = hi[k];
    for (int o = 16; o > 0; o >>= 1) {
      a = fminf(a, __shfl_xor_sync(0xFFFFFFFFu, a, o));
      b = fmaxf(b, __shfl_xor_sync(0xFFFFFFFFu, b, o));
    }
    if ((threadIdx.x & 31) == 0) {
      s_box[threadIdx.x >> 5][k] = a;
      s_box[threadIdx.x >> 5][3 + k] = b;
    }
  }
  __syncthreads();
  if (threadIdx.x < 6) {  // one atomic per CTA and component
    const int k = threadIdx.x;
    float v = s_box[0][k];
    for (int w = 1; w < (int)(blockDim.x >> 5); w++) v = k < 3 ? fminf(v, s_box[w][k]) : fmaxf(v, s_box[w][k]);
    if (k < 3)
      atomicMin(scene_keys + k, fkey(v));
    else
      atomicMax(scene_keys + k, fkey(v));
  }
}

__global__ void init_build_kernel(BNode *pool, BuildCounters *ctr, const uint32_t *scene_keys, uint32_t n,
                                  uint32_t min_leaf, uint32_t max_depth, uint32_t *active0, uint32_t *subtrees,
                                  uint32_t *mids) {
  BNode r;
  for (int k = 0; k < 3; k++) {
    r.bmin[k] = funkey(scene_keys[k]);
    r.bmax[k] = funkey(scene_keys[3 + k]);
  }
  r.l = 0;
  r.r = n;
  r.left = kInactive;
  r.depth = 0;
  r.rturns = 0;
  r.axis = 0;
  r.split_bin = 0;
  r.nleft = 0;
  r.slot = kInactive;
  r.pad = 0;
  ctr->pool = 1;
  ctr->n_active[0] = ctr->n_active[1] = 0;
  ctr->n_subtrees = 0;
  ctr->max_depth = 0;
  ctr->n_leaves = 0;
  ctr->error = 0;
  ctr->n_mids = 0;
  if (n <= min_leaf || max_depth == 0) {
    // single leaf
  } else if (n <= (uint32_t)kSubtree) {
    subtrees[0] = 0;
    ctr->n_subtrees = 1;
  } else if (n <= (uint32_t)kMid) {
    mids[0] = 0;
    ctr->n_mids = 1;
  } else {
    active0[0] = 0;
    r.slot = 0;
    ctr->n_active[0] = 1;
  }
  pool[0] = r;
}

__global__ void iota_kernel(uint32_t *a, uint32_t *b, uint32_t n) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    a[i] = i;
    b[i] = 0;
  }
}

// ------------------------------------------------------------------ phase A: binning
// Global bins: [slot][axis][bin][kBinWords] uint32 {count, kmin xyz, kmax xyz, -}
__global__ void __launch_bounds__(256)
    bin_large_kernel(const BNode *__restrict__ pool, const uint32_t *__restrict__ node_of,
                     const uint32_t *__restrict__ idx, const float4 *__restrict__ plo,
                     const float4 *__restrict__ phi, const float *__restrict__ pcz, uint32_t n, int B,
                     uint32_t *__restrict__ bins) {
  extern __shared__ uint32_t sbin[];  // 3*B*kBinWords when the tile lies inside one node
  const uint32_t tile0 = blockIdx.x * 1024u;
  const uint32_t tile1 = min(tile0 + 1024u, n);
  const uint32_t first_node = node_of[tile0];
  const bool uniform = (first_node == node_of[tile1 - 1]);
  if (uniform) {
    BNode nd = pool[first_node];
    if (nd.slot == kInactive) return;  // whole tile belongs to a finished / phase-B node
    for (int i = threadIdx.x; i < 3 * B * kBinWords; i += 256) {
      int w = i & (kBinWords - 1);
      sbin[i] = (w >= 1 && w <= 3) ? 0xFFFFFFFFu : 0u;
    }
    __syncthreads();
    float ivx = inv_extent(nd.bmin[0], nd.bmax[0], B), ivy = inv_extent(nd.bmin[1], nd.bmax[1], B),
          ivz = inv_extent(nd.bmin[2], nd.bmax[2], B);
    for (uint32_t p0 = tile0; p0 < tile1; p0 += 256) {  // whole warps iterate: the aggregation is warp-collective
      const uint32_t p = p0 + threadIdx.x;
      const bool valid = p < tile1;
      int b3[3] = {0, 0, 0};
      uint32_t kl[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}, kh[3] = {0u, 0u, 0u};
      if (valid) {
        uint32_t s = idx[p];
        float4 lo = plo[s], hi = phi[s];
        float cz = pcz[s];
        b3[0] = bin_of(lo.w, nd.bmin[0], ivx, B);
        b3[1] = bin_of(hi.w, nd.bmin[1], ivy, B);
        b3[2] = bin_of(cz, nd.bmin[2], ivz, B);
        kl[0] = fkey(lo.x), kl[1] = fkey(lo.y), kl[2] = fkey(lo.z);
        kh[0] = fkey(hi.x), kh[1] = fkey(hi.y), kh[2] = fkey(hi.z);
      }
#pragma unroll
      for (int a = 0; a < 3; a++)
        bin_add_aggregated(sbin + ((size_t)a * B + b3[a]) * kBinWords, (uint32_t)b3[a], valid, kl, kh);
    }
    __syncthreads();
    uint32_t *g = bins + (size_t)nd.slot * 3 * B * kBinWords;
    for (int i = threadIdx.x; i < 3 * B; i += 256) {
      const uint32_t *w = sbin + (size_t)i * kBinWords;
      if (w[0] == 0u) continue;
      uint32_t *gw = g + (size_t)i * kBinWords;
      atomicAdd(gw, w[0]);
#pragma unroll
      for (int k = 0; k < 3; k++) {
        atomicMin(gw + 1 + k, w[1 + k]);
        atomicMax(gw + 4 + k, w[4 + k]);
      }
    }
  } else {
    for (uint32_t p0 = tile0; p0 < tile1; p0 += 256) {
      const uint32_t p = p0 + threadIdx.x;
      bool valid = p < tile1;
      int b3[3] = {0, 0, 0};
      uint32_t kl[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}, kh[3] = {0u, 0u, 0u};
      uint32_t slot = 0;
      if (valid) {
        BNode nd = pool[node_of[p]];
        slot = nd.slot;
        valid = slot != kInactive;
        if (valid) {
          uint32_t s = idx[p];
          float4 lo = plo[s], hi = phi[s];
          float cz = pcz[s];
          b3[0] = bin_of(lo.w, nd.bmin[0], inv_extent(nd.bmin[0], nd.bmax[0], B), B);
          b3[1] = bin_of(hi.w, nd.bmin[1], inv_extent(nd.bmin[1], nd.bmax[1], B), B);
          b3[2] = bin_of(cz, nd.bmin[2], inv_extent(nd.bmin[2], nd.bmax[2], B), B);
          kl[0] = fkey(lo.x), kl[1] = fkey(lo.y), kl[2] = fkey(lo.z);
          kh[0] = fkey(hi.x), kh[1] = fkey(hi.y), kh[2] = fkey(hi.z);
        }
      }
      uint32_t *g = bins + (size_t)(valid ? slot : 0u) * 3 * B * kBinWords;
#pragma unroll
      for (int a = 0; a < 3; a++)  // key = record index: equal only for the same (node, axis, bin)
        bin_add_aggregated(g + ((size_t)a * B + b3[a]) * kBinWords, slot * (uint32_t)B + (uint32_t)b3[a], valid, kl, kh);
    }
  }
}

__global__ void clear_bins_kernel(uint32_t *bins, size_t words) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < words) {
    int w = (int)(i & (kBinWords - 1));
    bins[i] = (w >= 1 && w <= 3) ? 0xFFFFFFFFu : 0u;
  }
}

// Child bookkeeping shared by phases A and B (one thread).  Returns the class of the child:
// 0 leaf, 1 subtree (phase B), 2 large (phase A)
__device__ __forceinline__ int child_class(uint32_t n, uint32_t depth, uint32_t min_leaf, uint32_t max_depth) {
  if (n <= min_leaf || depth >= max_depth) return 0;
  return n <= (uint32_t)kSubtree ? 1 : 2;
}

// ------------------------------------------------------------------ phase A: split (one warp per node)
__global__ void __launch_bounds__(128)
    split_large_kernel(BNode *pool, BuildCounters *ctr, const uint32_t *__restrict__ active, int cur,
                       uint32_t *__restrict__ active_next, uint32_t *__restrict__ subtrees, uint32_t *__restrict__ mids,
                       uint32_t *bins, int B, uint32_t min_leaf, uint32_t max_depth) {
  extern __shared__ float scratch[];  // per warp: 2*B floats
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t a = blockIdx.x * 4 + warp;
  if (a >= ctr->n_active[cur]) return;
  const uint32_t nid = active[a];
  BNode nd = pool[nid];
  uint32_t *nb = bins + (size_t)a * 3 * B * kBinWords;
  float *cl = scratch + (size_t)warp * 2 * B, *cr = cl + B;
  float cost[3];
  int cut[3];
  for (int ax = 0; ax < 3; ax++) sweep_axis(nb + (size_t)ax * B * kBinWords, B, cl, cr, cost[ax], cut[ax]);
  int ax = 0;
  if (cost[0] > cost[1]) ax = 1;
  if (cost[ax] > cost[2]) ax = 2;
  const uint32_t n = nd.r - nd.l;
  Box6 lb, rb;
  uint32_t nl, nr;
  bool median = !(cost[ax] < FLT_MAX);
  if (!median) {
    range_union(nb + (size_t)ax * B * kBinWords, 0, cut[ax], lb, nl);
    range_union(nb + (size_t)ax * B * kBinWords, cut[ax], B, rb, nr);
  } else {
    nl = n >> 1;
    nr = n - nl;
    box_empty(lb);
    box_empty(rb);
    // the reference labels the node with the last axis it tried: (first + 2) % 3 (nanort.h:1833)
    ax = (ax + 2) % 3;
    // children boxes are gathered by the scatter pass into this node's (now free) bin words
    if (lane < 12) nb[lane] = (lane % 6) < 3 ? 0xFFFFFFFFu : 0u;
  }
  if (lane == 0) {
    uint32_t left = atomicAdd(&ctr->pool, 2u);
    nd.left = left;
    nd.axis = (uint32_t)ax;
    nd.split_bin = median ? kMedian : (uint32_t)cut[ax];
    nd.nleft = nl;
    pool[nid] = nd;
    for (int side = 0; side < 2; side++) {
      BNode c;
      const Box6 &bx = side ? rb : lb;
      for (int k = 0; k < 3; k++) {
        c.bmin[k] = bx.v[k];
        c.bmax[k] = bx.v[3 + k];
      }
      c.l = side ? nd.l + nl : nd.l;
      c.r = side ? nd.r : nd.l + nl;
      c.left = kInactive;
      c.depth = nd.depth + 1;
      c.rturns = nd.rturns + (uint32_t)side;
      c.axis = 0;
      c.split_bin = 0;
      c.nleft = 0;
      c.slot = kInactive;
      c.pad = 0;
      int cls = child_class(c.r - c.l, c.depth, min_leaf, max_depth);
      if (cls == 1) {
        subtrees[atomicAdd(&ctr->n_subtrees, 1u)] = left + side;
      } else if (cls == 2 && c.r - c.l <= (uint32_t)kMid) {
        mids[atomicAdd(&ctr->n_mids, 1u)] = left + side;  // its primitives drop out of the level-synchronous passes
      } else if (cls == 2) {
        uint32_t s = atomicAdd(&ctr->n_active[cur ^ 1], 1u);
        active_next[s] = left + side;
        c.slot = s;
      }
      pool[left + side] = c;
    }
  }
}

// ------------------------------------------------------------------ phase A: partition
__global__ void __launch_bounds__(256)
    flag_large_kernel(const BNode *__restrict__ pool, const uint32_t *__restrict__ node_of,
                      const uint32_t *__restrict__ idx, const float4 *__restrict__ plo,
                      const float4 *__restrict__ phi, const float *__restrict__ pcz, uint32_t n, int B,
                      uint32_t *__restrict__ flags) {
  uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const BNode nd = pool[node_of[p]];
  uint32_t f = 0;
  if (nd.slot != kInactive) {
    if (nd.split_bin == kMedian) {
      f = (p - nd.l) < nd.nleft;
    } else {
      uint32_t s = idx[p];
      float c = nd.axis == 0 ? plo[s].w : (nd.axis == 1 ? phi[s].w : pcz[s]);
      int b = bin_of(c, nd.bmin[nd.axis], inv_extent(nd.bmin[nd.axis], nd.bmax[nd.axis], B), B);
      f = (uint32_t)b < nd.split_bin;
    }
  }
  flags[p] = f;
}

__global__ void __launch_bounds__(256)
    scatter_large_kernel(const BNode *__restrict__ pool, const uint32_t *__restrict__ node_of,
                         const uint32_t *__restrict__ idx, const uint32_t *__restrict__ flags,
                         const uint32_t *__restrict__ scan, uint32_t n, uint32_t *__restrict__ node_of_out,
                         uint32_t *__restrict__ idx_out, const float4 *__restrict__ plo,
                         const float4 *__restrict__ phi, uint32_t *bins, int B) {
  uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint32_t nid = node_of[p];
  const BNode nd = pool[nid];
  if (nd.slot == kInactive) {
    node_of_out[p] = nid;
    idx_out[p] = idx[p];
    return;
  }
  const uint32_t before = scan[p] - scan[nd.l];  // lefts among [l, p)
  const uint32_t f = flags[p];
  const uint32_t dest = f ? nd.l + before : nd.l + nd.nleft + ((p - nd.l) - before);
  const uint32_t s = idx[p];
  idx_out[dest] = s;
  node_of_out[dest] = nd.left + (f ? 0u : 1u);
  if (nd.split_bin == kMedian) {
    // rare: children boxes of a median cut are gathered here (keys in the node's first 12 bin words)
    uint32_t *w = bins + (size_t)nd.slot * 3 * B * kBinWords + (f ? 0 : 6);
    float4 lo = plo[s], hi = phi[s];
    atomicMin(w + 0, fkey(lo.x));
    atomicMin(w + 1, fkey(lo.y));
    atomicMin(w + 2, fkey(lo.z));
    atomicMax(w + 3, fkey(hi.x));
    atomicMax(w + 4, fkey(hi.y));
    atomicMax(w + 5, fkey(hi.z));
  }
}

__global__ void fix_median_kernel(BNode *pool, const BuildCounters *ctr, const uint32_t *__restrict__ active, int cur,
                                  const uint32_t *__restrict__ bins, int B) {
  uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= ctr->n_active[cur]) return;
  const BNode nd = pool[active[a]];
  if (nd.split_bin != kMedian) return;
  const uint32_t *w = bins + (size_t)a * 3 * B * kBinWords;
  for (int side = 0; side < 2; side++) {
    BNode *c = pool + nd.left + side;
    for (int k = 0; k < 3; k++) {
      c->bmin[k] = funkey(w[side * 6 + k]);
      c->bmax[k] = funkey(w[side * 6 + 3 + k]);
    }
  }
}

__global__ void reset_count_kernel(BuildCounters *ctr, int which) { ctr->n_active[which] = 0; }

// ------------------------------------------------------------------ phase B: one WARP per subtree
// A subtree of at most kSubtree primitives is built to its leaves by a single warp, entirely out of that
// warp's slice of shared memory (primitive records, current order, bins, node stack) and with warp-level
// synchronisation only; a CTA is just kSubWarps independent warps.
struct WarpSub {
  float4 plo[kSubtree];
  float4 phi[kSubtree];
  float pcz[kSubtree];
  uint32_t gslot[kSubtree];  // global primitive slot of local primitive i
  // nodes still to split, as full descriptors {pool id, lo | n << 16, depth, rturns, box[6]}: the larger child is
  // parked and the smaller one split next, so the stack never holds more than log2(kSubtree) entries -- and no
  // split waits for a node record to come back from global memory
  uint32_t stack[kSubStack][10];
  uint16_t ids[kSubtree];    // current order (local ids) of the subtree's range
  uint16_t tmp[kSubtree];
};

// One warp's slice of subtree_kernel's shared memory: WarpSub, B bin records, 2*B sweep floats -- rounded up to 16
// bytes, because the next warp's WarpSub starts with float4 records (an odd bin_size would misalign them otherwise).
__host__ __device__ constexpr size_t sub_slice_bytes(int B) {
  return (sizeof(WarpSub) + (size_t)B * kBinWords * 4 + (size_t)2 * B * 4 + 15) & ~(size_t)15;
}

// Pool ids for one warp's subtree: reserved a chunk at a time (one atomic per chunk instead of one per split; the
// pre-order indices are computed in closed form in phase C, so pool order is free).  A subtree of t primitives has at
// most 2t - 2 nodes below its root and the reservations never exceed that, which keeps the whole pool within its 2n
// slots; what is left of the last chunk is marked dead for phase C.  All members are warp-uniform.
struct IdChunks {
  uint32_t next, end, cap_left;  // current chunk [next, end); slots this subtree may still reserve
  uint32_t next2, end2;          // a second chunk, while a request straddles two
  __device__ void init(BuildCounters *ctr, uint32_t total, int lane) {
    const uint32_t want = (total + 1u) & ~1u;  // enough whenever the leaves hold two primitives on average
    uint32_t b = 0;
    if (lane == 0) b = atomicAdd(&ctr->pool, want);
    next = __shfl_sync(0xFFFFFFFFu, b, 0);
    end = next + want;
    cap_left = 2u * total - 2u - want;  // want <= 2t - 2 for every t >= 2
    next2 = end2 = 0;
  }
  // makes `pairs` child pairs available: pair r lives at id(r), r < pairs; then call commit(pairs)
  __device__ void ensure(BuildCounters *ctr, uint32_t pairs, int lane) {
    const uint32_t need = 2u * pairs, avail = end - next;
    if (need > avail) {
      uint32_t chunk = need - avail < 32u ? 32u : need - avail;
      if (chunk > cap_left) chunk = cap_left;
      uint32_t b = 0;
      if (lane == 0) b = atomicAdd(&ctr->pool, chunk);
      next2 = __shfl_sync(0xFFFFFFFFu, b, 0);
      end2 = next2 + chunk;
      cap_left -= chunk;
    }
  }
  __device__ uint32_t id(uint32_t r) const {
    const uint32_t avail = end - next;  // even: ids are handed out in pairs
    return 2u * r < avail ? next + 2u * r : next2 + (2u * r - avail);
  }
  __device__ void commit(uint32_t pairs) {
    const uint32_t need = 2u * pairs, avail = end - next;
    if (need <= avail) {
      next += need;
    } else {
      next = next2 + (need - avail);
      end = end2;
      next2 = end2 = 0;
    }
  }
};

// the node a warp is splitting: warp-uniform registers
struct SubNode {
  uint32_t nid, lo, n, depth, rturns;
  float bmin[3], bmax[3];
};

// A node with at most 32 primitives, built to its leaves level by level: one primitive per lane, every node of the
// current level is a SEGMENT of consecutive lanes, and one pass of segmented warp operations splits them all -- per
// axis a 32-lane bitonic sort by (segment, bin), prefix / suffix box scans that stop at segment borders, candidates
// where the bin changes, a segmented argmin.  Same candidates, cost arithmetic and tie rules as the binned sweep
// (lowest boundary, then lowest axis), so the tree is the one a split-at-a-time build produces; a 32-primitive node
// takes three passes instead of seven splits.
__device__ void small_block(const SubNode &root, BNode *pool, BuildCounters *ctr, IdChunks &ids, WarpSub &S, uint32_t base,
                            int B, uint32_t min_leaf, uint32_t max_depth, int lane) {
  const unsigned FULL = 0xFFFFFFFFu;
  const unsigned lt = (1u << lane) - 1u;
  const bool valid = (uint32_t)lane < root.n;
  // segment state, identical in all lanes of a segment (lanes beyond the node: a dead segment of their own)
  uint32_t seg_start = valid ? 0u : (uint32_t)lane, seg_len = valid ? root.n : 1u;
  uint32_t seg_nid = root.nid, seg_depth = root.depth, seg_rturns = root.rturns;
  float sb_min[3] = {root.bmin[0], root.bmin[1], root.bmin[2]}, sb_max[3] = {root.bmax[0], root.bmax[1], root.bmax[2]};
  uint32_t q = valid ? (uint32_t)S.ids[root.lo + lane] : 0u;
  for (;;) {
    const bool active = valid && child_class(seg_len, seg_depth, min_leaf, max_depth) != 0;
    const unsigned act = __ballot_sync(FULL, active);
    if (act == 0u) break;
    const uint32_t seg_end = seg_start + seg_len;
    Box6 mine;
    box_empty(mine);
    float c3[3] = {0.0f, 0.0f, 0.0f};
    if (valid) {
      const float4 l4 = S.plo[q], h4 = S.phi[q];
      mine.v[0] = l4.x, mine.v[1] = l4.y, mine.v[2] = l4.z, mine.v[3] = h4.x, mine.v[4] = h4.y, mine.v[5] = h4.z;
      c3[0] = l4.w, c3[1] = h4.w, c3[2] = S.pcz[q];
    }
    const uint32_t maxlen = __reduce_max_sync(FULL, active ? seg_len : 0u);  // scans need ceil(log2(maxlen)) rounds
    float best = FLT_MAX;
    int ax = 0, cutbin = 0;
    uint32_t nl = 0;
    Box6 lb, rb;
    box_empty(lb);
    box_empty(rb);
    uint32_t mybin[3];
#pragma unroll
    for (int a = 0; a < 3; a++) {
      const float iv = inv_extent(sb_min[a], sb_max[a], B);
      const uint32_t bin = active ? (uint32_t)bin_of(c3[a], sb_min[a], iv, B) : 0u;
      mybin[a] = bin;
      uint32_t key = (seg_start << 13) | (bin << 5) | (uint32_t)lane;  // segments keep their lane ranges
#pragma unroll
      for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
          const uint32_t other = __shfl_xor_sync(FULL, key, j);
          const bool keep_min = ((lane & k) == 0) == ((lane & j) == 0);
          key = keep_min ? min(key, other) : max(key, other);
        }
      }
      const int src = (int)(key & 31u);
      const uint32_t sb = (key >> 5) & 0xFFu;
      Box6 pre, suf;
#pragma unroll
      for (int k = 0; k < 6; k++) pre.v[k] = suf.v[k] = __shfl_sync(FULL, mine.v[k], src);
      for (uint32_t o = 1; o < maxlen; o <<= 1) {
        Box6 t, u;
#pragma unroll
        for (int k = 0; k < 6; k++) {
          t.v[k] = __shfl_up_sync(FULL, pre.v[k], o);
          u.v[k] = __shfl_down_sync(FULL, suf.v[k], o);
        }
        if ((uint32_t)lane >= seg_start + o) box_merge(pre, t);
        if ((uint32_t)lane + o < seg_end) box_merge(suf, u);
      }
      Box6 epre;
#pragma unroll
      for (int k = 0; k < 6; k++) epre.v[k] = __shfl_up_sync(FULL, pre.v[k], 1);
      const uint32_t prev_bin = __shfl_up_sync(FULL, sb, 1);
      const bool cand = active && (uint32_t)lane > seg_start && sb != prev_bin;
      float bc = FLT_MAX;
      int bp = 0x7FFFFFFF;
      if (cand) {
        bc = (float)((uint32_t)lane - seg_start) * box_area(epre.v[0], epre.v[1], epre.v[2], epre.v[3], epre.v[4], epre.v[5]) +
             (float)(seg_end - (uint32_t)lane) * box_area(suf.v[0], suf.v[1], suf.v[2], suf.v[3], suf.v[4], suf.v[5]);
        bp = lane;
      }
      // segmented argmin (lowest position among equal costs): inclusive prefix-min, read at the segment's last lane
      for (uint32_t o = 1; o < maxlen; o <<= 1) {
        const float oc = __shfl_up_sync(FULL, bc, o);
        const int op = __shfl_up_sync(FULL, bp, o);
        if ((uint32_t)lane >= seg_start + o && (oc < bc || (oc == bc && op < bp))) {
          bc = oc;
          bp = op;
        }
      }
      bc = __shfl_sync(FULL, bc, (int)(seg_end - 1u));
      bp = __shfl_sync(FULL, bp, (int)(seg_end - 1u));
      const int bsrc = bp & 31;  // 0x7FFFFFFF (no candidate) reads lane 31: ignored below
      const uint32_t cb = __shfl_sync(FULL, prev_bin, bsrc) + 1u;
      Box6 cl, cr;
#pragma unroll
      for (int k = 0; k < 6; k++) {
        cl.v[k] = __shfl_sync(FULL, epre.v[k], bsrc);
        cr.v[k] = __shfl_sync(FULL, suf.v[k], bsrc);
      }
      if (bc < best) {  // uniform within a segment; strict, so a tie keeps the lower axis
        best = bc;
        ax = a;
        cutbin = (int)cb;
        nl = (uint32_t)bp - seg_start;
        lb = cl;
        rb = cr;
      }
    }
    const bool median = active && !(best < FLT_MAX);
    if (__any_sync(FULL, median)) {
      // no plane separates the centroids: cut at the median index of the current order, exact boxes of the halves
      Box6 pre = mine, suf = mine;
      for (uint32_t o = 1; o < maxlen; o <<= 1) {
        Box6 t, u;
#pragma unroll
        for (int k = 0; k < 6; k++) {
          t.v[k] = __shfl_up_sync(FULL, pre.v[k], o);
          u.v[k] = __shfl_down_sync(FULL, suf.v[k], o);
        }
        if ((uint32_t)lane >= seg_start + o) box_merge(pre, t);
        if ((uint32_t)lane + o < seg_end) box_merge(suf, u);
      }
      const uint32_t half = seg_len >> 1;
      const int ls = (int)((seg_start + half - 1u) & 31u), rs = (int)((seg_start + half) & 31u);
      Box6 ml, mr;
#pragma unroll
      for (int k = 0; k < 6; k++) {
        ml.v[k] = __shfl_sync(FULL, pre.v[k], ls);
        mr.v[k] = __shfl_sync(FULL, suf.v[k], rs);
      }
      if (median) {
        nl = half;
        lb = ml;
        rb = mr;
      }
    }
    // ---- stable partition inside every segment
    const uint32_t segmask = (seg_len >= 32u ? 0xFFFFFFFFu : ((1u << seg_len) - 1u)) << seg_start;
    const uint32_t mb = ax == 0 ? mybin[0] : (ax == 1 ? mybin[1] : mybin[2]);
    const bool f = median ? ((uint32_t)lane - seg_start) < nl : mb < (uint32_t)cutbin;
    const unsigned mf = __ballot_sync(FULL, active && f) & segmask, mr_ = __ballot_sync(FULL, active && !f) & segmask;
    if (active) {
      const uint32_t pos = f ? seg_start + (uint32_t)__popc(mf & lt) : seg_start + nl + (uint32_t)__popc(mr_ & lt);
      S.ids[root.lo + pos] = (uint16_t)q;
    }
    // ---- node records: the segment's first lane completes the parent and writes the left child, its second lane the
    // right child (an active segment has at least two primitives)
    const unsigned leaders = __ballot_sync(FULL, active && (uint32_t)lane == seg_start);
    const uint32_t pairs = (uint32_t)__popc(leaders);
    ids.ensure(ctr, pairs, lane);
    const uint32_t left = ids.id((uint32_t)__popc(leaders & ((seg_start >= 32u ? 0u : (1u << seg_start)) - 1u)));
    ids.commit(pairs);
    if (active) {
      const uint32_t rel = (uint32_t)lane - seg_start;
      if (rel == 0u) {
        BNode *me = pool + seg_nid;
        me->left = left;
        me->axis = (uint32_t)(median ? (ax + 2) % 3 : ax);
        me->split_bin = median ? kMedian : (uint32_t)cutbin;
        me->nleft = nl;
      }
      if (rel < 2u) {
        const Box6 &bx = rel ? rb : lb;
        BNode c;
        for (int k = 0; k < 3; k++) {
          c.bmin[k] = bx.v[k];
          c.bmax[k] = bx.v[3 + k];
        }
        c.l = base + root.lo + seg_start + (rel ? nl : 0u);
        c.r = base + root.lo + seg_start + (rel ? seg_len : nl);
        c.left = kInactive;
        c.depth = seg_depth + 1u;
        c.rturns = seg_rturns + rel;
        c.axis = 0;
        c.split_bin = 0;
        c.nleft = 0;
        c.slot = kInactive;
        c.pad = 0;
        pool[left + rel] = c;
      }
      // the lane now stands for the primitive at ITS position of the new order: which child is that?
      const uint32_t side = rel < nl ? 0u : 1u;
      const Box6 &nb = side ? rb : lb;
      seg_nid = left + side;
      seg_depth += 1u;
      seg_rturns += side;
      seg_len = side ? seg_len - nl : nl;
      seg_start = side ? seg_start + nl : seg_start;
      for (int k = 0; k < 3; k++) {
        sb_min[k] = nb.v[k];
        sb_max[k] = nb.v[3 + k];
      }
    }
    __syncwarp();
    if (valid) q = (uint32_t)S.ids[root.lo + lane];
  }
}

// ------------------------------------------------------------------ middle phase: one CTA per node
// Nodes of kSubtree+1 .. kMid primitives are split down to phase-B subtrees by one CTA each, entirely on chip: the
// level-synchronous passes of phase A touch all n primitives per level and bin such small nodes with global atomics
// (a 1024-slot tile spans several of them) -- seven of the 21 levels of a 10 M-triangle build, and the slowest ones.
// Same bins, sweep, tie rules and stable partition as phases A and B (shared code), so the tree does not change.
struct MidShared {
  uint32_t gslot[kMid];  // global primitive slot of local primitive i
  uint16_t ids[kMid];    // current order (local ids)
  uint16_t tmp[kMid];
  uint32_t stack[8][10];  // parked nodes: {pool id, lo | n << 16, depth, rturns, box[6]}
  float cost[3];
  int cut[3];
  float box[2][6];
  uint32_t cnt[2];
  uint32_t wcnt[2][kMidThreads / 32];
  uint32_t mkeys[12];
  uint32_t left;
};

__global__ void __launch_bounds__(kMidThreads)
    midtree_kernel(BNode *pool, BuildCounters *ctr, const uint32_t *__restrict__ mids, uint32_t *__restrict__ idx,
                   const float4 *__restrict__ plo, const float4 *__restrict__ phi, const float *__restrict__ pcz, int B,
                   uint32_t min_leaf, uint32_t max_depth, uint32_t *__restrict__ subtrees) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  MidShared &S = *reinterpret_cast<MidShared *>(smem_raw);
  uint32_t *sbin = reinterpret_cast<uint32_t *>(smem_raw + sizeof(MidShared));  // 3 * B * kBinWords
  float *sweep = reinterpret_cast<float *>(sbin + (size_t)3 * B * kBinWords);   // 3 * 2 * B floats
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const unsigned lt = (1u << lane) - 1u;
  const uint32_t root = mids[blockIdx.x];
  const BNode rootn = pool[root];
  const uint32_t base = rootn.l, total = rootn.r - rootn.l;
  for (uint32_t i = tid; i < total; i += kMidThreads) {
    S.gslot[i] = idx[base + i];
    S.ids[i] = (uint16_t)i;
  }
  SubNode nd;  // CTA-uniform registers
  nd.nid = root;
  nd.lo = 0;
  nd.n = total;
  nd.depth = rootn.depth;
  nd.rturns = rootn.rturns;
  for (int k = 0; k < 3; k++) {
    nd.bmin[k] = rootn.bmin[k];
    nd.bmax[k] = rootn.bmax[k];
  }
  int sp = 0;
  __syncthreads();

  for (;;) {
    const uint32_t nid = nd.nid, lo = nd.lo, n = nd.n;
    const float iv[3] = {inv_extent(nd.bmin[0], nd.bmax[0], B), inv_extent(nd.bmin[1], nd.bmax[1], B),
                         inv_extent(nd.bmin[2], nd.bmax[2], B)};
    // ---- bins of the three axes
    for (int i = tid; i < 3 * B * kBinWords; i += kMidThreads) {
      const int w = i & (kBinWords - 1);
      sbin[i] = (w >= 1 && w <= 3) ? 0xFFFFFFFFu : 0u;
    }
    if (tid < 12) S.mkeys[tid] = (tid % 6) < 3 ? 0xFFFFFFFFu : 0u;
    __syncthreads();
    for (uint32_t i0 = 0; i0 < n; i0 += kMidThreads) {  // whole warps iterate: the aggregation is warp-collective
      const uint32_t i = i0 + tid;
      const bool valid = i < n;
      int b3[3] = {0, 0, 0};
      uint32_t kl[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}, kh[3] = {0u, 0u, 0u};
      if (valid) {
        const uint32_t s = S.gslot[S.ids[lo + i]];
        const float4 l4 = plo[s], h4 = phi[s];
        const float cz = pcz[s];
        b3[0] = bin_of(l4.w, nd.bmin[0], iv[0], B);
        b3[1] = bin_of(h4.w, nd.bmin[1], iv[1], B);
        b3[2] = bin_of(cz, nd.bmin[2], iv[2], B);
        kl[0] = fkey(l4.x), kl[1] = fkey(l4.y), kl[2] = fkey(l4.z);
        kh[0] = fkey(h4.x), kh[1] = fkey(h4.y), kh[2] = fkey(h4.z);
      }
#pragma unroll
      for (int a = 0; a < 3; a++)
        bin_add_aggregated(sbin + ((size_t)a * B + b3[a]) * kBinWords, (uint32_t)b3[a], valid, kl, kh);
    }
    __syncthreads();
    // ---- sweep: one warp per axis
    if (warp < 3) {
      float c;
      int k;
      sweep_axis(sbin + (size_t)warp * B * kBinWords, B, sweep + (size_t)warp * 2 * B, sweep + (size_t)warp * 2 * B + B, c, k);
      if (lane == 0) {
        S.cost[warp] = c;
        S.cut[warp] = k;
      }
    }
    __syncthreads();
    int ax = 0;
    if (S.cost[0] > S.cost[1]) ax = 1;
    if (S.cost[ax] > S.cost[2]) ax = 2;
    const bool median = !(S.cost[ax] < FLT_MAX);
    const int cut = S.cut[ax];
    uint32_t nl;
    if (!median) {
      if (warp < 2) {  // child boxes: exact unions of the chosen axis' bins
        Box6 bx;
        uint32_t c;
        range_union(sbin + (size_t)ax * B * kBinWords, warp ? cut : 0, warp ? B : cut, bx, c);
        if (lane == 0) {
          for (int k = 0; k < 6; k++) S.box[warp][k] = bx.v[k];
          S.cnt[warp] = c;
        }
      }
      __syncthreads();
      nl = S.cnt[0];
    } else {
      nl = n >> 1;  // no plane separates the centroids: cut at the median index, exact boxes of the halves
      Box6 hb[2];
      box_empty(hb[0]);
      box_empty(hb[1]);
      for (uint32_t i = tid; i < n; i += kMidThreads) {
        const uint32_t s = S.gslot[S.ids[lo + i]];
        const float4 l4 = plo[s], h4 = phi[s];
        Box6 &t = i < nl ? hb[0] : hb[1];
        t.v[0] = fminf(t.v[0], l4.x);
        t.v[1] = fminf(t.v[1], l4.y);
        t.v[2] = fminf(t.v[2], l4.z);
        t.v[3] = fmaxf(t.v[3], h4.x);
        t.v[4] = fmaxf(t.v[4], h4.y);
        t.v[5] = fmaxf(t.v[5], h4.z);
      }
      for (int h = 0; h < 2; h++)
        for (int k = 0; k < 6; k++) {
          float v = hb[h].v[k];
          for (int o = 16; o > 0; o >>= 1) {
            const float w = __shfl_xor_sync(0xFFFFFFFFu, v, o);
            v = k < 3 ? fminf(v, w) : fmaxf(v, w);
          }
          if (lane == 0) {
            if (k < 3)
              atomicMin(&S.mkeys[h * 6 + k], fkey(v));
            else
              atomicMax(&S.mkeys[h * 6 + k], fkey(v));
          }
        }
      __syncthreads();
      if (tid < 12) S.box[tid / 6][tid % 6] = funkey(S.mkeys[tid]);
      __syncthreads();
    }
    // ---- stable partition of ids[lo, lo+n)
    {
      uint32_t done_l = 0, done_r = 0;
      for (uint32_t i0 = 0; i0 < n; i0 += kMidThreads) {
        const uint32_t i = i0 + tid;
        const bool valid = i < n;
        uint32_t q = 0;
        bool f = false;
        if (valid) {
          q = S.ids[lo + i];
          if (median) {
            f = i < nl;
          } else {
            const uint32_t s = S.gslot[q];
            const float c = ax == 0 ? plo[s].w : (ax == 1 ? phi[s].w : pcz[s]);
            f = (uint32_t)bin_of(c, nd.bmin[ax], iv[ax], B) < (uint32_t)cut;
          }
        }
        const unsigned ml = __ballot_sync(0xFFFFFFFFu, valid && f), mr = __ballot_sync(0xFFFFFFFFu, valid && !f);
        if (lane == 0) {
          S.wcnt[0][warp] = (uint32_t)__popc(ml);
          S.wcnt[1][warp] = (uint32_t)__popc(mr);
        }
        __syncthreads();
        uint32_t offl = 0, offr = 0, totl = 0, totr = 0;
#pragma unroll
        for (int w = 0; w < kMidThreads / 32; w++) {
          const uint32_t a = S.wcnt[0][w], b = S.wcnt[1][w];
          if (w < warp) {
            offl += a;
            offr += b;
          }
          totl += a;
          totr += b;
        }
        if (valid) {
          if (f)
            S.tmp[lo + done_l + offl + __popc(ml & lt)] = (uint16_t)q;
          else
            S.tmp[lo + nl + done_r + offr + __popc(mr & lt)] = (uint16_t)q;
        }
        done_l += totl;
        done_r += totr;
        __syncthreads();
      }
      for (uint32_t i = tid; i < n; i += kMidThreads) S.ids[lo + i] = S.tmp[lo + i];
    }
    // ---- children
    if (tid == 0) S.left = atomicAdd(&ctr->pool, 2u);
    __syncthreads();
    const uint32_t left = S.left;
    const uint32_t cdepth = nd.depth + 1;
    const uint32_t n_side[2] = {nl, n - nl};
    const int cls0 = child_class(n_side[0], cdepth, min_leaf, max_depth), cls1 = child_class(n_side[1], cdepth, min_leaf, max_depth);
    if (tid == 0) {
      BNode *me = pool + nid;
      me->left = left;
      me->axis = (uint32_t)(median ? (ax + 2) % 3 : ax);
      me->split_bin = median ? kMedian : (uint32_t)cut;
      me->nleft = nl;
    }
    if (tid < 2) {
      const int side = tid;
      BNode c;
      for (int k = 0; k < 3; k++) {
        c.bmin[k] = S.box[side][k];
        c.bmax[k] = S.box[side][3 + k];
      }
      c.l = base + lo + (side ? nl : 0u);
      c.r = base + lo + (side ? n : nl);
      c.left = kInactive;
      c.depth = cdepth;
      c.rturns = nd.rturns + (uint32_t)side;
      c.axis = 0;
      c.split_bin = 0;
      c.nleft = 0;
      c.slot = kInactive;
      c.pad = 0;
      pool[left + side] = c;
      if ((side ? cls1 : cls0) == 1) subtrees[atomicAdd(&ctr->n_subtrees, 1u)] = left + side;
    }
    // next node: a child that is still too large for a warp (the smaller one first), else a parked node
    const bool more0 = cls0 == 2, more1 = cls1 == 2;
    Box6 cb[2];
    for (int k = 0; k < 6; k++) {
      cb[0].v[k] = S.box[0][k];
      cb[1].v[k] = S.box[1][k];
    }
    if (more0 || more1) {
      const int go = (more0 && more1) ? (n_side[1] < n_side[0] ? 1 : 0) : (more1 ? 1 : 0);
      if (more0 && more1) {
        const int park = go ^ 1;
        if (tid == 0) {
          uint32_t *e = S.stack[sp];
          e[0] = left + (uint32_t)park;
          e[1] = (lo + (park ? nl : 0u)) | (n_side[park] << 16);
          e[2] = cdepth;
          e[3] = nd.rturns + (uint32_t)park;
          for (int k = 0; k < 6; k++) e[4 + k] = __float_as_uint(cb[park].v[k]);
        }
        sp++;
      }
      nd.nid = left + (uint32_t)go;
      nd.lo = lo + (go ? nl : 0u);
      nd.n = n_side[go];
      nd.depth = cdepth;
      nd.rturns = nd.rturns + (uint32_t)go;
      for (int k = 0; k < 3; k++) {
        nd.bmin[k] = cb[go].v[k];
        nd.bmax[k] = cb[go].v[3 + k];
      }
    } else {
      if (sp == 0) break;
      --sp;
      __syncthreads();
      const uint32_t *e = S.stack[sp];
      nd.nid = e[0];
      nd.lo = e[1] & 0xFFFFu;
      nd.n = e[1] >> 16;
      nd.depth = e[2];
      nd.rturns = e[3];
      for (int k = 0; k < 3; k++) {
        nd.bmin[k] = __uint_as_float(e[4 + k]);
        nd.bmax[k] = __uint_as_float(e[7 + k]);
      }
    }
    __syncthreads();
  }
  __syncthreads();
  for (uint32_t i = tid; i < total; i += kMidThreads) idx[base + i] = S.gslot[S.ids[i]];
}

__global__ void __launch_bounds__(kSubWarps * 32, 6)
    subtree_kernel(BNode *pool, BuildCounters *ctr, const uint32_t *__restrict__ subtrees, uint32_t n_subtrees,
                   uint32_t *__restrict__ idx, const float4 *__restrict__ plo, const float4 *__restrict__ phi,
                   const float *__restrict__ pcz, int B, uint32_t min_leaf, uint32_t max_depth) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t sub = blockIdx.x * kSubWarps + warp;
  if (sub >= n_subtrees) return;
  unsigned char *mine = smem_raw + (size_t)warp * sub_slice_bytes(B);
  WarpSub &S = *reinterpret_cast<WarpSub *>(mine);
  uint32_t *sbin = reinterpret_cast<uint32_t *>(mine + sizeof(WarpSub));  // B*kBinWords: one axis at a time
  float *sweep = reinterpret_cast<float *>(sbin + (size_t)B * kBinWords);  // 2*B floats
  const uint32_t root = subtrees[sub];
  const BNode rootn = pool[root];
  const uint32_t base = rootn.l, total = rootn.r - rootn.l;
  for (uint32_t i = lane; i < total; i += 32) {
    const uint32_t s = idx[base + i];
    S.gslot[i] = s;
    S.plo[i] = plo[s];
    S.phi[i] = phi[s];
    S.pcz[i] = pcz[s];
    S.ids[i] = (uint16_t)i;
  }
  IdChunks ids;
  ids.init(ctr, total, lane);
  SubNode nd;
  nd.nid = root;
  nd.lo = 0;
  nd.n = total;
  nd.depth = rootn.depth;
  nd.rturns = rootn.rturns;
  for (int k = 0; k < 3; k++) {
    nd.bmin[k] = rootn.bmin[k];
    nd.bmax[k] = rootn.bmax[k];
  }
  int sp = 0;  // warp-uniform
  __syncwarp();

  for (;;) {
    bool pop = false;
    if (nd.n <= 32u) {
      small_block(nd, pool, ctr, ids, S, base, B, min_leaf, max_depth, lane);
      pop = true;
    } else {
      // ---- more than 32 primitives (3 of the 31 splits of a full subtree): bin ONE axis at a time into a single
      // B-bin array -- a third of the shared memory, i.e. half again as many resident warps for the whole kernel
      const uint32_t nid = nd.nid, lo = nd.lo, n = nd.n;
      const float iv[3] = {inv_extent(nd.bmin[0], nd.bmax[0], B), inv_extent(nd.bmin[1], nd.bmax[1], B),
                           inv_extent(nd.bmin[2], nd.bmax[2], B)};
      auto bin_axis = [&](int a) {
        for (int i = lane; i < B * kBinWords; i += 32) {
          const int w = i & (kBinWords - 1);
          sbin[i] = (w >= 1 && w <= 3) ? 0xFFFFFFFFu : 0u;
        }
        __syncwarp();
        for (uint32_t i = lane; i < n; i += 32) {
          const uint32_t q = S.ids[lo + i];
          const float4 l4 = S.plo[q], h4 = S.phi[q];
          const float c = a == 0 ? l4.w : (a == 1 ? h4.w : S.pcz[q]);
          uint32_t *w = sbin + (size_t)bin_of(c, nd.bmin[a], iv[a], B) * kBinWords;
          atomicAdd(w, 1u);
          atomicMin(w + 1, fkey(l4.x));
          atomicMin(w + 2, fkey(l4.y));
          atomicMin(w + 3, fkey(l4.z));
          atomicMax(w + 4, fkey(h4.x));
          atomicMax(w + 5, fkey(h4.y));
          atomicMax(w + 6, fkey(h4.z));
        }
        __syncwarp();
      };
      float cost[3];
      int cut[3];
      int ax = 0;
      Box6 lb, rb;
      uint32_t nl = 0, nr = 0;
      for (int a = 0; a < 3; a++) {
        bin_axis(a);
        sweep_axis(sbin, B, sweep, sweep + B, cost[a], cut[a]);
      }
      if (cost[0] > cost[1]) ax = 1;
      if (cost[ax] > cost[2]) ax = 2;
      if (ax != 2 && cost[ax] < FLT_MAX) bin_axis(ax);  // the child boxes come from the chosen axis' bins
      const bool median = !(cost[ax] < FLT_MAX);
      if (!median) {
        range_union(sbin, 0, cut[ax], lb, nl);
        range_union(sbin, cut[ax], B, rb, nr);
      } else {
        nl = n >> 1;
        box_empty(lb);
        box_empty(rb);
        for (uint32_t i = lane; i < n; i += 32) {  // exact boxes of the two halves of the current order
          const uint32_t q = S.ids[lo + i];
          const float4 l4 = S.plo[q], h4 = S.phi[q];
          Box6 &t = i < nl ? lb : rb;
          t.v[0] = fminf(t.v[0], l4.x);
          t.v[1] = fminf(t.v[1], l4.y);
          t.v[2] = fminf(t.v[2], l4.z);
          t.v[3] = fmaxf(t.v[3], h4.x);
          t.v[4] = fmaxf(t.v[4], h4.y);
          t.v[5] = fmaxf(t.v[5], h4.z);
        }
        for (int o = 16; o > 0; o >>= 1) {
          for (int k = 0; k < 3; k++) {
            lb.v[k] = fminf(lb.v[k], __shfl_xor_sync(0xFFFFFFFFu, lb.v[k], o));
            rb.v[k] = fminf(rb.v[k], __shfl_xor_sync(0xFFFFFFFFu, rb.v[k], o));
            lb.v[3 + k] = fmaxf(lb.v[3 + k], __shfl_xor_sync(0xFFFFFFFFu, lb.v[3 + k], o));
            rb.v[3 + k] = fmaxf(rb.v[3 + k], __shfl_xor_sync(0xFFFFFFFFu, rb.v[3 + k], o));
          }
        }
      }
      // ---- stable partition of ids[lo, lo+n) by warp ballots
      {
        uint32_t done_l = 0, done_r = 0;
        for (uint32_t i0 = 0; i0 < n; i0 += 32) {
          const uint32_t i = i0 + lane;
          const bool valid = i < n;
          uint32_t q = 0;
          bool f = false;
          if (valid) {
            q = S.ids[lo + i];
            if (median) {
              f = i < nl;
            } else {
              const float c = ax == 0 ? S.plo[q].w : (ax == 1 ? S.phi[q].w : S.pcz[q]);
              f = (uint32_t)bin_of(c, nd.bmin[ax], iv[ax], B) < (uint32_t)cut[ax];
            }
          }
          const unsigned ml = __ballot_sync(0xFFFFFFFFu, valid && f), mr = __ballot_sync(0xFFFFFFFFu, valid && !f);
          const unsigned lt = (1u << lane) - 1u;
          if (valid) {
            if (f)
              S.tmp[lo + done_l + __popc(ml & lt)] = (uint16_t)q;
            else
              S.tmp[lo + nl + done_r + __popc(mr & lt)] = (uint16_t)q;
          }
          done_l += __popc(ml);
          done_r += __popc(mr);
        }
        __syncwarp();
        for (uint32_t i = lane; i < n; i += 32) S.ids[lo + i] = S.tmp[lo + i];
      }
      // ---- children
      ids.ensure(ctr, 1u, lane);
      const uint32_t left = ids.id(0u);
      ids.commit(1u);
      const uint32_t cdepth = nd.depth + 1;
      const uint32_t n_side[2] = {nl, n - nl};
      if (lane == 0) {  // the parent's record is complete now; range, box, depth, right turns came from its own parent
        BNode *me = pool + nid;
        me->left = left;
        me->axis = (uint32_t)(median ? (ax + 2) % 3 : ax);
        me->split_bin = median ? kMedian : (uint32_t)cut[ax];
        me->nleft = nl;
      }
      if (lane < 2) {
        const int side = lane;
        const Box6 &bx = side ? rb : lb;
        BNode c;
        for (int k = 0; k < 3; k++) {
          c.bmin[k] = bx.v[k];
          c.bmax[k] = bx.v[3 + k];
        }
        c.l = base + lo + (side ? nl : 0u);
        c.r = base + lo + (side ? n : nl);
        c.left = kInactive;
        c.depth = cdepth;
        c.rturns = nd.rturns + (uint32_t)side;
        c.axis = 0;
        c.split_bin = 0;
        c.nleft = 0;
        c.slot = kInactive;
        c.pad = 0;
        pool[left + side] = c;
      }
      // next node: a child that still splits (the smaller one first, the other parked), else a parked node
      const bool more0 = child_class(n_side[0], cdepth, min_leaf, max_depth) != 0;
      const bool more1 = child_class(n_side[1], cdepth, min_leaf, max_depth) != 0;
      if (more0 || more1) {
        const int go = (more0 && more1) ? (n_side[1] < n_side[0] ? 1 : 0) : (more1 ? 1 : 0);
        if (more0 && more1) {
          const int park = go ^ 1;
          const Box6 &pb = park ? rb : lb;
          if (lane == 0) {
            uint32_t *e = S.stack[sp];
            e[0] = left + (uint32_t)park;
            e[1] = (lo + (park ? nl : 0u)) | (n_side[park] << 16);
            e[2] = cdepth;
            e[3] = nd.rturns + (uint32_t)park;
            for (int k = 0; k < 6; k++) e[4 + k] = __float_as_uint(pb.v[k]);
          }
          sp++;
        }
        const Box6 &gb = go ? rb : lb;
        nd.nid = left + (uint32_t)go;
        nd.lo = lo + (go ? nl : 0u);
        nd.n = n_side[go];
        nd.depth = cdepth;
        nd.rturns = nd.rturns + (uint32_t)go;
        for (int k = 0; k < 3; k++) {
          nd.bmin[k] = gb.v[k];
          nd.bmax[k] = gb.v[3 + k];
        }
      } else {
        pop = true;
      }
    }
    if (pop) {
      if (sp == 0) break;
      --sp;
      __syncwarp();
      const uint32_t *e = S.stack[sp];
      nd.nid = e[0];
      nd.lo = e[1] & 0xFFFFu;
      nd.n = e[1] >> 16;
      nd.depth = e[2];
      nd.rturns = e[3];
      for (int k = 0; k < 3; k++) {
        nd.bmin[k] = __uint_as_float(e[4 + k]);
        nd.bmax[k] = __uint_as_float(e[7 + k]);
      }
    }
    __syncwarp();
  }
  // reserved slots this subtree did not need
  for (uint32_t i = ids.next + lane; i < ids.end; i += 32) pool[i].depth = kDeadNode;
  // final order of this subtree's range
  for (uint32_t i = lane; i < total; i += 32) idx[base + i] = S.gslot[S.ids[i]];
}

// ------------------------------------------------------------------ phase C: emission
__global__ void mark_leaves_kernel(const BNode *__restrict__ pool, uint32_t n_nodes, uint32_t *__restrict__ leaf_start,
                                   BuildCounters *ctr) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t depth = 0, leaf = 0;
  if (i < n_nodes && pool[i].depth != kDeadNode) {
    const BNode nd = pool[i];
    depth = nd.depth;
    if (nd.left == kInactive) {
      leaf_start[nd.l] = 1u;
      leaf = 1;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    depth = max(depth, __shfl_xor_sync(0xFFFFFFFFu, depth, o));
    leaf += __shfl_xor_sync(0xFFFFFFFFu, leaf, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMax(&ctr->max_depth, depth);
    if (leaf) atomicAdd(&ctr->n_leaves, leaf);
  }
}

// pre-order index of a node = 2*(leaves starting before its range) - right turns + depth
__global__ void emit_nodes_kernel(const BNode *__restrict__ pool, uint32_t n_nodes,
                                  const uint32_t *__restrict__ leaves_before, Node40 *__restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_nodes) return;
  const BNode nd = pool[i];
  if (nd.depth == kDeadNode) return;  // reserved by a subtree, never used
  const uint32_t lb = leaves_before[nd.l];
  const uint32_t pre = 2u * lb - nd.rturns + nd.depth;
  Node40 o;
  for (int k = 0; k < 3; k++) {
    o.bmin[k] = nd.bmin[k];
    o.bmax[k] = nd.bmax[k];
  }
  if (nd.left == kInactive) {
    o.flag = 1;
    o.axis = 0;
    o.data[0] = nd.r - nd.l;
    o.data[1] = nd.l;
  } else {
    o.flag = 0;
    o.axis = (int32_t)nd.axis;
    const uint32_t mid = nd.l + nd.nleft;
    o.data[0] = pre + 1u;
    o.data[1] = pre + 2u * (leaves_before[mid] - lb);
  }
  out[pre] = o;
}

}  // namespace

#define BUILD_CHECK(expr)       \
  do {                          \
    rc = (expr);                \
    if (rc != NRT_OK) goto done; \
  } while (0)
#define BUILD_CUDA(expr)                                        \
  do {                                                          \
    cudaError_t _e = (expr);                                    \
    if (_e != cudaSuccess) {                                    \
      rc = cuda_fail(_e, #expr, __FILE__, __LINE__);            \
      goto done;                                                \
    }                                                           \
  } while (0)

int build_on_device(Accel *a, cudaStream_t s) {
  const uint32_t n = a->n_prims;
  const BuildOptions28 &opt = a->options;
  const int B = (int)opt.bin_size;
  // min_leaf_primitives == 0 would ask for empty leaves (the reference then recurses to max_tree_depth)
  const uint32_t min_leaf = opt.min_leaf_primitives < 1 ? 1u : opt.min_leaf_primitives;
  if (B > kMaxBins) {
    set_error("nrt_build: bin_size > 256 is not supported by the device builder");
    return NRT_ERR_INVALID;
  }
  if (n > 0x7FFFFFF0u) {
    set_error("nrt_build: too many primitives");
    return NRT_ERR_INVALID;
  }
  int rc = NRT_OK;
  float4 *d_plo = nullptr, *d_phi = nullptr, *d_plo_u = nullptr, *d_phi_u = nullptr;
  float *d_pcz = nullptr, *d_pcz_u = nullptr;
  uint32_t *d_order = nullptr, *d_table = nullptr;
  uint32_t *d_idx[2] = {nullptr, nullptr}, *d_nodeof[2] = {nullptr, nullptr};
  uint32_t *d_flags = nullptr, *d_scan = nullptr, *d_scratch = nullptr, *d_active[2] = {nullptr, nullptr};
  uint32_t *d_subtrees = nullptr, *d_bins = nullptr, *d_scene = nullptr, *d_mids = nullptr;
  BNode *d_pool = nullptr;
  BuildCounters *d_ctr = nullptr;
  BuildCounters hc;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  const size_t max_active = (size_t)n / (kSubtree + 1) + 2;   // nodes with > kSubtree prims per level
  const size_t max_subtrees = (size_t)n / ((size_t)min_leaf + 1) + 2;
  const size_t bin_words = max_active * 3 * (size_t)B * kBinWords;
  const uint32_t grid_n = (n + 255) / 256;
  int cur = 0, which = 0;
  uint32_t n_active = 0;
  uint32_t n_nodes = 0;
  const size_t sub_smem = kSubWarps * sub_slice_bytes(B);

  BUILD_CUDA(cudaEventCreate(&ev0));
  BUILD_CUDA(cudaEventCreate(&ev1));
  BUILD_CUDA(cudaMalloc(&d_plo, sizeof(float4) * (size_t)n));
  BUILD_CUDA(cudaMalloc(&d_phi, sizeof(float4) * (size_t)n));
  BUILD_CUDA(cudaMalloc(&d_pcz, sizeof(float) * (size_t)n));
  BUILD_CUDA(cudaMalloc(&d_plo_u, sizeof(float4) * (size_t)n));
  BUILD_CUDA(cudaMalloc(&d_phi_u, sizeof(float4) * (size_t)n));
  BUILD_CUDA(cudaMalloc(&d_pcz_u, sizeof(float) * (size_t)n));
  BUILD_CUDA(cudaMalloc(&d_order, sizeof(uint32_t) * (size_t)n));
  BUILD_CUDA(cudaMalloc(&d_table, sizeof(uint32_t) * ((size_t)kSortDigits * ((n + kSortTile - 1) / kSortTile) + 1)));
  for (int i = 0; i < 2; i++) {
    BUILD_CUDA(cudaMalloc(&d_idx[i], sizeof(uint32_t) * (size_t)n));
    BUILD_CUDA(cudaMalloc(&d_nodeof[i], sizeof(uint32_t) * (size_t)n));
    BUILD_CUDA(cudaMalloc(&d_active[i], sizeof(uint32_t) * max_active));
  }
  BUILD_CUDA(cudaMalloc(&d_flags, sizeof(uint32_t) * ((size_t)n + 1)));
  BUILD_CUDA(cudaMalloc(&d_scan, sizeof(uint32_t) * ((size_t)n + 1)));
  BUILD_CUDA(cudaMalloc(&d_scratch, sizeof(uint32_t) * scan_scratch_words(n + 1)));
  BUILD_CUDA(cudaMalloc(&d_subtrees, sizeof(uint32_t) * max_subtrees));
  BUILD_CUDA(cudaMalloc(&d_mids, sizeof(uint32_t) * max_active));  // nodes with more than kSubtree primitives
  BUILD_CUDA(cudaMalloc(&d_bins, sizeof(uint32_t) * bin_words));
  BUILD_CUDA(cudaMalloc(&d_scene, sizeof(uint32_t) * 8));
  BUILD_CUDA(cudaMalloc(&d_pool, sizeof(BNode) * 2 * (size_t)n));
  BUILD_CUDA(cudaMalloc(&d_ctr, sizeof(BuildCounters)));
  BUILD_CUDA(cudaMemsetAsync(d_ctr, 0, sizeof(BuildCounters), s));  // incl. the padding the host reads back
  {
    const uint32_t init[8] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u, 0u, 0u, 0u};
    BUILD_CUDA(cudaMemcpyAsync(d_scene, init, sizeof(init), cudaMemcpyHostToDevice, s));
  }
  // outputs are allocated up front (2n-1 is the node bound) so that no allocation stalls the build
  BUILD_CUDA(cudaMalloc(&a->d_nodes, sizeof(Node40) * (2 * (size_t)n)));
  BUILD_CUDA(cudaMalloc(&a->d_indices, sizeof(uint32_t) * (size_t)n));
  BUILD_CUDA(cudaEventRecord(ev0, s));
  if (a->d_prim_boxes)
    box_setup_kernel<<<grid_n, 256, 0, s>>>(a->d_prim_boxes, n, d_plo_u, d_phi_u, d_pcz_u, d_scene);
  else
    prim_setup_kernel<<<grid_n, 256, 0, s>>>(a->d_verts, a->d_faces, n, d_plo_u, d_phi_u, d_pcz_u, d_scene);
  BUILD_CUDA(cudaGetLastError());
  {
    // Morton pre-order: sort the primitives along a 30-bit Z-curve over the scene box, then lay their
    // records out in that order (slot s of the builder = primitive d_order[s])
    uint32_t keys6[6];
    BUILD_CUDA(cudaMemcpyAsync(keys6, d_scene, sizeof(keys6), cudaMemcpyDeviceToHost, s));
    BUILD_CUDA(cudaStreamSynchronize(s));
    float lo[3], hi[3];
    for (int k = 0; k < 3; k++) {
      uint32_t kmin = keys6[k], kmax = keys6[3 + k];
      uint32_t umin = (kmin & 0x80000000u) ? (kmin ^ 0x80000000u) : ~kmin;
      uint32_t umax = (kmax & 0x80000000u) ? (kmax ^ 0x80000000u) : ~kmax;
      memcpy(&lo[k], &umin, 4);
      memcpy(&hi[k], &umax, 4);
      a->root_bmin[k] = lo[k];
      a->root_bmax[k] = hi[k];
    }
    float3 smin = make_float3(lo[0], lo[1], lo[2]);
    float3 sinv = make_float3(hi[0] > lo[0] ? 1024.0f / (hi[0] - lo[0]) : 0.0f, hi[1] > lo[1] ? 1024.0f / (hi[1] - lo[1]) : 0.0f,
                              hi[2] > lo[2] ? 1024.0f / (hi[2] - lo[2]) : 0.0f);
    if (n > (uint32_t)kSubtree) {
      uint32_t *keys = d_flags, *keys_tmp = d_scan, *vals = d_order, *vals_tmp = d_nodeof[1];
      morton_kernel<<<grid_n, 256, 0, s>>>(d_plo_u, d_phi_u, d_pcz_u, n, smin, sinv, keys, vals);
      BUILD_CUDA(cudaGetLastError());
      // the curve order is a locality device, not part of the tree's definition: the top 24 of the 30 code bits
      // (cells of 1/256 of the scene box per axis) give the sweep the same coherence in 6 passes instead of 8
      BUILD_CHECK(radix_sort_pairs(keys, vals, keys_tmp, vals_tmp, n, 6, 30, d_table, d_scratch, s));
      if (vals != d_order) {  // odd number of passes: keep the result in d_order
        BUILD_CUDA(cudaMemcpyAsync(d_order, vals, sizeof(uint32_t) * (size_t)n, cudaMemcpyDeviceToDevice, s));
      }
      gather_prims_kernel<<<grid_n, 256, 0, s>>>(d_order, d_plo_u, d_phi_u, d_pcz_u, n, d_plo, d_phi, d_pcz);
      BUILD_CUDA(cudaGetLastError());
    } else {
      // the whole scene is one phase-B subtree (a Cornell box, the top level of a small two-level scene): the order
      // of the records does not matter there, so the 18 launches of the sort are skipped
      iota_kernel<<<grid_n, 256, 0, s>>>(d_order, d_flags, n);
      BUILD_CUDA(cudaGetLastError());
      std::swap(d_plo, d_plo_u);
      std::swap(d_phi, d_phi_u);
      std::swap(d_pcz, d_pcz_u);
    }
  }
  iota_kernel<<<grid_n, 256, 0, s>>>(d_idx[0], d_nodeof[0], n);
  init_build_kernel<<<1, 1, 0, s>>>(d_pool, d_ctr, d_scene, n, min_leaf, opt.max_tree_depth,
                                    d_active[0], d_subtrees, d_mids);
  BUILD_CUDA(cudaGetLastError());
  BUILD_CUDA(cudaMemcpyAsync(&hc, d_ctr, sizeof(hc), cudaMemcpyDeviceToHost, s));
  BUILD_CUDA(cudaStreamSynchronize(s));
  n_active = hc.n_active[0];

  // ---- phase A
  BUILD_CUDA(cudaFuncSetAttribute(bin_large_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  3 * kMaxBins * kBinWords * 4));
  while (n_active > 0) {
    const size_t words = (size_t)n_active * 3 * B * kBinWords;
    clear_bins_kernel<<<(unsigned)((words + 255) / 256), 256, 0, s>>>(d_bins, words);
    bin_large_kernel<<<(n + 1023) / 1024, 256, (size_t)3 * B * kBinWords * 4, s>>>(
        d_pool, d_nodeof[which], d_idx[which], d_plo, d_phi, d_pcz, n, B, d_bins);
    reset_count_kernel<<<1, 1, 0, s>>>(d_ctr, cur ^ 1);
    split_large_kernel<<<(n_active + 3) / 4, 128, (size_t)4 * 2 * B * 4, s>>>(
        d_pool, d_ctr, d_active[cur], cur, d_active[cur ^ 1], d_subtrees, d_mids, d_bins, B, min_leaf,
        opt.max_tree_depth);
    flag_large_kernel<<<grid_n, 256, 0, s>>>(d_pool, d_nodeof[which], d_idx[which], d_plo, d_phi, d_pcz, n, B,
                                             d_flags);
    BUILD_CUDA(cudaGetLastError());
    BUILD_CHECK(exclusive_scan_u32_async(d_flags, d_scan, n, d_scratch, s));
    scatter_large_kernel<<<grid_n, 256, 0, s>>>(d_pool, d_nodeof[which], d_idx[which], d_flags, d_scan, n,
                                                d_nodeof[which ^ 1], d_idx[which ^ 1], d_plo, d_phi, d_bins, B);
    fix_median_kernel<<<(n_active + 127) / 128, 128, 0, s>>>(d_pool, d_ctr, d_active[cur], cur, d_bins, B);
    BUILD_CUDA(cudaGetLastError());
    which ^= 1;
    cur ^= 1;
    BUILD_CUDA(cudaMemcpyAsync(&hc, d_ctr, sizeof(hc), cudaMemcpyDeviceToHost, s));
    BUILD_CUDA(cudaStreamSynchronize(s));
    n_active = hc.n_active[cur];
  }

  // ---- middle phase: nodes of kSubtree+1 .. kMid primitives, one CTA each, down to phase-B subtrees
  if (hc.n_mids > 0) {
    const size_t mid_smem = sizeof(MidShared) + (size_t)3 * B * kBinWords * 4 + (size_t)3 * 2 * B * 4;
    BUILD_CUDA(cudaFuncSetAttribute(midtree_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mid_smem));
    midtree_kernel<<<hc.n_mids, kMidThreads, mid_smem, s>>>(d_pool, d_ctr, d_mids, d_idx[which], d_plo, d_phi, d_pcz, B,
                                                           min_leaf, opt.max_tree_depth, d_subtrees);
    BUILD_CUDA(cudaGetLastError());
    BUILD_CUDA(cudaMemcpyAsync(&hc, d_ctr, sizeof(hc), cudaMemcpyDeviceToHost, s));
    BUILD_CUDA(cudaStreamSynchronize(s));
  }

  // ---- phase B
  if (hc.n_subtrees > 0) {
    BUILD_CUDA(cudaFuncSetAttribute(subtree_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sub_smem));
    subtree_kernel<<<(hc.n_subtrees + kSubWarps - 1) / kSubWarps, kSubWarps * 32, sub_smem, s>>>(
        d_pool, d_ctr, d_subtrees, hc.n_subtrees, d_idx[which], d_plo, d_phi,
                                                              d_pcz, B, min_leaf, opt.max_tree_depth);
    BUILD_CUDA(cudaGetLastError());
  }
  BUILD_CUDA(cudaMemcpyAsync(&hc, d_ctr, sizeof(hc), cudaMemcpyDeviceToHost, s));
  BUILD_CUDA(cudaStreamSynchronize(s));
  n_nodes = hc.pool;

  // ---- phase C
  BUILD_CUDA(cudaMemsetAsync(d_flags, 0, sizeof(uint32_t) * ((size_t)n + 1), s));
  mark_leaves_kernel<<<(n_nodes + 255) / 256, 256, 0, s>>>(d_pool, n_nodes, d_flags, d_ctr);
  BUILD_CUDA(cudaGetLastError());
  BUILD_CHECK(exclusive_scan_u32_async(d_flags, d_scan, n + 1, d_scratch, s));
  emit_nodes_kernel<<<(n_nodes + 255) / 256, 256, 0, s>>>(d_pool, n_nodes, d_scan, a->d_nodes);
  BUILD_CUDA(cudaGetLastError());
  // indices_ holds ORIGINAL primitive ids: slot -> primitive through the Morton order
  map_indices_kernel<<<grid_n, 256, 0, s>>>(d_idx[which], d_order, n, a->d_indices);
  BUILD_CUDA(cudaGetLastError());
  BUILD_CUDA(cudaEventRecord(ev1, s));
  BUILD_CUDA(cudaMemcpyAsync(&hc, d_ctr, sizeof(hc), cudaMemcpyDeviceToHost, s));
  BUILD_CUDA(cudaStreamSynchronize(s));
  {
    float ms = 0.0f;
    BUILD_CUDA(cudaEventElapsedTime(&ms, ev0, ev1));
    n_nodes = 2u * hc.n_leaves - 1u;  // live nodes (the pool also holds the slots subtrees reserved and left unused)
    a->n_nodes = n_nodes;
    a->stats.max_tree_depth = hc.max_depth;
    a->stats.num_leaf_nodes = hc.n_leaves;
    a->stats.num_branch_nodes = n_nodes - hc.n_leaves;
    a->stats.build_secs = ms * 1e-3f;
    a->mirror.invalidate();
  }

done:
  cudaFree(d_plo);
  cudaFree(d_phi);
  cudaFree(d_pcz);
  cudaFree(d_plo_u);
  cudaFree(d_phi_u);
  cudaFree(d_pcz_u);
  cudaFree(d_order);
  cudaFree(d_table);
  for (int i = 0; i < 2; i++) {
    cudaFree(d_idx[i]);
    cudaFree(d_nodeof[i]);
    cudaFree(d_active[i]);
  }
  cudaFree(d_flags);
  cudaFree(d_scan);
  cudaFree(d_scratch);
  cudaFree(d_subtrees);
  cudaFree(d_mids);
  cudaFree(d_bins);
  cudaFree(d_scene);
  cudaFree(d_pool);
  cudaFree(d_ctr);
  if (ev0) cudaEventDestroy(ev0);
  if (ev1) cudaEventDestroy(ev1);
  return rc;
}

}  // namespace nrt
