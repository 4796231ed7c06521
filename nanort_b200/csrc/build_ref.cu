// Reference-exact builder ("conformance build"): produces, on the device, the very node array and indices_
// that CPU nanort's BVHAccel<T>::Build writes at the pinned commit, for T = float and T = double -- bit for bit,
// including
//   * the x-only binning caused by the guard at nanort.h:1357 (SURVEY.md F1): y/z never get a binned plane, their
//     fallback planes are bmin + extent/bin_size (FindCutFromBinBuffer with empty bins, nanort.h:1381-1430),
//   * the try-next-axis / object-median fallback of BuildTree (nanort.h:1827-1857) with the node's axis label
//     being the last axis tried,
//   * TriangleSAHPred (p0+p1+p2 < 3*pos, nanort.h:897-911) and the element order libstdc++'s bidirectional
//     std::partition leaves behind (two pointers swapping the k-th misplaced element from the left with the
//     k-th misplaced element from the right),
//   * the node order: depth-first pre-order of BuildTree (nanort.h:1759-1890) -- or, for more than
//     min_primitives_for_parallel_build primitives in the C++11 build, the shallow tree followed by the joined
//     sub-arrays (nanort.h:1996-2067).
// Every piece of arithmetic that decides a split is done in T, as BVHAccel<T> does it: primitive boxes and centres
// (BoundingBoxAndCenter, nanort.h:958-971), bin indices and bin boxes (ContributeBinBuffer, nanort.h:1314-1367), SAH
// costs (FindCutFromBinBuffer, nanort.h:1381-1430; CalculateSurfaceArea, nanort.h:1278-1283), cut positions and the
// predicate (TriangleSAHPred, nanort.h:897-911).  Min/max boxes travel as order-preserving 32- or 64-bit keys through
// atomicMin / atomicMax (OrderedKey in build_common.cuh).
// It exists for conformance (the oracle compares its output with the reference's arrays directly,
// tests/test_gpu_build_ref.py for float, tests/test_gpu_f64.py for double) and to let the GPU traverse the
// reference's own topology without a CPU build; the production builder is build.cu.  Level-synchronous,
// position-parallel, global atomics; speed is not a goal (the reference tree is up to 256 levels deep).
#include <algorithm>
#include <type_traits>
#include <vector>

#include "build_common.cuh"
#include "common.cuh"
#include "scan.cuh"

namespace nrt {
namespace {

// per-primitive records: float4 / float2, or a 32-byte / 16-byte double vector
struct alignas(32) Double4 {
  double x, y, z, w;
};
template <typename T>
using V4 = typename std::conditional<std::is_same<T, float>::value, float4, Double4>::type;
template <typename T>
using V2 = typename std::conditional<std::is_same<T, float>::value, float2, double2>::type;
template <typename T>
using Key = typename OrderedKey<T>::Key;

// build node: the range [l, r) of the primitive order it owns and where it stands in the level loop
template <typename T>
struct RefNode {
  T bmin[3], bmax[3];
  uint32_t l, r;
  uint32_t left;    // pool index of the left child (right = left + 1); kInactive for a leaf
  uint32_t depth;
  uint32_t rturns;  // right turns on the root path
  uint32_t axis;
  uint32_t nleft;   // mid - l once split
  uint32_t level;   // level in which the node was created
  uint32_t fresh;   // index in that level's fresh list
  uint32_t active;  // index in that level's active list; kInactive for a node that will not be split
};

template <typename T>
__device__ __forceinline__ RefNode<T> new_node(uint32_t l, uint32_t r, uint32_t depth, uint32_t rturns,
                                               uint32_t level, uint32_t fresh) {
  RefNode<T> c;
  for (int k = 0; k < 3; k++) c.bmin[k] = c.bmax[k] = T(0);
  c.l = l;
  c.r = r;
  c.left = kInactive;
  c.depth = depth;
  c.rturns = rturns;
  c.axis = 0;
  c.nleft = 0;
  c.level = level;
  c.fresh = fresh;
  c.active = kInactive;
  return c;
}

// per primitive: A = (bmin.xyz, center.x), B = (bmax.xyz, sum.x), C = (sum.y, sum.z); sum = (p0+p1)+p2,
// center = sum * (T(1)/T(3))  (TriangleMesh::BoundingBoxAndCenter, nanort.h:958-971)
template <typename T>
__global__ void ref_prim_kernel(const T *__restrict__ verts, const uint32_t *__restrict__ faces, uint32_t n,
                                V4<T> *__restrict__ A, V4<T> *__restrict__ B, V2<T> *__restrict__ C) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t f0 = faces[3 * (size_t)i], f1 = faces[3 * (size_t)i + 1], f2 = faces[3 * (size_t)i + 2];
  const T *p0 = verts + 3 * (size_t)f0, *p1 = verts + 3 * (size_t)f1, *p2 = verts + 3 * (size_t)f2;
  T lo[3], hi[3], s[3];
  for (int k = 0; k < 3; k++) {
    lo[k] = fmin(p0[k], fmin(p1[k], p2[k]));
    hi[k] = fmax(p0[k], fmax(p1[k], p2[k]));
    s[k] = (p0[k] + p1[k]) + p2[k];
  }
  A[i] = V4<T>{lo[0], lo[1], lo[2], s[0] * (T(1) / T(3))};
  B[i] = V4<T>{hi[0], hi[1], hi[2], s[0]};
  C[i] = V2<T>{s[1], s[2]};
}

// box primitives (two-level scene, top level; float only): centre = (bmax + bmin) / 2 in every slot the predicate
// reads
__global__ void ref_box_prim_kernel(const float *__restrict__ boxes6, uint32_t n, float4 *__restrict__ A,
                                    float4 *__restrict__ B, float2 *__restrict__ C) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float lo[3], hi[3], c[3];
  for (int k = 0; k < 3; k++) {
    lo[k] = boxes6[6 * (size_t)i + k];
    hi[k] = boxes6[6 * (size_t)i + 3 + k];
    c[k] = (hi[k] + lo[k]) / 2.0f;
  }
  A[i] = make_float4(lo[0], lo[1], lo[2], c[0]);
  B[i] = make_float4(hi[0], hi[1], hi[2], c[0]);
  C[i] = make_float2(c[1], c[2]);
}

struct RefCounters {
  uint32_t pool;
  uint32_t n_fresh[2];   // nodes created by the previous / this level (ping-pong)
  uint32_t n_active[2];  // the ones of them that will be split
  uint32_t pad[3];
};

template <typename T>
__global__ void ref_init_kernel(RefNode<T> *pool, RefCounters *ctr, uint32_t n, uint32_t min_leaf,
                                uint32_t max_depth, uint32_t *fresh0, uint32_t *active0) {
  RefNode<T> r = new_node<T>(0, n, 0, 0, 0, 0);
  ctr->pool = 1;
  ctr->n_fresh[0] = 1;
  ctr->n_fresh[1] = 0;
  ctr->n_active[0] = ctr->n_active[1] = 0;
  fresh0[0] = 0;
  if (!(n <= min_leaf || 0 >= max_depth)) {
    active0[0] = 0;
    r.active = 0;
    ctr->n_active[0] = 1;
  }
  pool[0] = r;
}

__global__ void ref_iota_kernel(uint32_t *idx, uint32_t *node_of, uint32_t n) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    idx[i] = i;
    node_of[i] = 0;
  }
}

template <typename T>
__global__ void ref_keys_init_kernel(Key<T> *keys, uint32_t n_fresh) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_fresh * 6) keys[i] = (i % 6) < 3 ? OrderedKey<T>::kMax : Key<T>(0);
}

// min / max of a key over the warp: one reduction instruction for 32-bit keys, a shuffle loop for 64-bit keys
__device__ __forceinline__ uint32_t warp_min(uint32_t k) { return __reduce_min_sync(0xFFFFFFFFu, k); }
__device__ __forceinline__ uint32_t warp_max(uint32_t k) { return __reduce_max_sync(0xFFFFFFFFu, k); }
__device__ __forceinline__ unsigned long long warp_min(unsigned long long k) {
  for (int o = 16; o > 0; o >>= 1) k = min(k, __shfl_xor_sync(0xFFFFFFFFu, k, o));
  return k;
}
__device__ __forceinline__ unsigned long long warp_max(unsigned long long k) {
  for (int o = 16; o > 0; o >>= 1) k = max(k, __shfl_xor_sync(0xFFFFFFFFu, k, o));
  return k;
}

// exact box of every fresh node: min/max over the boxes of its primitives (ComputeBoundingBox, nanort.h:1545-1567),
// taken in key order -- the order the atomics use -- so the box does not depend on how primitives fall into warps
template <typename T>
__global__ void __launch_bounds__(256)
    ref_bbox_kernel(const RefNode<T> *__restrict__ pool, const uint32_t *__restrict__ node_of,
                    const uint32_t *__restrict__ idx, const V4<T> *__restrict__ A, const V4<T> *__restrict__ B,
                    uint32_t n, uint32_t level, Key<T> *__restrict__ keys) {
  typedef OrderedKey<T> K;
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  uint32_t slot = kInactive;
  Key<T> v[6] = {K::kMax, K::kMax, K::kMax, 0, 0, 0};
  if (p < n) {
    const RefNode<T> nd = pool[node_of[p]];
    if (nd.level == level) {
      slot = nd.fresh;
      const uint32_t s = idx[p];
      const V4<T> a = A[s], b = B[s];
      v[0] = K::key(a.x), v[1] = K::key(a.y), v[2] = K::key(a.z);
      v[3] = K::key(b.x), v[4] = K::key(b.y), v[5] = K::key(b.z);
    }
  }
  // whole warp inside one fresh node: lane 0 issues the atomics for the warp
  if (__match_any_sync(0xFFFFFFFFu, slot) == 0xFFFFFFFFu) {
    for (int c = 0; c < 3; c++) {
      v[c] = warp_min(v[c]);
      v[3 + c] = warp_max(v[3 + c]);
    }
    if (lane != 0) return;
  }
  if (slot == kInactive) return;
  Key<T> *k = keys + (size_t)slot * 6;
  for (int c = 0; c < 3; c++) {
    atomicMin(k + c, v[c]);
    atomicMax(k + 3 + c, v[3 + c]);
  }
}

template <typename T>
__global__ void ref_bbox_store_kernel(RefNode<T> *pool, const uint32_t *__restrict__ fresh, uint32_t n_fresh,
                                      const Key<T> *__restrict__ keys) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_fresh) return;
  RefNode<T> *nd = pool + fresh[i];
  for (int k = 0; k < 3; k++) {
    nd->bmin[k] = OrderedKey<T>::unkey(keys[(size_t)i * 6 + k]);
    nd->bmax[k] = OrderedKey<T>::unkey(keys[(size_t)i * 6 + 3 + k]);
  }
}

template <typename T>
__global__ void ref_bins_clear_kernel(Key<T> *bins, size_t words) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < words) {
    int w = (int)(i & (kBinWords - 1));
    bins[i] = (w >= 1 && w <= 3) ? OrderedKey<T>::kMax : Key<T>(0);
  }
}

// x-axis bins only (the pinned commit's guard, nanort.h:1357): count + exact box per bin
template <typename T>
__global__ void __launch_bounds__(256)
    ref_bins_kernel(const RefNode<T> *__restrict__ pool, const uint32_t *__restrict__ node_of,
                    const uint32_t *__restrict__ idx, const V4<T> *__restrict__ A, const V4<T> *__restrict__ B,
                    uint32_t n, uint32_t level, int nbins, Key<T> *__restrict__ bins) {
  typedef OrderedKey<T> K;
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const RefNode<T> nd = pool[node_of[p]];
  if (nd.level != level || nd.active == kInactive) return;
  const uint32_t s = idx[p];
  const V4<T> a = A[s], b = B[s];
  const int bx = bin_of(a.w, nd.bmin[0], inv_extent(nd.bmin[0], nd.bmax[0], nbins), nbins);
  Key<T> *w = bins + ((size_t)nd.active * nbins + bx) * kBinWords;
  atomicAdd(w, Key<T>(1));
  atomicMin(w + 1, K::key(a.x));
  atomicMin(w + 2, K::key(a.y));
  atomicMin(w + 3, K::key(a.z));
  atomicMax(w + 4, K::key(b.x));
  atomicMax(w + 5, K::key(b.y));
  atomicMax(w + 6, K::key(b.z));
}

// one warp per active node: the three candidate planes (nanort.h:1423) and the per-node round state.
// Dynamic shared memory: 4 warps x 2 x nbins values of T.
template <typename T>
__global__ void __launch_bounds__(128)
    ref_cut_kernel(const RefNode<T> *__restrict__ pool, const uint32_t *__restrict__ active, uint32_t n_active,
                   const Key<T> *__restrict__ bins, int nbins, T *__restrict__ cut3, uint32_t *__restrict__ cnt,
                   uint32_t *__restrict__ state) {
  extern __shared__ __align__(16) unsigned char ref_cut_smem[];
  T *scratch = reinterpret_cast<T *>(ref_cut_smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t a = blockIdx.x * 4 + warp;
  if (a >= n_active) return;
  const RefNode<T> nd = pool[active[a]];
  T cost;
  int cut;
  sweep_axis(bins + (size_t)a * nbins * kBinWords, nbins, scratch + (size_t)warp * 2 * nbins,
             scratch + (size_t)warp * 2 * nbins + nbins, cost, cut);
  if (lane == 0) {
    const T fB = (T)nbins;
    // no separating plane: minBin keeps its initial 1
    const int min_bin_x = cost < cuda::std::numeric_limits<T>::max() ? cut : 1;
    cut3[(size_t)a * 3 + 0] = (T)min_bin_x * ((nd.bmax[0] - nd.bmin[0]) / fB) + nd.bmin[0];
    cut3[(size_t)a * 3 + 1] = T(1) * ((nd.bmax[1] - nd.bmin[1]) / fB) + nd.bmin[1];
    cut3[(size_t)a * 3 + 2] = T(1) * ((nd.bmax[2] - nd.bmin[2]) / fB) + nd.bmin[2];
    cnt[a] = 0;
    state[a] = 0;  // bit 31 = decided, bit 30 = partition needed, low bits = axis
  }
}

// triangles: (p0+p1)+p2 < pos*3 (TriangleSAHPred, nanort.h:897-911), mul = 3; boxes: (bmin+bmax)/2 < pos
// (NodeBBoxPred, examples/nanosg/nanosg.h:520-532), mul = 1 (pos * 1 is exact)
template <typename T>
__device__ __forceinline__ bool ref_pred(const V4<T> &b, const V2<T> &c, int axis, T pos, T mul) {
  const T s = axis == 0 ? b.w : (axis == 1 ? c.x : c.y);
  return s < pos * mul;
}

// round k: how many primitives of every undecided node satisfy the predicate on axis k
template <typename T>
__global__ void __launch_bounds__(256)
    ref_count_kernel(const RefNode<T> *__restrict__ pool, const uint32_t *__restrict__ node_of,
                     const uint32_t *__restrict__ idx, const V4<T> *__restrict__ B, const V2<T> *__restrict__ C,
                     uint32_t n, uint32_t level, int axis, const T *__restrict__ cut3,
                     const uint32_t *__restrict__ state, uint32_t *__restrict__ cnt, T pred_mul) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t slot = kInactive;
  bool t = false;
  if (p < n) {
    const RefNode<T> nd = pool[node_of[p]];
    if (nd.level == level && nd.active != kInactive && !(state[nd.active] >> 31)) {
      slot = nd.active;
      const uint32_t s = idx[p];
      t = ref_pred<T>(B[s], C[s], axis, cut3[(size_t)slot * 3 + axis], pred_mul);
    }
  }
  const unsigned same = __match_any_sync(0xFFFFFFFFu, slot);
  if (same == 0xFFFFFFFFu) {
    const unsigned m = __ballot_sync(0xFFFFFFFFu, t);
    if (slot != kInactive && (threadIdx.x & 31) == 0 && m) atomicAdd(cnt + slot, (uint32_t)__popc(m));
  } else if (t) {
    atomicAdd(cnt + slot, 1u);
  }
}

template <typename T>
__global__ void ref_decide_kernel(RefNode<T> *pool, const uint32_t *__restrict__ active, uint32_t n_active, int axis,
                                  uint32_t *__restrict__ cnt, uint32_t *__restrict__ state) {
  const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n_active || (state[a] >> 31)) return;
  RefNode<T> *nd = pool + active[a];
  const uint32_t n = nd->r - nd->l, c = cnt[a];
  if (c > 0 && c < n) {
    state[a] = 0xC0000000u | (uint32_t)axis;  // decided, partition on this axis
    nd->axis = (uint32_t)axis;
    nd->nleft = c;
  } else if (axis == 2) {
    state[a] = 0x80000000u | 2u;  // all three attempts failed: object median, order untouched, label = last axis
    nd->axis = 2u;
    nd->nleft = n >> 1;
  } else {
    cnt[a] = 0;
  }
}

// flags of the elements std::partition will move: falses in the left part, trues in the right part
template <typename T>
__global__ void __launch_bounds__(256)
    ref_flags_kernel(const RefNode<T> *__restrict__ pool, const uint32_t *__restrict__ node_of,
                     const uint32_t *__restrict__ idx, const V4<T> *__restrict__ B, const V2<T> *__restrict__ C,
                     uint32_t n, uint32_t level, const T *__restrict__ cut3, const uint32_t *__restrict__ state,
                     uint32_t *__restrict__ mf, uint32_t *__restrict__ mt, T pred_mul) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > n) return;
  uint32_t f = 0, t = 0;
  if (p < n) {
    const RefNode<T> nd = pool[node_of[p]];
    if (nd.level == level && nd.active != kInactive && (state[nd.active] & 0x40000000u)) {
      const int axis = (int)(state[nd.active] & 3u);
      const uint32_t s = idx[p];
      const bool pr = ref_pred<T>(B[s], C[s], axis, cut3[(size_t)nd.active * 3 + axis], pred_mul);
      const bool left_part = p < nd.l + nd.nleft;
      f = (left_part && !pr) ? 1u : 0u;
      t = (!left_part && pr) ? 1u : 0u;
    }
  }
  mf[p] = f;  // entry n stays 0: the scans then hold totals at index n
  mt[p] = t;
}

__global__ void ref_compact_kernel(const uint32_t *__restrict__ mf, const uint32_t *__restrict__ mt,
                                   const uint32_t *__restrict__ smf, const uint32_t *__restrict__ smt, uint32_t n,
                                   uint32_t *__restrict__ mf_list, uint32_t *__restrict__ mt_list) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  if (mf[p]) mf_list[smf[p]] = p;
  if (mt[p]) mt_list[smt[p]] = p;
}

// the k-th misplaced false from the left trades places with the k-th misplaced true from the right
template <typename T>
__global__ void __launch_bounds__(256)
    ref_permute_kernel(const RefNode<T> *__restrict__ pool, const uint32_t *__restrict__ node_of,
                       const uint32_t *__restrict__ idx, const uint32_t *__restrict__ mf,
                       const uint32_t *__restrict__ mt, const uint32_t *__restrict__ smf,
                       const uint32_t *__restrict__ smt, const uint32_t *__restrict__ mf_list,
                       const uint32_t *__restrict__ mt_list, uint32_t n, uint32_t *__restrict__ out) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  uint32_t v = idx[p];
  if (mf[p] || mt[p]) {
    const RefNode<T> nd = pool[node_of[p]];
    const uint32_t mid = nd.l + nd.nleft;
    const uint32_t m = smf[mid] - smf[nd.l];  // misplaced pairs of this node
    if (mf[p]) {
      const uint32_t k = smf[p] - smf[nd.l];
      v = idx[mt_list[smt[mid] + (m - 1u - k)]];
    } else {
      const uint32_t k_from_right = (m - 1u) - (smt[p] - smt[mid]);
      v = idx[mf_list[smf[nd.l] + k_from_right]];
    }
  }
  out[p] = v;
}

template <typename T>
__global__ void ref_children_kernel(RefNode<T> *pool, RefCounters *ctr, const uint32_t *__restrict__ active,
                                    uint32_t n_active, int cur, uint32_t level, uint32_t min_leaf, uint32_t max_depth,
                                    uint32_t *__restrict__ fresh_next, uint32_t *__restrict__ active_next) {
  const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n_active) return;
  RefNode<T> *nd = pool + active[a];
  const uint32_t left = atomicAdd(&ctr->pool, 2u);
  const uint32_t fs = atomicAdd(&ctr->n_fresh[cur ^ 1], 2u);
  nd->left = left;
  const uint32_t mid = nd->l + nd->nleft;
  for (int side = 0; side < 2; side++) {
    RefNode<T> c = new_node<T>(side ? mid : nd->l, side ? nd->r : mid, nd->depth + 1, nd->rturns + (uint32_t)side,
                               level + 1, fs + side);
    fresh_next[fs + side] = left + side;
    const uint32_t cn = c.r - c.l;
    if (!(cn <= min_leaf || c.depth >= max_depth)) {
      const uint32_t as = atomicAdd(&ctr->n_active[cur ^ 1], 1u);
      active_next[as] = left + side;
      c.active = as;
    }
    pool[left + side] = c;
  }
}

template <typename T>
__global__ void ref_nodeof_kernel(const RefNode<T> *__restrict__ pool, uint32_t *__restrict__ node_of, uint32_t n,
                                  uint32_t level) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint32_t nid = node_of[p];
  const RefNode<T> nd = pool[nid];
  if (nd.level == level && nd.active != kInactive) node_of[p] = nd.left + (p < nd.l + nd.nleft ? 0u : 1u);
}

__global__ void ref_reset_kernel(RefCounters *ctr, int which) {
  ctr->n_fresh[which] = 0;
  ctr->n_active[which] = 0;
}

// ---- emission
template <typename T>
__global__ void ref_mark_kernel(const RefNode<T> *__restrict__ pool, uint32_t n_nodes,
                                uint32_t *__restrict__ leaf_start, uint32_t *stats /* [0] max depth, [1] leaves */) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_nodes) return;
  const RefNode<T> nd = pool[i];
  atomicMax(stats + 0, nd.depth);
  if (nd.left == kInactive) {
    leaf_start[nd.l] = 1u;
    atomicAdd(stats + 1, 1u);
  }
}

// deferred sub-tree roots of the C++11 build: branch nodes at depth == shallow_depth (nanort.h:1656-1670)
template <typename T>
__global__ void ref_collect_deferred_kernel(const RefNode<T> *__restrict__ pool, uint32_t n_nodes, uint32_t shallow,
                                            const uint32_t *__restrict__ leaves_before, uint2 *__restrict__ table,
                                            uint32_t *count, uint32_t cap) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_nodes) return;
  const RefNode<T> nd = pool[i];
  if (nd.depth != shallow || nd.left == kInactive) return;
  const uint32_t pre = 2u * leaves_before[nd.l] - nd.rturns + nd.depth;
  const uint32_t size = 2u * (leaves_before[nd.r] - leaves_before[nd.l]) - 1u;
  const uint32_t k = atomicAdd(count, 1u);
  if (k < cap) table[k] = make_uint2(pre, size);
}

// serial pre-order index -> index in the array the C++11 parallel build leaves behind.
// tab[j] = (pre of the j-th deferred root, nodes appended before its sub-array), sorted by pre.
__device__ __forceinline__ uint32_t ref_map_index(uint32_t pre, uint32_t depth, uint32_t shallow, const uint4 *tab,
                                                  uint32_t n_tab, uint32_t n_shallow) {
  if (n_tab == 0) return pre;
  // j = number of deferred roots with pre(R) < pre  (for a deep node: its own root is the last of them or equal)
  uint32_t lo = 0, hi = n_tab;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (tab[mid].x < pre)
      lo = mid + 1;
    else
      hi = mid;
  }
  if (depth <= shallow) {
    // shallow node: drop the deep nodes of the deferred sub-trees that precede it
    const uint32_t skipped = lo == 0 ? 0u : tab[lo - 1].z;  // sum of (size - 1) over roots before it
    return pre - skipped;
  }
  const uint32_t j = lo - 1;  // deep node: root j is the last root with pre(R) < pre
  return n_shallow + tab[j].y + (pre - tab[j].x - 1u);
}

template <typename T>
__global__ void ref_emit_kernel(const RefNode<T> *__restrict__ pool, uint32_t n_nodes,
                                const uint32_t *__restrict__ leaves_before, uint32_t shallow, const uint4 *__restrict__ tab,
                                uint32_t n_tab, uint32_t n_shallow, BVHNodeOf<T> *__restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_nodes) return;
  const RefNode<T> nd = pool[i];
  const uint32_t lb = leaves_before[nd.l];
  const uint32_t pre = 2u * lb - nd.rturns + nd.depth;
  BVHNodeOf<T> o;
  for (int k = 0; k < 3; k++) {
    o.bmin[k] = nd.bmin[k];
    o.bmax[k] = nd.bmax[k];
  }
  if (nd.left == kInactive) {
    o.flag = 1;
    o.axis = 0;  // the reference leaves leaf.axis uninitialised
    o.data[0] = nd.r - nd.l;
    o.data[1] = nd.l;
  } else {
    o.flag = 0;
    o.axis = (int32_t)nd.axis;
    const uint32_t mid = nd.l + nd.nleft;
    o.data[0] = ref_map_index(pre + 1u, nd.depth + 1u, shallow, tab, n_tab, n_shallow);
    o.data[1] = ref_map_index(pre + 2u * (leaves_before[mid] - lb), nd.depth + 1u, shallow, tab, n_tab, n_shallow);
  }
  out[ref_map_index(pre, nd.depth, shallow, tab, n_tab, n_shallow)] = o;
}

template <typename T>
__global__ void ref_count_shallow_kernel(const RefNode<T> *__restrict__ pool, uint32_t n_nodes, uint32_t shallow,
                                         uint32_t *count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_nodes && pool[i].depth <= shallow) atomicAdd(count, 1u);
}

}  // namespace

#define RB_CUDA(expr)                                          \
  do {                                                         \
    cudaError_t _e = (expr);                                   \
    if (_e != cudaSuccess) {                                   \
      rc = cuda_fail(_e, #expr, __FILE__, __LINE__);           \
      goto done;                                               \
    }                                                          \
  } while (0)
#define RB_CHECK(expr)           \
  do {                           \
    rc = (expr);                 \
    if (rc != NRT_OK) goto done; \
  } while (0)

template <typename T>
int build_reference_tree(const T *d_verts, const uint32_t *d_faces, const float *d_boxes, uint32_t n,
                         uint32_t bin_size, uint32_t min_leaf_primitives, uint32_t max_tree_depth,
                         uint32_t shallow_depth, uint32_t min_primitives_for_parallel_build, bool cpp11_order,
                         BVHNodeOf<T> **d_nodes_out, uint32_t **d_indices_out, size_t *n_nodes_out,
                         BuildStats16 *stats_out, T root_bmin[3], T root_bmax[3], cudaStream_t s) {
  static_assert(std::is_same<T, float>::value || std::is_same<T, double>::value, "BVHAccel<float> or <double>");
  const int nbins = (int)bin_size;
  const T pred_mul = d_boxes ? T(1) : T(3);
  const uint32_t min_leaf = min_leaf_primitives < 1 ? 1u : min_leaf_primitives;
  if (nbins > 256) {
    set_error("nrt_build: bin_size > 256 is not supported by the device builders");
    return NRT_ERR_INVALID;
  }
  const bool joined = cpp11_order && n > min_primitives_for_parallel_build;
  if (joined && shallow_depth > 12) {
    set_error("nrt_build: shallow_depth > 12 is not supported by the reference-order emission");
    return NRT_ERR_INVALID;
  }
  int rc = NRT_OK;
  V4<T> *dA = nullptr, *dB = nullptr;
  V2<T> *dC = nullptr;
  BVHNodeOf<T> *d_nodes = nullptr;
  uint32_t *d_indices = nullptr;
  uint32_t *d_idx[2] = {nullptr, nullptr}, *d_nodeof = nullptr, *d_fresh[2] = {nullptr, nullptr},
           *d_active[2] = {nullptr, nullptr};
  Key<T> *d_keys = nullptr, *d_bins = nullptr;
  uint32_t *d_cnt = nullptr, *d_state = nullptr, *d_mf = nullptr, *d_mt = nullptr, *d_smf = nullptr, *d_smt = nullptr,
           *d_mfl = nullptr, *d_mtl = nullptr, *d_scratch = nullptr, *d_small = nullptr;
  T *d_cut = nullptr;
  RefNode<T> *d_pool = nullptr;
  RefCounters *d_ctr = nullptr, hc;
  uint2 *d_tab2 = nullptr;
  uint4 *d_tab4 = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  const size_t max_nodes = 2 * (size_t)n + 2;
  const size_t max_active = (size_t)n / ((size_t)min_leaf + 1) + 2;
  const uint32_t grid_n = (n + 255) / 256, grid_n1 = (n + 1 + 255) / 256;
  int cur = 0, which = 0;
  uint32_t level = 0, n_nodes = 0, n_tab = 0, n_shallow = 0;
  uint32_t hstats[2] = {0, 0};
  std::vector<uint2> tab2;
  std::vector<uint4> tab4;

  RB_CUDA(cudaEventCreate(&ev0));
  RB_CUDA(cudaEventCreate(&ev1));
  RB_CUDA(cudaMalloc(&dA, sizeof(V4<T>) * (size_t)n));
  RB_CUDA(cudaMalloc(&dB, sizeof(V4<T>) * (size_t)n));
  RB_CUDA(cudaMalloc(&dC, sizeof(V2<T>) * (size_t)n));
  for (int i = 0; i < 2; i++) {
    RB_CUDA(cudaMalloc(&d_idx[i], sizeof(uint32_t) * (size_t)n));
    RB_CUDA(cudaMalloc(&d_fresh[i], sizeof(uint32_t) * (2 * max_active + 2)));
    RB_CUDA(cudaMalloc(&d_active[i], sizeof(uint32_t) * max_active));
  }
  RB_CUDA(cudaMalloc(&d_nodeof, sizeof(uint32_t) * (size_t)n));
  RB_CUDA(cudaMalloc(&d_keys, sizeof(Key<T>) * 6 * (2 * max_active + 2)));
  RB_CUDA(cudaMalloc(&d_bins, sizeof(Key<T>) * max_active * (size_t)nbins * kBinWords));
  RB_CUDA(cudaMalloc(&d_cut, sizeof(T) * 3 * max_active));
  RB_CUDA(cudaMalloc(&d_cnt, sizeof(uint32_t) * max_active));
  RB_CUDA(cudaMalloc(&d_state, sizeof(uint32_t) * max_active));
  RB_CUDA(cudaMalloc(&d_mf, sizeof(uint32_t) * ((size_t)n + 1)));
  RB_CUDA(cudaMalloc(&d_mt, sizeof(uint32_t) * ((size_t)n + 1)));
  RB_CUDA(cudaMalloc(&d_smf, sizeof(uint32_t) * ((size_t)n + 1)));
  RB_CUDA(cudaMalloc(&d_smt, sizeof(uint32_t) * ((size_t)n + 1)));
  RB_CUDA(cudaMalloc(&d_mfl, sizeof(uint32_t) * ((size_t)n + 1)));
  RB_CUDA(cudaMalloc(&d_mtl, sizeof(uint32_t) * ((size_t)n + 1)));
  RB_CUDA(cudaMalloc(&d_scratch, sizeof(uint32_t) * scan_scratch_words(n + 1)));
  RB_CUDA(cudaMalloc(&d_small, sizeof(uint32_t) * 8));
  RB_CUDA(cudaMalloc(&d_pool, sizeof(RefNode<T>) * max_nodes));
  RB_CUDA(cudaMalloc(&d_ctr, sizeof(RefCounters)));
  RB_CUDA(cudaMemsetAsync(d_ctr, 0, sizeof(RefCounters), s));  // incl. the padding the host reads back
  RB_CUDA(cudaMalloc(&d_nodes, sizeof(BVHNodeOf<T>) * max_nodes));
  RB_CUDA(cudaMalloc(&d_indices, sizeof(uint32_t) * (size_t)n));

  RB_CUDA(cudaEventRecord(ev0, s));
  if constexpr (std::is_same<T, float>::value) {
    if (d_boxes) ref_box_prim_kernel<<<grid_n, 256, 0, s>>>(d_boxes, n, dA, dB, dC);
  }
  if (!d_boxes) ref_prim_kernel<T><<<grid_n, 256, 0, s>>>(d_verts, d_faces, n, dA, dB, dC);
  ref_iota_kernel<<<grid_n, 256, 0, s>>>(d_idx[0], d_nodeof, n);
  ref_init_kernel<T><<<1, 1, 0, s>>>(d_pool, d_ctr, n, min_leaf, max_tree_depth, d_fresh[0], d_active[0]);
  RB_CUDA(cudaGetLastError());

  for (;;) {
    RB_CUDA(cudaMemcpyAsync(&hc, d_ctr, sizeof(hc), cudaMemcpyDeviceToHost, s));
    RB_CUDA(cudaStreamSynchronize(s));
    const uint32_t n_fresh = hc.n_fresh[cur], n_active = hc.n_active[cur];
    if (n_fresh == 0) break;
    // ---- boxes of the nodes created by the previous level
    ref_keys_init_kernel<T><<<(n_fresh * 6 + 255) / 256, 256, 0, s>>>(d_keys, n_fresh);
    ref_bbox_kernel<T><<<grid_n, 256, 0, s>>>(d_pool, d_nodeof, d_idx[which], dA, dB, n, level, d_keys);
    ref_bbox_store_kernel<T><<<(n_fresh + 255) / 256, 256, 0, s>>>(d_pool, d_fresh[cur], n_fresh, d_keys);
    ref_reset_kernel<<<1, 1, 0, s>>>(d_ctr, cur ^ 1);
    RB_CUDA(cudaGetLastError());
    if (n_active > 0) {
      // ---- candidate planes
      const size_t words = (size_t)n_active * nbins * kBinWords;
      ref_bins_clear_kernel<T><<<(unsigned)((words + 255) / 256), 256, 0, s>>>(d_bins, words);
      ref_bins_kernel<T><<<grid_n, 256, 0, s>>>(d_pool, d_nodeof, d_idx[which], dA, dB, n, level, nbins, d_bins);
      ref_cut_kernel<T><<<(n_active + 3) / 4, 128, (size_t)4 * 2 * nbins * sizeof(T), s>>>(
          d_pool, d_active[cur], n_active, d_bins, nbins, d_cut, d_cnt, d_state);
      // ---- up to three partition attempts (nanort.h:1827-1857)
      for (int axis = 0; axis < 3; axis++) {
        ref_count_kernel<T><<<grid_n, 256, 0, s>>>(d_pool, d_nodeof, d_idx[which], dB, dC, n, level, axis, d_cut,
                                                   d_state, d_cnt, pred_mul);
        ref_decide_kernel<T><<<(n_active + 255) / 256, 256, 0, s>>>(d_pool, d_active[cur], n_active, axis, d_cnt,
                                                                    d_state);
      }
      RB_CUDA(cudaGetLastError());
      // ---- std::partition's element order
      ref_flags_kernel<T><<<grid_n1, 256, 0, s>>>(d_pool, d_nodeof, d_idx[which], dB, dC, n, level, d_cut, d_state,
                                                  d_mf, d_mt, pred_mul);
      RB_CHECK(exclusive_scan_u32_async(d_mf, d_smf, n + 1, d_scratch, s));
      RB_CHECK(exclusive_scan_u32_async(d_mt, d_smt, n + 1, d_scratch, s));
      ref_compact_kernel<<<grid_n, 256, 0, s>>>(d_mf, d_mt, d_smf, d_smt, n, d_mfl, d_mtl);
      ref_permute_kernel<T><<<grid_n, 256, 0, s>>>(d_pool, d_nodeof, d_idx[which], d_mf, d_mt, d_smf, d_smt, d_mfl,
                                                   d_mtl, n, d_idx[which ^ 1]);
      which ^= 1;
      // ---- children
      ref_children_kernel<T><<<(n_active + 255) / 256, 256, 0, s>>>(d_pool, d_ctr, d_active[cur], n_active, cur,
                                                                   level, min_leaf, max_tree_depth, d_fresh[cur ^ 1],
                                                                   d_active[cur ^ 1]);
      ref_nodeof_kernel<T><<<grid_n, 256, 0, s>>>(d_pool, d_nodeof, n, level);
      RB_CUDA(cudaGetLastError());
    }
    cur ^= 1;
    level++;
    if (level > max_tree_depth + 2u) {
      set_error("reference-exact build: level loop did not terminate");
      rc = NRT_ERR_INVALID;
      goto done;
    }
  }
  n_nodes = hc.pool;

  // ---- emission
  RB_CUDA(cudaMemsetAsync(d_mf, 0, sizeof(uint32_t) * ((size_t)n + 1), s));
  RB_CUDA(cudaMemsetAsync(d_small, 0, sizeof(uint32_t) * 8, s));
  ref_mark_kernel<T><<<(n_nodes + 255) / 256, 256, 0, s>>>(d_pool, n_nodes, d_mf, d_small);
  RB_CHECK(exclusive_scan_u32_async(d_mf, d_smf, n + 1, d_scratch, s));  // leaves starting before a position
  if (joined) {
    const uint32_t cap = 1u << shallow_depth;
    RB_CUDA(cudaMalloc(&d_tab2, sizeof(uint2) * cap));
    RB_CUDA(cudaMalloc(&d_tab4, sizeof(uint4) * cap));
    ref_collect_deferred_kernel<T><<<(n_nodes + 255) / 256, 256, 0, s>>>(d_pool, n_nodes, shallow_depth, d_smf,
                                                                         d_tab2, d_small + 2, cap);
    ref_count_shallow_kernel<T><<<(n_nodes + 255) / 256, 256, 0, s>>>(d_pool, n_nodes, shallow_depth, d_small + 3);
    uint32_t hs[4];
    RB_CUDA(cudaMemcpyAsync(hs, d_small, sizeof(hs), cudaMemcpyDeviceToHost, s));
    RB_CUDA(cudaStreamSynchronize(s));
    n_tab = std::min(hs[2], cap);
    n_shallow = hs[3];
    tab2.resize(n_tab);
    if (n_tab) RB_CUDA(cudaMemcpy(tab2.data(), d_tab2, sizeof(uint2) * n_tab, cudaMemcpyDeviceToHost));
    std::sort(tab2.begin(), tab2.end(), [](const uint2 &x, const uint2 &y) { return x.x < y.x; });
    tab4.resize(n_tab);
    uint32_t before = 0;  // nodes appended before root j's sub-array = sum over i<j of (size_i - 1)
    for (uint32_t j = 0; j < n_tab; j++) {
      tab4[j].x = tab2[j].x;
      tab4[j].y = before;
      before += tab2[j].y - 1u;
      tab4[j].z = before;  // deep nodes of roots 0..j: what a later shallow node has to skip
      tab4[j].w = 0;
    }
    if (n_tab) RB_CUDA(cudaMemcpyAsync(d_tab4, tab4.data(), sizeof(uint4) * n_tab, cudaMemcpyHostToDevice, s));
  }
  ref_emit_kernel<T><<<(n_nodes + 255) / 256, 256, 0, s>>>(d_pool, n_nodes, d_smf, shallow_depth, d_tab4, n_tab,
                                                           n_shallow, d_nodes);
  RB_CUDA(cudaGetLastError());
  RB_CUDA(cudaMemcpyAsync(d_indices, d_idx[which], sizeof(uint32_t) * (size_t)n, cudaMemcpyDeviceToDevice, s));
  RB_CUDA(cudaEventRecord(ev1, s));
  RB_CUDA(cudaMemcpyAsync(hstats, d_small, sizeof(hstats), cudaMemcpyDeviceToHost, s));
  {
    RefNode<T> root;
    RB_CUDA(cudaMemcpyAsync(&root, d_pool, sizeof(root), cudaMemcpyDeviceToHost, s));
    RB_CUDA(cudaStreamSynchronize(s));
    for (int k = 0; k < 3; k++) {
      root_bmin[k] = root.bmin[k];
      root_bmax[k] = root.bmax[k];
    }
    float ms = 0.0f;
    RB_CUDA(cudaEventElapsedTime(&ms, ev0, ev1));
    *n_nodes_out = n_nodes;
    stats_out->max_tree_depth = hstats[0];
    stats_out->num_leaf_nodes = hstats[1];
    stats_out->num_branch_nodes = n_nodes - hstats[1];
    stats_out->build_secs = ms * 1e-3f;
    *d_nodes_out = d_nodes;
    *d_indices_out = d_indices;
    d_nodes = nullptr;
    d_indices = nullptr;
  }

done:
  cudaFree(d_nodes);  // only on failure: success hands them to the caller
  cudaFree(d_indices);
  cudaFree(dA);
  cudaFree(dB);
  cudaFree(dC);
  for (int i = 0; i < 2; i++) {
    cudaFree(d_idx[i]);
    cudaFree(d_fresh[i]);
    cudaFree(d_active[i]);
  }
  cudaFree(d_nodeof);
  cudaFree(d_keys);
  cudaFree(d_bins);
  cudaFree(d_cut);
  cudaFree(d_cnt);
  cudaFree(d_state);
  cudaFree(d_mf);
  cudaFree(d_mt);
  cudaFree(d_smf);
  cudaFree(d_smt);
  cudaFree(d_mfl);
  cudaFree(d_mtl);
  cudaFree(d_scratch);
  cudaFree(d_small);
  cudaFree(d_pool);
  cudaFree(d_ctr);
  cudaFree(d_tab2);
  cudaFree(d_tab4);
  if (ev0) cudaEventDestroy(ev0);
  if (ev1) cudaEventDestroy(ev1);
  return rc;
}

template int build_reference_tree<float>(const float *, const uint32_t *, const float *, uint32_t, uint32_t, uint32_t,
                                         uint32_t, uint32_t, uint32_t, bool, Node40 **, uint32_t **, size_t *,
                                         BuildStats16 *, float *, float *, cudaStream_t);
template int build_reference_tree<double>(const double *, const uint32_t *, const float *, uint32_t, uint32_t,
                                          uint32_t, uint32_t, uint32_t, uint32_t, bool, Node64 **, uint32_t **,
                                          size_t *, BuildStats16 *, double *, double *, cudaStream_t);

int build_reference_tree_on_device(Accel *a, bool cpp11_order, cudaStream_t s) {
  const BuildOptions28 &o = a->options;
  const int rc = build_reference_tree<float>(a->d_verts, a->d_faces, a->d_prim_boxes, a->n_prims, o.bin_size,
                                             o.min_leaf_primitives, o.max_tree_depth, o.shallow_depth,
                                             o.min_primitives_for_parallel_build, cpp11_order, &a->d_nodes,
                                             &a->d_indices, &a->n_nodes, &a->stats, a->root_bmin, a->root_bmax, s);
  if (rc == NRT_OK) a->mirror.invalidate();
  return rc;
}

}  // namespace nrt
