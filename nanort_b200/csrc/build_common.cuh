// Device helpers shared by the two builders (build.cu: the fast binned-SAH builder; build_ref.cu: the
// reference-exact builder): build-node record, ordered-uint keys for atomic min/max, bin arithmetic of
// ContributeBinBuffer (nanort.h:1314-1367), the warp-cooperative SAH sweep of FindCutFromBinBuffer
// (nanort.h:1381-1430).  The key, bin and sweep helpers are templates on the scalar type: build.cu uses them with
// float, build_ref.cu with float and double.
#pragma once
#include <float.h>

#include <cuda/std/limits>

#include "common.cuh"

namespace nrt {
namespace {

constexpr uint32_t kInactive = 0xFFFFFFFFu;
constexpr uint32_t kMedian = 0xFFFFFFFEu;
constexpr int kMaxBins = 256;     // bin_size limit of this implementation
constexpr int kBinWords = 8;      // count, min xyz, max xyz, pad

struct BNode {  // 64 bytes
  float bmin[3];
  uint32_t l;
  float bmax[3];
  uint32_t r;
  uint32_t left;   // pool index of the left child (right = left + 1); kInactive for a leaf
  uint32_t depth;
  uint32_t rturns;  // right turns on the root path
  uint32_t axis;
  uint32_t split_bin;  // left iff bin < split_bin; kMedian = cut at the median index
  uint32_t nleft;
  uint32_t slot;  // index in the current level's active list; kInactive otherwise
  uint32_t pad;
};
static_assert(sizeof(BNode) == 64, "BNode");

struct BuildCounters {
  uint32_t pool;        // nodes allocated
  uint32_t n_active[2]; // phase-A active lists (ping-pong)
  uint32_t n_subtrees;
  uint32_t max_depth;
  uint32_t n_leaves;
  uint32_t error;
  uint32_t n_mids;      // nodes handed to the one-CTA-per-node middle phase
};

// order-preserving float <-> uint key for atomicMin / atomicMax
__device__ __forceinline__ uint32_t fkey(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float funkey(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k ^ 0x80000000u) : ~k);
}

// The ordered key of a scalar type: key(a) < key(b) iff a < b (and -0 < +0); kMax is above every key.
template <typename T>
struct OrderedKey;
template <>
struct OrderedKey<float> {
  typedef uint32_t Key;
  static constexpr Key kMax = 0xFFFFFFFFu;
  static __device__ __forceinline__ Key key(float f) { return fkey(f); }
  static __device__ __forceinline__ float unkey(Key k) { return funkey(k); }
};
template <>
struct OrderedKey<double> {
  typedef unsigned long long Key;
  static constexpr Key kMax = 0xFFFFFFFFFFFFFFFFull;
  static __device__ __forceinline__ Key key(double f) {
    const Key u = (Key)__double_as_longlong(f);
    return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
  }
  static __device__ __forceinline__ double unkey(Key k) {
    return __longlong_as_double((long long)((k & 0x8000000000000000ull) ? (k ^ 0x8000000000000000ull) : ~k));
  }
};

template <typename T>
__device__ __forceinline__ T box_area(T lx, T ly, T lz, T hx, T hy, T hz) {
  T dx = hx - lx, dy = hy - ly, dz = hz - lz;
  return T(2) * ((dx * dy + dy * dz) + dz * dx);  // CalculateSurfaceArea, nanort.h:1278-1283
}

template <typename T>
__device__ __forceinline__ int bin_of(T c, T nmin, T inv, int B) {
  T q = (c - nmin) * inv;
  int qi = (int)q;  // truncation, as the reference's int(quantized_center[j])
  qi = qi < 0 ? 0 : qi;
  return qi > B - 1 ? B - 1 : qi;
}

template <typename T>
__device__ __forceinline__ T inv_extent(T lo, T hi, int B) {
  T sz = hi - lo;
  return sz > T(0) ? (T)B / sz : T(0);
}

constexpr int kAggregateMin = 6;

// One primitive into its bin record {count, kmin xyz, kmax xyz} -- warp-aggregated: lanes whose primitives fall
// into the same record (after the Morton pre-sort that is most of the warp) are combined with match_any + redux
// first, then ONE lane per distinct record issues the seven atomics.  `key` identifies the record (any value that
// is equal exactly for equal `rec`); every lane of the warp must call, lanes without a primitive pass valid=false.
__device__ __forceinline__ void bin_add_aggregated(uint32_t *rec, uint32_t key, bool valid, const uint32_t kl[3],
                                                   const uint32_t kh[3]) {
  const unsigned group = __match_any_sync(0xFFFFFFFFu, valid ? key : 0xFFFFFFFFu);
  if (!valid) return;
  const int members = __popc(group);
  if (members < kAggregateMin) {  // few lanes share the record: plain atomics are cheaper than six reductions
    atomicAdd(rec, 1u);
    atomicMin(rec + 1, kl[0]);
    atomicMin(rec + 2, kl[1]);
    atomicMin(rec + 3, kl[2]);
    atomicMax(rec + 4, kh[0]);
    atomicMax(rec + 5, kh[1]);
    atomicMax(rec + 6, kh[2]);
    return;
  }
  const uint32_t l0 = __reduce_min_sync(group, kl[0]), l1 = __reduce_min_sync(group, kl[1]),
                 l2 = __reduce_min_sync(group, kl[2]);
  const uint32_t h0 = __reduce_max_sync(group, kh[0]), h1 = __reduce_max_sync(group, kh[1]),
                 h2 = __reduce_max_sync(group, kh[2]);
  if ((int)(threadIdx.x & 31) == __ffs(group) - 1) {
    atomicAdd(rec, (uint32_t)members);
    atomicMin(rec + 1, l0);
    atomicMin(rec + 2, l1);
    atomicMin(rec + 3, l2);
    atomicMax(rec + 4, h0);
    atomicMax(rec + 5, h1);
    atomicMax(rec + 6, h2);
  }
}

// ------------------------------------------------------------------ SAH sweep (one warp, one axis)
template <typename T>
struct Box6T {
  T v[6];  // min xyz, max xyz
};
typedef Box6T<float> Box6;
template <typename T>
__device__ __forceinline__ void box_empty(Box6T<T> &b) {
  const T m = cuda::std::numeric_limits<T>::max();
  b.v[0] = b.v[1] = b.v[2] = m;
  b.v[3] = b.v[4] = b.v[5] = -m;
}
template <typename T>
__device__ __forceinline__ void box_merge_bin(Box6T<T> &b, const typename OrderedKey<T>::Key *w) {
  if (w[0] == 0u) return;
#pragma unroll
  for (int k = 0; k < 3; k++) {
    b.v[k] = fmin(b.v[k], OrderedKey<T>::unkey(w[1 + k]));
    b.v[3 + k] = fmax(b.v[3 + k], OrderedKey<T>::unkey(w[4 + k]));
  }
}
template <typename T>
__device__ __forceinline__ void box_merge(Box6T<T> &b, const Box6T<T> &o) {
#pragma unroll
  for (int k = 0; k < 3; k++) {
    b.v[k] = fmin(b.v[k], o.v[k]);
    b.v[3 + k] = fmax(b.v[3 + k], o.v[3 + k]);
  }
}

// For one axis (bins: B x kBinWords keys, any address space) finds the boundary i in [1, B-1] that
// minimises N_L*area(L) + N_R*area(R) with both sides non-empty; first minimum wins.  All 32 lanes call
// it; cost_l / cost_r are B-element scratch areas (shared).  Returns cost = numeric_limits<T>::max() when no
// boundary separates the centroids.
template <typename T>
__device__ void sweep_axis(const typename OrderedKey<T>::Key *bins, int B, T *cost_l, T *cost_r, T &best_cost,
                           int &best_i) {
  const int lane = threadIdx.x & 31;
  const int chunk = (B + 31) / 32;
  const int b0 = lane * chunk, b1 = min(B, b0 + chunk);
  // chunk totals
  Box6T<T> tot;
  box_empty(tot);
  uint32_t cnt = 0;
  for (int b = b0; b < b1; b++) {
    box_merge_bin(tot, bins + (size_t)b * kBinWords);
    cnt += (uint32_t)bins[(size_t)b * kBinWords];
  }
  // exclusive prefix (left) and exclusive suffix (right) of the chunk totals across lanes
  Box6T<T> pre = tot, suf = tot;
  uint32_t pcnt = cnt, scnt = cnt;
  for (int o = 1; o < 32; o <<= 1) {
    Box6T<T> t;
    uint32_t tc = __shfl_up_sync(0xFFFFFFFFu, pcnt, o);
    for (int k = 0; k < 6; k++) t.v[k] = __shfl_up_sync(0xFFFFFFFFu, pre.v[k], o);
    if (lane >= o) {
      box_merge(pre, t);
      pcnt += tc;
    }
    uint32_t uc = __shfl_down_sync(0xFFFFFFFFu, scnt, o);
    for (int k = 0; k < 6; k++) t.v[k] = __shfl_down_sync(0xFFFFFFFFu, suf.v[k], o);
    if (lane + o < 32) {
      box_merge(suf, t);
      scnt += uc;
    }
  }
  // inclusive -> exclusive
  Box6T<T> epre, esuf;
  uint32_t epc = __shfl_up_sync(0xFFFFFFFFu, pcnt, 1), esc = __shfl_down_sync(0xFFFFFFFFu, scnt, 1);
  for (int k = 0; k < 6; k++) {
    epre.v[k] = __shfl_up_sync(0xFFFFFFFFu, pre.v[k], 1);
    esuf.v[k] = __shfl_down_sync(0xFFFFFFFFu, suf.v[k], 1);
  }
  if (lane == 0) {
    box_empty(epre);
    epc = 0;
  }
  if (lane == 31) {
    box_empty(esuf);
    esc = 0;
  }
  // walk the chunk: cost_l[i] = cost of the left side for boundary i (bins [0,i)); cost_r[i] for [i,B)
  {
    Box6T<T> run = epre;
    uint32_t rc = epc;
    for (int b = b0; b < b1; b++) {
      // boundary i = b: left side is everything before bin b
      cost_l[b] = rc ? (T)rc * box_area(run.v[0], run.v[1], run.v[2], run.v[3], run.v[4], run.v[5]) : T(-1);
      box_merge_bin(run, bins + (size_t)b * kBinWords);
      rc += (uint32_t)bins[(size_t)b * kBinWords];
    }
    run = esuf;
    rc = esc;
    for (int b = b1 - 1; b >= b0; b--) {
      box_merge_bin(run, bins + (size_t)b * kBinWords);
      rc += (uint32_t)bins[(size_t)b * kBinWords];
      // boundary i = b: right side is bins [b, B)
      cost_r[b] = rc ? (T)rc * box_area(run.v[0], run.v[1], run.v[2], run.v[3], run.v[4], run.v[5]) : T(-1);
    }
  }
  __syncwarp();
  T bc = cuda::std::numeric_limits<T>::max();
  int bi = 0x7FFFFFFF;
  for (int i = 1 + lane; i < B; i += 32) {
    T cl = cost_l[i], cr = cost_r[i];
    if (cl < T(0) || cr < T(0)) continue;  // an empty side never wins (the reference's 0*inf = NaN)
    T c = cl + cr;
    if (c < bc) {
      bc = c;
      bi = i;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    T oc = __shfl_xor_sync(0xFFFFFFFFu, bc, o);
    int oi = __shfl_xor_sync(0xFFFFFFFFu, bi, o);
    if (oc < bc || (oc == bc && oi < bi)) {
      bc = oc;
      bi = oi;
    }
  }
  best_cost = bc;
  best_i = bi;
  __syncwarp();
}

// union / count of bins [lo, hi) of one axis, all lanes get the result
__device__ void range_union(const uint32_t *bins, int lo, int hi, Box6 &out, uint32_t &cnt) {
  const int lane = threadIdx.x & 31;
  Box6 b;
  box_empty(b);
  uint32_t c = 0;
  for (int i = lo + lane; i < hi; i += 32) {
    box_merge_bin(b, bins + (size_t)i * kBinWords);
    c += bins[(size_t)i * kBinWords];
  }
  for (int o = 16; o > 0; o >>= 1) {
    c += __shfl_xor_sync(0xFFFFFFFFu, c, o);
    for (int k = 0; k < 3; k++) {
      b.v[k] = fminf(b.v[k], __shfl_xor_sync(0xFFFFFFFFu, b.v[k], o));
      b.v[3 + k] = fmaxf(b.v[3 + k], __shfl_xor_sync(0xFFFFFFFFu, b.v[3 + k], o));
    }
  }
  out = b;
  cnt = c;
}


}  // namespace
}  // namespace nrt
