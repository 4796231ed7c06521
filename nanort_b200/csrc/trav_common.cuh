// Per-ray device helpers shared by the traversal kernels (traverse.cu, f64.cu), the two-level scene kernels (scene.cu)
// and the primitive kernels (prims.cu): ray constants, the slab test, the watertight triangle test and the
// reference-order walk, all in the reference's arithmetic order (compiled with --fmad=false).
#pragma once
#include <float.h>
#include <math_constants.h>

#include "common.cuh"

namespace nrt {

#define FULL_MASK 0xFFFFFFFFu

// ------------------------------------------------------------------ per-ray constants
// The reference's per-ray pieces are templates over its scalar type (BVHAccel<float> / BVHAccel<double>); so are these.
// Real<T>: what differs between the two: vsafe_inverse's epsilon, the far-plane widening, the sign bit.
template <typename T>
struct Real;
template <>
struct Real<float> {
  static constexpr float kEps = FLT_EPSILON;
  static constexpr float kWiden = 1.00000024f;  // far planes widened by 2 ulp (nanort.h:2305)
  static constexpr int kSignBit = 31;
  __device__ __forceinline__ static float inf() { return CUDART_INF_F; }
  __device__ __forceinline__ static uint32_t bits(float d) { return __float_as_uint(d); }
};
template <>
struct Real<double> {
  static constexpr double kEps = DBL_EPSILON;
  static constexpr double kWiden = 1.0000000000000004;  // likewise (nanort.h:2348)
  static constexpr int kSignBit = 63;
  __device__ __forceinline__ static double inf() { return CUDART_INF; }
  __device__ __forceinline__ static unsigned long long bits(double d) {
    return (unsigned long long)__double_as_longlong(d);
  }
};

template <typename T>
struct RayCtxT {
  T ox, oy, oz;
  T ix, iy, iz;  // vsafe_inverse(dir)
  T Sx, Sy, Sz;  // watertight shear constants
  T t_min;
  int sx, sy, sz;  // dir < 0
  int kx, ky, kz;
};
using RayCtx = RayCtxT<float>;

template <typename T>
__device__ __forceinline__ T safe_inverse(T d, bool cpp03) {
  if (fabs(d) < Real<T>::kEps) {
    // C++11 mode: copysign(1, d) -> -0 gives -inf; C++03 mode: (d < 0) ? -1 : 1 -> -0 gives +inf
    bool neg = cpp03 ? (d < T(0)) : (Real<T>::bits(d) >> Real<T>::kSignBit) != 0u;
    return neg ? -Real<T>::inf() : Real<T>::inf();
  }
  return T(1) / d;
}

template <typename T>
__device__ __forceinline__ T sel3(int k, T x, T y, T z) {
  return k == 0 ? x : (k == 1 ? y : z);
}

template <typename T>
__device__ __forceinline__ void setup_ray(RayCtxT<T> &c, T ox, T oy, T oz, T dx, T dy, T dz, T min_t, bool cpp03) {
  c.ox = ox;
  c.oy = oy;
  c.oz = oz;
  c.sx = dx < T(0);
  c.sy = dy < T(0);
  c.sz = dz < T(0);
  c.ix = safe_inverse(dx, cpp03);
  c.iy = safe_inverse(dy, cpp03);
  c.iz = safe_inverse(dz, cpp03);
  int kz = 0;
  T m = fabs(dx);
  if (m < fabs(dy)) {
    kz = 1;
    m = fabs(dy);
  }
  if (m < fabs(dz)) kz = 2;
  int kx = (kz == 2) ? 0 : kz + 1;
  int ky = (kx == 2) ? 0 : kx + 1;
  T dkz = sel3(kz, dx, dy, dz);
  if (dkz < T(0)) {
    int t = kx;
    kx = ky;
    ky = t;
  }
  c.kx = kx;
  c.ky = ky;
  c.kz = kz;
  c.Sx = sel3(kx, dx, dy, dz) / dkz;
  c.Sy = sel3(ky, dx, dy, dz) / dkz;
  c.Sz = T(1) / dkz;
  c.t_min = min_t;
}

// The fast kernels retire a ray with a NaN in min_t or max_t before it starts: the reference's safemax / safemin
// chains keep that NaN (it sits in the slot whose NaN is NOT dropped, nanort.h:2316-2321), so every slab test fails
// and the ray misses everything, while their fmaxf / fminf would drop it.
__device__ __forceinline__ bool range_has_nan(float min_t, float max_t) { return (min_t != min_t) | (max_t != max_t); }

// Slab test of one box (nanort.h:2284-2325) in fmaxf / fminf form, for kernels that also want the entry distance.
// fmaxf/fminf drop a NaN operand exactly like the reference's safemax/safemin do for the per-axis value in
// the first slot (SURVEY.md 7.4); the running value is never NaN (range_has_nan() rays never get here).
__device__ __forceinline__ bool slab(const RayCtx &c, float lox, float loy, float loz, float hix,
                                     float hiy, float hiz, float min_t, float max_t, float &tnear) {
  float nx = c.sx ? hix : lox, fx = c.sx ? lox : hix;
  float ny = c.sy ? hiy : loy, fy = c.sy ? loy : hiy;
  float nz = c.sz ? hiz : loz, fz = c.sz ? loz : hiz;
  float tnx = (nx - c.ox) * c.ix;
  float tny = (ny - c.oy) * c.iy;
  float tnz = (nz - c.oz) * c.iz;
  float tfx = ((fx - c.ox) * c.ix) * 1.00000024f;
  float tfy = ((fy - c.oy) * c.iy) * 1.00000024f;
  float tfz = ((fz - c.oz) * c.iz) * 1.00000024f;
  float tmin = fmaxf(tnz, fmaxf(tny, fmaxf(tnx, min_t)));
  float tmax = fminf(tfz, fminf(tfy, fminf(tfx, max_t)));
  tnear = tmin;
  return tmin <= tmax;
}

template <typename T>
struct BestT {
  T t, u, v;
  uint32_t prim;
};
using Best = BestT<float>;

// Watertight ray/triangle test, arithmetic order of nanort.h:1073-1147, vertices a, b, cc (x, y, z) of primitive
// `prim` already loaded.  Accepts t_min <= tt <= best.t (ties replace, like the reference).
template <typename T, typename Vec>
__device__ __forceinline__ bool tri_test(const RayCtxT<T> &c, const TraceOptions16 &opt, uint32_t prim, const Vec &a,
                                         const Vec &b, const Vec &cc, BestT<T> &best) {
  if (prim < opt.prim_ids_range[0] || prim >= opt.prim_ids_range[1]) return false;
  if (prim == opt.skip_prim_id) return false;
  T A0 = a.x - c.ox, A1 = a.y - c.oy, A2 = a.z - c.oz;
  T B0 = b.x - c.ox, B1 = b.y - c.oy, B2 = b.z - c.oz;
  T C0 = cc.x - c.ox, C1 = cc.y - c.oy, C2 = cc.z - c.oz;
  T Akz = sel3(c.kz, A0, A1, A2), Bkz = sel3(c.kz, B0, B1, B2), Ckz = sel3(c.kz, C0, C1, C2);
  T Ax = sel3(c.kx, A0, A1, A2) - c.Sx * Akz;
  T Ay = sel3(c.ky, A0, A1, A2) - c.Sy * Akz;
  T Bx = sel3(c.kx, B0, B1, B2) - c.Sx * Bkz;
  T By = sel3(c.ky, B0, B1, B2) - c.Sy * Bkz;
  T Cx = sel3(c.kx, C0, C1, C2) - c.Sx * Ckz;
  T Cy = sel3(c.ky, C0, C1, C2) - c.Sy * Ckz;
  T U = Cx * By - Cy * Bx;
  T V = Ax * Cy - Ay * Cx;
  T W = Bx * Ay - By * Ax;
  if (U == T(0) || V == T(0) || W == T(0)) {
    // the reference's "double precision fallback": exact products in binary64, one rounding in the subtraction, one
    // in the narrowing (for T = double the same expressions again, the same values)
    U = (T)((double)Cx * (double)By - (double)Cy * (double)Bx);
    V = (T)((double)Ax * (double)Cy - (double)Ay * (double)Cx);
    W = (T)((double)Bx * (double)Ay - (double)By * (double)Ax);
  }
  if (U < T(0) || V < T(0) || W < T(0)) {
    if (opt.cull_back_face || U > T(0) || V > T(0) || W > T(0)) return false;
  }
  T det = (U + V) + W;
  if (det == T(0)) return false;
  T Az = c.Sz * Akz, Bz = c.Sz * Bkz, Cz = c.Sz * Ckz;
  T D = (U * Az + V * Bz) + W * Cz;
  T rcp = T(1) / det;
  T tt = D * rcp;
  if (tt > best.t) return false;
  if (tt < c.t_min) return false;
  best.t = tt;
  best.u = V * rcp;
  best.v = W * rcp;
  best.prim = prim;
  return true;
}

// safemax / safemin of the reference: (a > b) ? a : b, (a < b) ? a : b -- a NaN in the first operand is dropped, a
// NaN in the second one wins
template <typename T>
__device__ __forceinline__ T smax(T a, T b) { return (a > b) ? a : b; }
template <typename T>
__device__ __forceinline__ T smin(T a, T b) { return (a < b) ? a : b; }

// ------------------------------------------------------------------ reference-order walk
// BVHAccel<T>::Traverse (nanort.h:2526-2547) over a nanort-layout node array (Node40 / Node64), one thread per ray:
// pop a node, slab-test it against [min_t, hit_t] (IntersectRayAABB, nanort.h:2284-2370, safemax / safemin form),
// push the far child and then the near one by dir_sign[axis], hand a leaf to leaf(first, count, hit_t), which tests
// the primitives in indices_ order and may lower hit_t.  With the reference's NaN rule a NaN in min_t, max_t or in an
// accepted t makes every later slab test fail: the walk pops what is left and visits nothing else, as the reference
// does.  counts (optional): += popped nodes, tested primitives.
constexpr int kRefStack = 512;  // kNANORT_MAX_STACK_DEPTH

template <typename T, typename NodeT, typename Leaf>
__device__ __forceinline__ void reference_walk(const NodeT *nodes, const RayCtxT<T> &c, T min_t, T hit_t, Leaf &&leaf,
                                               unsigned long long *counts = nullptr) {
  uint32_t stack[kRefStack];
  int sp = 0;
  stack[0] = 0;
  while (sp >= 0) {
    const NodeT *nd = nodes + stack[sp];
    sp--;
    if (counts) counts[0]++;
    const T *f = reinterpret_cast<const T *>(nd);  // bmin[3], bmax[3]
    const T lox = __ldg(f + 0), loy = __ldg(f + 1), loz = __ldg(f + 2);
    const T hix = __ldg(f + 3), hiy = __ldg(f + 4), hiz = __ldg(f + 5);
    const T tnx = ((c.sx ? hix : lox) - c.ox) * c.ix;
    const T tny = ((c.sy ? hiy : loy) - c.oy) * c.iy;
    const T tnz = ((c.sz ? hiz : loz) - c.oz) * c.iz;
    const T tfx = (((c.sx ? lox : hix) - c.ox) * c.ix) * Real<T>::kWiden;
    const T tfy = (((c.sy ? loy : hiy) - c.oy) * c.iy) * Real<T>::kWiden;
    const T tfz = (((c.sz ? loz : hiz) - c.oz) * c.iz) * Real<T>::kWiden;
    const T tmin = smax(tnz, smax(tny, smax(tnx, min_t)));
    const T tmax = smin(tfz, smin(tfy, smin(tfx, hit_t)));
    if (!(tmin <= tmax)) continue;
    const uint32_t d0 = __ldg(&nd->data[0]), d1 = __ldg(&nd->data[1]);
    if (__ldg(&nd->flag) == 0) {
      const int axis = __ldg(&nd->axis);
      const int sgn = axis == 0 ? c.sx : (axis == 1 ? c.sy : c.sz);
      if (sp + 2 < kRefStack) {  // the reference only asserts here (nanort.h:2550)
        stack[++sp] = sgn ? d0 : d1;
        stack[++sp] = sgn ? d1 : d0;
      }
    } else {
      if (counts) counts[1] += d0;
      leaf(d1, d0, hit_t);
    }
  }
}

// The leaf of the float walks over PackedTri slots (the triangles in indices_ order, layout.cu)
struct PackedTriLeaf {
  const PackedTri *tris;
  const RayCtx &c;
  const TraceOptions16 &opt;
  Best &best;
  __device__ __forceinline__ void operator()(uint32_t first, uint32_t count, float &hit_t) const {
    bool any = false;
    for (uint32_t k = 0; k < count; k++) {
      const float4 *t = reinterpret_cast<const float4 *>(tris + (size_t)first + k);
      const float4 a = __ldg(t), b = __ldg(t + 1), cc = __ldg(t + 2);
      if (tri_test(c, opt, __float_as_uint(a.w), a, b, cc, best)) any = true;
    }
    if (any) hit_t = best.t;
  }
};

__device__ __forceinline__ void write_result(Hit16 *hits, uint8_t *mask, size_t i, const Best &best,
                                             float max_t) {
  bool hit = best.t < max_t;  // a hit exactly at max_t is a miss (nanort.h:2552)
  float4 r;
  if (hit) {
    r = make_float4(best.u, best.v, best.t, __uint_as_float(best.prim));
  } else {
    r = make_float4(0.0f, 0.0f, max_t, __uint_as_float(0xFFFFFFFFu));
  }
  reinterpret_cast<float4 *>(hits)[i] = r;
  if (mask) mask[i] = hit ? 1 : 0;
}

// Branch-free form of tri_test for the fast kernels (same arithmetic, same acceptance rule).
__device__ __forceinline__ void tri_test2(const RayCtx &c, const TraceOptions16 &opt, float4 a, float4 b, float4 cc,
                                          Best &best) {
  const uint32_t prim = __float_as_uint(a.w);
  bool rej = (prim < opt.prim_ids_range[0]) | (prim >= opt.prim_ids_range[1]) | (prim == opt.skip_prim_id);
  const float A0 = a.x - c.ox, A1 = a.y - c.oy, A2 = a.z - c.oz;
  const float B0 = b.x - c.ox, B1 = b.y - c.oy, B2 = b.z - c.oz;
  const float C0 = cc.x - c.ox, C1 = cc.y - c.oy, C2 = cc.z - c.oz;
  const float Akz = sel3(c.kz, A0, A1, A2), Bkz = sel3(c.kz, B0, B1, B2), Ckz = sel3(c.kz, C0, C1, C2);
  const float Ax = sel3(c.kx, A0, A1, A2) - c.Sx * Akz;
  const float Ay = sel3(c.ky, A0, A1, A2) - c.Sy * Akz;
  const float Bx = sel3(c.kx, B0, B1, B2) - c.Sx * Bkz;
  const float By = sel3(c.ky, B0, B1, B2) - c.Sy * Bkz;
  const float Cx = sel3(c.kx, C0, C1, C2) - c.Sx * Ckz;
  const float Cy = sel3(c.ky, C0, C1, C2) - c.Sy * Ckz;
  float U = Cx * By - Cy * Bx;
  float V = Ax * Cy - Ay * Cx;
  float W = Bx * Ay - By * Ax;
  if (U == 0.0f || V == 0.0f || W == 0.0f) {  // rare: exact edge / vertex hits
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

}  // namespace nrt
