// Fast path of BVHAccel<double>::Traverse (included by f64.cu, inside its anonymous namespace): the design of
// traverse_fast3_kernel (traverse3.cuh) with every value the reference computes in double kept in double.
//
//   * PairNodeD, 256 B per branch: per axis {lo0 lo1 hi0 hi1 | hi0 hi1 lo0 lo1}; a ray reads four doubles per axis at
//     element offset (dir < 0 ? 4 : 0) and finds {near0 near1 far0 far1} -- the `ray_dir_sign ? bmax : bmin` selection
//     of IntersectRayAABB<double> (nanort.h:2327-2370) is an address.
//   * TriD, 96 B per indices_ slot in leaf order, component-major {a.k b.k c.k w}, w = prim id | last-in-leaf << 31:
//     the (kx, ky, kz) permutation of the watertight test (nanort.h:1073-1081) is the load address, and the
//     indices_ -> faces -> vertices chain of the reference-order kernel is gone.
//   * persistent warps, rays pulled from a global cursor when >= 16 lanes have retired, while-while over child pairs
//     with one postponed leaf per lane, near child first by entry distance, per-lane stack of (ref, entry distance).
//
// Arithmetic: (plane - org) * inv_dir per plane, far planes widened by 1.0000000000000004 (once per box: rounding is
// monotonic, min(a w, b w, c w) == min(a, b, c) w), NaN plane values dropped like safemax / safemin do, the triangle
// test operation for operation that of tri_test<double> -- so a reported record carries the reference's bits for its
// primitive.
// Visiting order differs from the reference's, hence which of two primitives hit at exactly the same t is reported may
// differ (the same contract as the float fast kernel; NRT_TRAVERSE_CONFORMANCE selects the reference-order kernel).
#pragma once

struct PairNodeD {
  double x[8], y[8], z[8];
  int ref0, ref1;
  int pad[14];
};
static_assert(sizeof(PairNodeD) == 256, "PairNodeD");
struct TriD {
  double c[3][4];
};
static_assert(sizeof(TriD) == 96, "TriD");

__device__ __forceinline__ double word_as_double(uint32_t w) { return __longlong_as_double((long long)(unsigned long long)w); }
__device__ __forceinline__ uint32_t double_as_word(double d) { return (uint32_t)(unsigned long long)__double_as_longlong(d); }

__global__ void f64_tris_kernel(const uint32_t *__restrict__ indices, const uint32_t *__restrict__ faces,
                                const double *__restrict__ verts, uint32_t n, TriD *__restrict__ out) {
  const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= n) return;
  const uint32_t prim = indices[slot];
  const double *p0 = verts + 3 * (size_t)faces[3 * (size_t)prim];
  const double *p1 = verts + 3 * (size_t)faces[3 * (size_t)prim + 1];
  const double *p2 = verts + 3 * (size_t)faces[3 * (size_t)prim + 2];
  TriD t;
  for (int k = 0; k < 3; k++) {
    t.c[k][0] = p0[k];
    t.c[k][1] = p1[k];
    t.c[k][2] = p2[k];
    t.c[k][3] = word_as_double(prim & 0x7FFFFFFFu);
  }
  out[slot] = t;
}

__device__ __forceinline__ void f64_put_child(PairNodeD &p, int which, const Node64 &c, bool empty) {
  double lo[3], hi[3];
  for (int k = 0; k < 3; k++) {
    // a child without primitives carries an inverted box: it can never pass the slab test
    lo[k] = empty ? DBL_MAX : c.bmin[k];
    hi[k] = empty ? -DBL_MAX : c.bmax[k];
  }
  double *ax[3] = {p.x, p.y, p.z};
  for (int k = 0; k < 3; k++) {
    ax[k][0 + which] = lo[k];
    ax[k][2 + which] = hi[k];
    ax[k][4 + which] = hi[k];
    ax[k][6 + which] = lo[k];
  }
}

__global__ void f64_pair_kernel(const Node64 *__restrict__ nodes, uint32_t n, const uint32_t *__restrict__ widx,
                                PairNodeD *__restrict__ pair, TriD *__restrict__ tris) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Node64 nd = nodes[i];
  if (nd.flag != 0) {
    if (nd.data[0] > 0) {  // mark the leaf's last triangle: the traversal needs no count
      TriD *t = tris + (size_t)nd.data[1] + nd.data[0] - 1;
      for (int k = 0; k < 3; k++) t->c[k][3] = word_as_double(double_as_word(t->c[k][3]) | 0x80000000u);
    }
    if (i == 0) {  // the whole tree is one leaf: a pair whose second child is empty
      PairNodeD p;
      f64_put_child(p, 0, nd, nd.data[0] == 0);
      f64_put_child(p, 1, nd, true);
      p.ref0 = nd.data[0] ? ~(int)nd.data[1] : kEmptyLeaf;
      p.ref1 = kEmptyLeaf;
      for (int k = 0; k < 14; k++) p.pad[k] = 0;
      pair[0] = p;
    }
    return;
  }
  const Node64 c0 = nodes[nd.data[0]], c1 = nodes[nd.data[1]];
  PairNodeD p;
  f64_put_child(p, 0, c0, c0.flag != 0 && c0.data[0] == 0);
  f64_put_child(p, 1, c1, c1.flag != 0 && c1.data[0] == 0);
  p.ref0 = child_ref(c0, nd.data[0], widx);
  p.ref1 = child_ref(c1, nd.data[1], widx);
  for (int k = 0; k < 14; k++) p.pad[k] = 0;
  pair[widx[i]] = p;
}

struct FastCtxD {
  double ox, oy, oz, ix, iy, iz, Sx, Sy, Sz, okx, oky, okz, t_min;
  uint32_t nx, ny, nz;  // element offset of {near0 near1 far0 far1} inside an axis block: 0 or 4
  uint32_t tx, ty, tz;  // component kx / ky / kz
};

__device__ __forceinline__ void ld4(const double *p, double &a, double &b, double &c, double &d) {
  const double2 u = __ldg(reinterpret_cast<const double2 *>(p));
  const double2 v = __ldg(reinterpret_cast<const double2 *>(p) + 1);
  a = u.x, b = u.y, c = v.x, d = v.y;
}

constexpr int kNoneD = kEmptyLeaf;
constexpr int kFastBlockD = 128;
constexpr int kFastBlocksPerSmD = 4;

template <int DEPTH>
__global__ void __launch_bounds__(kFastBlockD, kFastBlocksPerSmD)
    traverse_fast_f64_kernel(const PairNodeD *__restrict__ pair, const TriD *__restrict__ tris,
                             const Ray72 *__restrict__ rays, size_t n, Hit32 *__restrict__ hits,
                             uint8_t *__restrict__ mask, TraceOptions16 opt, uint32_t flags, unsigned long long *cursor) {
  const int lane = threadIdx.x & 31;
  const unsigned lt_mask = (1u << lane) - 1u;
  const unsigned FULL = 0xFFFFFFFFu;
  const bool cpp03 = (flags & NRT_TRAVERSE_CPP03_INVERSE) != 0;
  int sref[DEPTH];
  double sdist[DEPTH];
  int sp = 0;
  FastCtxD c;
  BestT<double> best;
  double min_t = 0.0, max_t = 0.0;
  size_t ray_idx = 0;
  bool alive = false, exhausted = false;
  int cur = kNoneD, leaf = kNoneD;

  for (;;) {
    // ---- replace retired rays (warp-ballot compaction of the ray pool)
    const unsigned dead = __ballot_sync(FULL, !alive);
    if (dead != 0u && !exhausted && (dead == FULL || __popc(dead) >= 16)) {
      const int cnt = __popc(dead);
      const int leader = __ffs(dead) - 1;
      unsigned long long base = 0;
      if (lane == leader) base = atomicAdd(cursor, (unsigned long long)cnt);
      base = __shfl_sync(FULL, base, leader);
      if (base + (unsigned long long)cnt >= (unsigned long long)n) exhausted = true;
      if (!alive) {
        const unsigned long long mine = base + (unsigned long long)__popc(dead & lt_mask);
        if (mine < (unsigned long long)n) {
          const Ray72 r = rays[mine];
          RayCtxT<double> rc;
          setup_ray(rc, r.org[0], r.org[1], r.org[2], r.dir[0], r.dir[1], r.dir[2], r.min_t, cpp03);
          c.ox = rc.ox, c.oy = rc.oy, c.oz = rc.oz;
          c.ix = rc.ix, c.iy = rc.iy, c.iz = rc.iz;
          c.Sx = rc.Sx, c.Sy = rc.Sy, c.Sz = rc.Sz;
          c.okx = sel3(rc.kx, rc.ox, rc.oy, rc.oz);
          c.oky = sel3(rc.ky, rc.ox, rc.oy, rc.oz);
          c.okz = sel3(rc.kz, rc.ox, rc.oy, rc.oz);
          c.t_min = r.min_t;
          c.nx = rc.sx ? 4u : 0u;
          c.ny = rc.sy ? 4u : 0u;
          c.nz = rc.sz ? 4u : 0u;
          c.tx = (uint32_t)rc.kx, c.ty = (uint32_t)rc.ky, c.tz = (uint32_t)rc.kz;
          min_t = r.min_t;
          max_t = r.max_t;
          best.t = r.max_t;
          best.u = 0.0;
          best.v = 0.0;
          best.prim = 0xFFFFFFFFu;
          ray_idx = (size_t)mine;
          alive = true;
          sp = 0;
          // a NaN in min_t / max_t makes every slab test of the reference fail (safemax / safemin keep the NaN that sits
          // in their second slot): such a ray misses everything
          cur = (min_t != min_t || max_t != max_t) ? kNoneD : 0;
          leaf = kNoneD;
        }
      }
    }
    if (__all_sync(FULL, !alive)) {
      if (exhausted) break;
      continue;
    }

    // ---- inner nodes
    for (;;) {
      const bool want = cur >= 0 || (cur == kNoneD && sp > 0);
      const unsigned desc = __ballot_sync(FULL, want);
      if (desc == 0u) break;
      if (__popc(desc) < 8 && __any_sync(FULL, leaf != kNoneD)) break;
      if (want) {
        while (cur == kNoneD && sp > 0) {  // entries that start behind the current best are dropped (nanort.h:2532)
          --sp;
          if (sdist[sp] <= best.t) {
            cur = sref[sp];
            if (cur < 0 && leaf == kNoneD) {
              leaf = cur;
              cur = kNoneD;
            }
          }
        }
        if (cur >= 0) {
          const PairNodeD *nd = pair + cur;
          double n0, n1, f0, f1;
          ld4(nd->x + c.nx, n0, n1, f0, f1);
          const double n0x = (n0 - c.ox) * c.ix, n1x = (n1 - c.ox) * c.ix;
          const double f0x = (f0 - c.ox) * c.ix, f1x = (f1 - c.ox) * c.ix;
          ld4(nd->y + c.ny, n0, n1, f0, f1);
          const double n0y = (n0 - c.oy) * c.iy, n1y = (n1 - c.oy) * c.iy;
          const double f0y = (f0 - c.oy) * c.iy, f1y = (f1 - c.oy) * c.iy;
          ld4(nd->z + c.nz, n0, n1, f0, f1);
          const double n0z = (n0 - c.oz) * c.iz, n1z = (n1 - c.oz) * c.iz;
          const double f0z = (f0 - c.oz) * c.iz, f1z = (f1 - c.oz) * c.iz;
          const int2 R = __ldg(reinterpret_cast<const int2 *>(&nd->ref0));
          const double t0 = fmax(fmax(fmax(n0x, n0y), n0z), min_t);
          const double t1 = fmax(fmax(fmax(n1x, n1y), n1z), min_t);
          const double e0 = fmin(fmin(fmin(f0x, f0y), f0z) * 1.0000000000000004, best.t);
          const double e1 = fmin(fmin(fmin(f1x, f1y), f1z) * 1.0000000000000004, best.t);
          const bool h0 = t0 <= e0, h1 = t1 <= e1;
          const bool swap = t1 < t0;
          const bool both = h0 & h1;
          if (both) {
            sref[sp] = swap ? R.x : R.y;
            sdist[sp] = swap ? t0 : t1;
            sp++;
          }
          cur = both ? (swap ? R.y : R.x) : (h0 ? R.x : (h1 ? R.y : kNoneD));
          if (cur < 0 && cur != kNoneD && leaf == kNoneD) {  // postpone the first leaf, keep descending
            leaf = cur;
            cur = kNoneD;
          }
        }
      }
    }

    // ---- leaves
    for (;;) {
      if (!__any_sync(FULL, leaf != kNoneD)) break;
      if (leaf != kNoneD) {
        uint32_t slot = (uint32_t)(~leaf);
        for (;;) {
          const TriD *t = tris + slot;
          double ax, bx, cx, wx, ay, by, cy, wy, az, bz, cz, wz;
          ld4(t->c[c.tx], ax, bx, cx, wx);
          ld4(t->c[c.ty], ay, by, cy, wy);
          ld4(t->c[c.tz], az, bz, cz, wz);
          (void)wy;
          (void)wz;
          const uint32_t w = double_as_word(wx);
          const uint32_t prim = w & 0x7FFFFFFFu;
          bool rej = (prim < opt.prim_ids_range[0]) | (prim >= opt.prim_ids_range[1]) | (prim == opt.skip_prim_id);
          // arithmetic order of nanort.h:1073-1147 (tri_test<double>), the permutation already applied by the loads
          const double Akx = ax - c.okx, Bkx = bx - c.okx, Ckx = cx - c.okx;
          const double Aky = ay - c.oky, Bky = by - c.oky, Cky = cy - c.oky;
          const double Akz = az - c.okz, Bkz = bz - c.okz, Ckz = cz - c.okz;
          const double Ax = Akx - c.Sx * Akz, Ay = Aky - c.Sy * Akz;
          const double Bx = Bkx - c.Sx * Bkz, By = Bky - c.Sy * Bkz;
          const double Cx = Ckx - c.Sx * Ckz, Cy = Cky - c.Sy * Ckz;
          const double U = Cx * By - Cy * Bx;
          const double V = Ax * Cy - Ay * Cx;
          const double W = Bx * Ay - By * Ax;
          const bool neg = (U < 0.0) | (V < 0.0) | (W < 0.0);
          const bool pos = (U > 0.0) | (V > 0.0) | (W > 0.0);
          rej |= neg & ((opt.cull_back_face != 0) | pos);
          const double det = (U + V) + W;
          rej |= (det == 0.0);
          if (!rej) {
            const double Az = c.Sz * Akz, Bz = c.Sz * Bkz, Cz = c.Sz * Ckz;
            const double D = (U * Az + V * Bz) + W * Cz;
            const double rcp = 1.0 / det;
            const double tt = D * rcp;
            if (!(tt > best.t) && !(tt < c.t_min)) {
              best.t = tt;
              best.u = V * rcp;
              best.v = W * rcp;
              best.prim = prim;
            }
          }
          if ((int)w < 0) break;  // last triangle of the leaf
          slot++;
        }
        leaf = kNoneD;
        if (cur < 0 && cur != kNoneD) {  // a second leaf was waiting
          leaf = cur;
          cur = kNoneD;
        }
      }
    }

    // ---- retire
    const bool retiring = alive && cur == kNoneD && leaf == kNoneD && sp == 0;
    if (retiring) {
      const bool hit = best.t < max_t;  // a hit exactly at max_t is a miss (nanort.h:2552)
      Hit32 h;
      h.u = hit ? best.u : 0.0;
      h.v = hit ? best.v : 0.0;
      h.t = hit ? best.t : max_t;
      h.prim_id = hit ? best.prim : 0xFFFFFFFFu;
      h.pad = 0;
      hits[ray_idx] = h;
      if (mask) mask[ray_idx] = hit ? 1 : 0;
      alive = false;
    }
  }
}
