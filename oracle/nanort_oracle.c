/*
 * TEST INFRASTRUCTURE ONLY -- CPU restatement ("port") of the nanort hot path.
 *
 * This file is the parity oracle for the CUDA path.  Only tests/, the smoke()
 * entry point and bench.py's cpu_baseline / --impl reference legs may load it;
 * the product library (nanort_b200/libnanort_b200.so) never links or calls it
 * and has no CPU fallback.
 *
 * It restates, in plain C, the algorithm of the reference's nanort.h at commit
 * 3bbea5e for BVHAccel<float>::Build and BVHAccel<float>::Traverse with the
 * built-in triangle classes.  All arithmetic is IEEE binary32 with every
 * operation individually rounded: compile with -ffp-contract=off and without
 * -ffast-math (oracle/Makefile does).
 *
 * The same source compiled with -DORC_DOUBLE (oracle/liborc64.so) is the restatement of BVHAccel<double>; it is
 * pinned the same way against the reference's double instantiation (tests/test_oracle_f64.py).
 *
 * Parity status: PINNED.  tests/test_oracle_vs_reference.py checks this port
 * bit-for-bit (nodes, indices, statistics, hit flag, prim_id and the raw bits
 * of t/u/v) against the unmodified reference compiled into
 * oracle/_ref/libnanort_ref{,03}.so, and against the committed golden vectors
 * under tests/golden/ that were produced by that reference.
 *
 * Reference map (file:line in the reference tree):
 *   orc_prim_bbox            TriangleMesh::BoundingBox          nanort.h:934-956
 *   orc_prim_bbox_center     TriangleMesh::BoundingBoxAndCenter nanort.h:958-971
 *   orc_range_bbox           ComputeBoundingBox                 nanort.h:1545-1567
 *   orc_fill_bins            ContributeBinBuffer                nanort.h:1314-1367
 *   orc_find_cut             FindCutFromBinBuffer               nanort.h:1381-1430
 *   orc_area                 CalculateSurfaceArea               nanort.h:1278-1283
 *   orc_pred / orc_partition TriangleSAHPred::operator() nanort.h:897-911 and
 *                            std::partition (libstdc++ bidirectional variant,
 *                            bits/stl_algo.h __partition) used at nanort.h:1841
 *   orc_build_rec            BuildTree                          nanort.h:1759-1890
 *   orc_build_shallow_rec    BuildShallowTree                   nanort.h:1600-1757
 *   orc_build                Build (+ parallel join)            nanort.h:1892-2149
 *   orc_safe_inverse         vsafe_inverse                      nanort.h:414-465
 *   orc_slab                 IntersectRayAABB<float>            nanort.h:2284-2325
 *   orc_tri                  TriangleIntersector::Intersect     nanort.h:1054-1150
 *   orc_prepare              PrepareTraversal                   nanort.h:1163-1201
 *   orc_traverse_one         Traverse + TestLeafNode            nanort.h:2487-2556, 2372-2407
 */
#include <float.h>
#include <math.h>
#include <pthread.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ---- precision: the same restatement serves BVHAccel<float> (liborc.so) and, compiled with -DORC_DOUBLE,
 * BVHAccel<double> (liborc64.so).  The reference is a template over T; the only T-specific pieces are the far-plane
 * widening constant of IntersectRayAABB (nanort.h:2284-2325 float, 2327-2370 double) and numeric_limits<T>. */
#ifdef ORC_DOUBLE
typedef double real;
#define RC(x) x
#define R_MAX DBL_MAX
#define R_EPS DBL_EPSILON
#define R_FABS fabs
#define R_COPYSIGN copysign
#define R_MAXMULT 1.0000000000000004
#else
typedef float real;
#define RC(x) x##f
#define R_MAX FLT_MAX
#define R_EPS FLT_EPSILON
#define R_FABS fabsf
#define R_COPYSIGN copysignf
#define R_MAXMULT 1.00000024f
#endif

/* ---- value types, byte-compatible with the reference (SURVEY.md section 0.5) ---- */
typedef struct {
  real bmin[3];
  real bmax[3];
  int32_t flag; /* 1 leaf, 0 branch */
  int32_t axis;
  uint32_t data[2]; /* leaf {count, first}; branch {left, right} */
} orc_node; /* 40 B */

typedef struct {
  real org[3];
  real dir[3];
  real min_t;
  real max_t;
  uint32_t type;
} orc_ray; /* 36 B */

typedef struct {
  real u, v, t;
  uint32_t prim_id;
} orc_hit; /* 16 B */

typedef struct {
  real cost_t_aabb;
  uint32_t min_leaf_primitives;
  uint32_t max_tree_depth;
  uint32_t bin_size;
  uint32_t shallow_depth;
  uint32_t min_primitives_for_parallel_build;
  uint8_t cache_bbox;
  uint8_t pad[3];
} orc_build_options; /* 28 B */

typedef struct {
  uint32_t prim_ids_range[2];
  uint32_t skip_prim_id;
  uint8_t cull_back_face;
  uint8_t pad[3];
} orc_trace_options; /* 16 B */

typedef struct {
  uint32_t max_tree_depth;
  uint32_t num_leaf_nodes;
  uint32_t num_branch_nodes;
} orc_stats;

/* Build mode flags */
#define ORC_MODE_CPP11 1u    /* shallow tree + joined sub-arrays for n > threshold (nanort.h:1996-2068) */
#define ORC_MODE_FIXBINS 2u  /* NOT reference behaviour: bins all three axes (guard at nanort.h:1357 widened) */

void orc_default_build_options(orc_build_options *o) {
  memset(o, 0, sizeof(*o));
  o->cost_t_aabb = RC(0.2);
  o->min_leaf_primitives = 4;
  o->max_tree_depth = 256;
  o->bin_size = 64;
  o->shallow_depth = 4;
  o->min_primitives_for_parallel_build = 1024 * 8;
  o->cache_bbox = 0;
}

void orc_default_trace_options(orc_trace_options *o) {
  memset(o, 0, sizeof(*o));
  o->prim_ids_range[0] = 0;
  o->prim_ids_range[1] = 0x7FFFFFFFu;
  o->skip_prim_id = 0xFFFFFFFFu;
  o->cull_back_face = 0;
}

void orc_sizes(uint32_t out[5]) {
  out[0] = (uint32_t)sizeof(orc_node);
  out[1] = (uint32_t)sizeof(orc_ray);
  out[2] = (uint32_t)sizeof(orc_hit);
  out[3] = (uint32_t)sizeof(orc_build_options);
  out[4] = (uint32_t)sizeof(orc_trace_options);
}

/* std::min / std::max argument-order semantics (matters for -0.0 and NaN) */
static inline real stdmin(real a, real b) { return (b < a) ? b : a; }
static inline real stdmax(real a, real b) { return (a < b) ? b : a; }

/* ------------------------------------------------------------------ geometry */
typedef struct {
  const unsigned char *verts;
  size_t stride;
  const uint32_t *faces;
  /* box primitives (the two-level scene's top-level build): boxes[6*i] = bmin.xyz bmax.xyz; when set, the
   * accessors below follow NodeBBoxGeometry / NodeBBoxPred (examples/nanosg/nanosg.h:511-573) instead */
  const real *boxes;
} orc_mesh;

static inline const real *vtx(const orc_mesh *m, uint32_t i) {
  return (const real *)(m->verts + (size_t)i * m->stride);
}

static void orc_prim_bbox(const orc_mesh *m, uint32_t prim, real bmin[3], real bmax[3]) {
  if (m->boxes) {
    for (int k = 0; k < 3; k++) {
      bmin[k] = m->boxes[6 * (size_t)prim + k];
      bmax[k] = m->boxes[6 * (size_t)prim + 3 + k];
    }
    return;
  }
  const real *p = vtx(m, m->faces[3 * (size_t)prim]);
  for (int k = 0; k < 3; k++) bmin[k] = bmax[k] = p[k];
  for (int c = 1; c < 3; c++) {
    p = vtx(m, m->faces[3 * (size_t)prim + c]);
    for (int k = 0; k < 3; k++) {
      bmin[k] = stdmin(bmin[k], p[k]);
      bmax[k] = stdmax(bmax[k], p[k]);
    }
  }
}

static void orc_prim_bbox_center(const orc_mesh *m, uint32_t prim, real bmin[3], real bmax[3],
                                 real ctr[3]) {
  if (m->boxes) {
    orc_prim_bbox(m, prim, bmin, bmax);
    for (int k = 0; k < 3; k++) ctr[k] = (bmax[k] + bmin[k]) / RC(2.0);
    return;
  }
  const real *p0 = vtx(m, m->faces[3 * (size_t)prim + 0]);
  const real *p1 = vtx(m, m->faces[3 * (size_t)prim + 1]);
  const real *p2 = vtx(m, m->faces[3 * (size_t)prim + 2]);
  const real third = RC(1.0) / RC(3.0);
  for (int k = 0; k < 3; k++) {
    bmin[k] = stdmin(p0[k], stdmin(p1[k], p2[k]));
    bmax[k] = stdmax(p0[k], stdmax(p1[k], p2[k]));
    ctr[k] = ((p0[k] + p1[k]) + p2[k]) * third;
  }
}

static void orc_range_bbox(const orc_mesh *m, const uint32_t *idx, uint32_t l, uint32_t r,
                           real bmin[3], real bmax[3]) {
  orc_prim_bbox(m, idx[l], bmin, bmax);
  for (uint32_t i = l + 1; i < r; i++) {
    real a[3], b[3];
    orc_prim_bbox(m, idx[i], a, b);
    for (int k = 0; k < 3; k++) {
      bmin[k] = stdmin(bmin[k], a[k]);
      bmax[k] = stdmax(bmax[k], b[k]);
    }
  }
}

/* ------------------------------------------------------------------ SAH bins */
typedef struct {
  real bmin[3], bmax[3];
  size_t count;
  real cost;
} orc_bin;

static inline real orc_area(const real lo[3], const real hi[3]) {
  real dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
  return RC(2.0) * ((dx * dy + dy * dz) + dz * dx);
}

static void orc_bins_clear(orc_bin *bins, uint32_t B) {
  for (uint32_t i = 0; i < 3 * B; i++) {
    for (int k = 0; k < 3; k++) {
      bins[i].bmin[k] = R_MAX;
      bins[i].bmax[k] = -R_MAX;
    }
    bins[i].count = 0;
    bins[i].cost = RC(0.0);
  }
}

static void orc_fill_bins(orc_bin *bins, uint32_t B, uint32_t guard, const real nmin[3],
                          const real nmax[3], const orc_mesh *m, const uint32_t *idx, uint32_t l,
                          uint32_t r) {
  real inv[3];
  const real fB = (real)B;
  for (int k = 0; k < 3; k++) {
    real sz = nmax[k] - nmin[k];
    inv[k] = (sz > RC(0.0)) ? fB / sz : RC(0.0);
  }
  orc_bins_clear(bins, B);
  for (uint32_t i = l; i < r; i++) {
    real lo[3], hi[3], c[3];
    orc_prim_bbox_center(m, idx[i], lo, hi, c);
    for (int j = 0; j < 3; j++) {
      real q = (c[j] - nmin[j]) * inv[j];
      int qi = (int)q;
      if (qi < 0) qi = 0;
      uint32_t b = (uint32_t)qi;
      if (b > B - 1) b = B - 1;
      uint32_t slot = (uint32_t)j * B + b;
      /* guard == B reproduces the pinned commit: only axis 0 is ever binned
       * (SURVEY.md F1, nanort.h:1357).  guard == 3B is the ORC_MODE_FIXBINS
       * experiment, never used as the reference. */
      if (slot < guard) {
        orc_bin *bn = &bins[slot];
        bn->count++;
        for (int k = 0; k < 3; k++) {
          bn->bmin[k] = stdmin(bn->bmin[k], lo[k]);
          bn->bmax[k] = stdmax(bn->bmax[k], hi[k]);
        }
      }
    }
  }
}

static void orc_find_cut(orc_bin *bins, uint32_t B, const real nmin[3], const real nmax[3],
                         real cut_pos[3], int *best_axis) {
  real best[3];
  for (int j = 0; j < 3; j++) {
    orc_bin *ax = bins + (size_t)j * B;
    real lo[3] = {R_MAX, R_MAX, R_MAX}, hi[3] = {-R_MAX, -R_MAX, -R_MAX};
    size_t cnt = 0;
    best[j] = R_MAX;
    /* right-to-left: cost of the right-hand side starting at bin i */
    for (size_t i = B - 1; i > 0; i--) {
      for (int k = 0; k < 3; k++) {
        lo[k] = stdmin(ax[i].bmin[k], lo[k]);
        hi[k] = stdmax(ax[i].bmax[k], hi[k]);
      }
      cnt += ax[i].count;
      ax[i].cost = (real)cnt * orc_area(lo, hi);
    }
    for (int k = 0; k < 3; k++) {
      lo[k] = R_MAX;
      hi[k] = -R_MAX;
    }
    cnt = 0;
    size_t arg = 1;
    for (size_t i = 0; i + 1 < B; i++) {
      for (int k = 0; k < 3; k++) {
        lo[k] = stdmin(ax[i].bmin[k], lo[k]);
        hi[k] = stdmax(ax[i].bmax[k], hi[k]);
      }
      cnt += ax[i].count;
      real c = (real)cnt * orc_area(lo, hi) + ax[i + 1].cost;
      if (c < best[j]) {
        best[j] = c;
        arg = i + 1;
      }
    }
    cut_pos[j] = (real)arg * ((nmax[j] - nmin[j]) / (real)B) + nmin[j];
  }
  int a = 0;
  if (best[0] > best[1]) a = 1;
  if (best[a] > best[2]) a = 2;
  *best_axis = a;
}

static inline int orc_pred(const orc_mesh *m, uint32_t prim, int axis, real pos) {
  if (m->boxes) {
    const real *b = m->boxes + 6 * (size_t)prim;
    return (b[axis] + b[3 + axis]) / RC(2.0) < pos;
  }
  const real *p0 = vtx(m, m->faces[3 * (size_t)prim + 0]);
  const real *p1 = vtx(m, m->faces[3 * (size_t)prim + 1]);
  const real *p2 = vtx(m, m->faces[3 * (size_t)prim + 2]);
  real s = (p0[axis] + p1[axis]) + p2[axis];
  return s < pos * RC(3.0);
}

/* two-pointer in-place partition: element order after the call is the one
 * libstdc++'s std::partition (bidirectional iterators) leaves behind */
static uint32_t orc_partition(uint32_t *idx, uint32_t l, uint32_t r, const orc_mesh *m, int axis,
                              real pos) {
  uint32_t first = l, last = r;
  for (;;) {
    for (;;) {
      if (first == last) return first;
      if (orc_pred(m, idx[first], axis, pos))
        ++first;
      else
        break;
    }
    --last;
    for (;;) {
      if (first == last) return first;
      if (!orc_pred(m, idx[last], axis, pos))
        --last;
      else
        break;
    }
    uint32_t t = idx[first];
    idx[first] = idx[last];
    idx[last] = t;
    ++first;
  }
}

/* ------------------------------------------------------------------ builder */
typedef struct {
  orc_node *v;
  size_t n, cap;
} node_vec;

static size_t nv_push(node_vec *a, const orc_node *x) {
  if (a->n == a->cap) {
    a->cap = a->cap ? a->cap * 2 : 64;
    a->v = (orc_node *)realloc(a->v, a->cap * sizeof(orc_node));
  }
  a->v[a->n] = *x;
  return a->n++;
}

typedef struct {
  uint32_t l, r, offset;
} deferred_t;

typedef struct {
  orc_mesh mesh;
  orc_build_options opt;
  uint32_t guard;
  uint32_t *idx;
  orc_bin *bins; /* scratch 3*B, reused: recursion only needs it before descending */
  deferred_t *deferred;
  size_t n_deferred, cap_deferred;
} build_ctx;

/* chooses the split of [l,r): returns mid and the axis label the node gets */
static uint32_t orc_split(build_ctx *c, uint32_t l, uint32_t r, const real bmin[3],
                          const real bmax[3], int *axis_out) {
  real cut[3] = {RC(0.0), RC(0.0), RC(0.0)};
  int first_axis = 0;
  uint32_t n = r - l;
  orc_fill_bins(c->bins, c->opt.bin_size, c->guard, bmin, bmax, &c->mesh, c->idx, l, r);
  orc_find_cut(c->bins, c->opt.bin_size, bmin, bmax, cut, &first_axis);
  uint32_t mid = l;
  int axis = first_axis;
  for (int attempt = 0; attempt < 3; attempt++) {
    axis = (first_axis + attempt) % 3;
    mid = orc_partition(c->idx, l, r, &c->mesh, axis, cut[axis]);
    if (mid == l || mid == r) {
      mid = l + (n >> 1); /* object-median fallback; next axis is still tried */
    } else {
      break;
    }
  }
  *axis_out = axis;
  return mid;
}

static void set_box(orc_node *nd, const real bmin[3], const real bmax[3]) {
  for (int k = 0; k < 3; k++) {
    nd->bmin[k] = bmin[k];
    nd->bmax[k] = bmax[k];
  }
}

static uint32_t orc_build_rec(build_ctx *c, orc_stats *st, node_vec *out, uint32_t l, uint32_t r,
                              uint32_t depth) {
  uint32_t self = (uint32_t)out->n;
  if (st->max_tree_depth < depth) st->max_tree_depth = depth;
  real bmin[3], bmax[3];
  orc_range_bbox(&c->mesh, c->idx, l, r, bmin, bmax);
  uint32_t n = r - l;
  orc_node nd;
  memset(&nd, 0, sizeof(nd));
  if (n <= c->opt.min_leaf_primitives || depth >= c->opt.max_tree_depth) {
    set_box(&nd, bmin, bmax);
    nd.flag = 1;
    nd.axis = 0; /* the reference leaves leaf.axis uninitialised; never read */
    nd.data[0] = n;
    nd.data[1] = l;
    nv_push(out, &nd);
    st->num_leaf_nodes++;
    return self;
  }
  int axis;
  uint32_t mid = orc_split(c, l, r, bmin, bmax, &axis);
  nd.axis = axis;
  nd.flag = 0;
  nv_push(out, &nd);
  uint32_t lc = orc_build_rec(c, st, out, l, mid, depth + 1);
  uint32_t rc = orc_build_rec(c, st, out, mid, r, depth + 1);
  out->v[self].data[0] = lc;
  out->v[self].data[1] = rc;
  set_box(&out->v[self], bmin, bmax);
  st->num_branch_nodes++;
  return self;
}

static uint32_t orc_build_shallow_rec(build_ctx *c, orc_stats *st, node_vec *out, uint32_t l,
                                      uint32_t r, uint32_t depth, uint32_t max_shallow) {
  uint32_t self = (uint32_t)out->n;
  if (st->max_tree_depth < depth) st->max_tree_depth = depth;
  real bmin[3], bmax[3];
  orc_range_bbox(&c->mesh, c->idx, l, r, bmin, bmax);
  uint32_t n = r - l;
  orc_node nd;
  memset(&nd, 0, sizeof(nd));
  if (n <= c->opt.min_leaf_primitives || depth >= c->opt.max_tree_depth) {
    set_box(&nd, bmin, bmax);
    nd.flag = 1;
    nd.data[0] = n;
    nd.data[1] = l;
    nv_push(out, &nd);
    st->num_leaf_nodes++;
    return self;
  }
  if (depth >= max_shallow) {
    if (c->n_deferred == c->cap_deferred) {
      c->cap_deferred = c->cap_deferred ? c->cap_deferred * 2 : 32;
      c->deferred = (deferred_t *)realloc(c->deferred, c->cap_deferred * sizeof(deferred_t));
    }
    c->deferred[c->n_deferred].l = l;
    c->deferred[c->n_deferred].r = r;
    c->deferred[c->n_deferred].offset = self;
    c->n_deferred++;
    nd.flag = -1;
    nd.axis = -1;
    nv_push(out, &nd); /* placeholder, overwritten by the join */
    return self;
  }
  int axis;
  uint32_t mid = orc_split(c, l, r, bmin, bmax, &axis);
  nd.axis = axis;
  nd.flag = 0;
  nv_push(out, &nd);
  uint32_t lc = orc_build_shallow_rec(c, st, out, l, mid, depth + 1, max_shallow);
  uint32_t rc = orc_build_shallow_rec(c, st, out, mid, r, depth + 1, max_shallow);
  out->v[self].data[0] = lc;
  out->v[self].data[1] = rc;
  set_box(&out->v[self], bmin, bmax);
  st->num_branch_nodes++;
  return self;
}

/*
 * Builds the tree.  *nodes_out is malloc'ed (free with orc_free), indices_out
 * must hold n_prims entries.  Returns the node count, 0 when n_prims == 0
 * (reference Build returns false, nanort.h:1907-1909).
 */
static size_t orc_build_core(const orc_mesh *mesh, uint32_t n_prims, const orc_build_options *opts,
                             uint32_t mode, orc_node **nodes_out, uint32_t *indices_out,
                             orc_stats *stats_out) {
  build_ctx c;
  memset(&c, 0, sizeof(c));
  c.mesh = *mesh;
  if (opts)
    c.opt = *opts;
  else
    orc_default_build_options(&c.opt);
  orc_stats st = {0, 0, 0};
  *nodes_out = NULL;
  if (stats_out) *stats_out = st;
  if (n_prims == 0 || c.opt.bin_size < 2) return 0;
  c.guard = (mode & ORC_MODE_FIXBINS) ? 3 * c.opt.bin_size : c.opt.bin_size;
  c.idx = indices_out;
  for (uint32_t i = 0; i < n_prims; i++) c.idx[i] = i;
  c.bins = (orc_bin *)malloc(sizeof(orc_bin) * 3 * c.opt.bin_size);
  node_vec out = {NULL, 0, 0};

  if ((mode & ORC_MODE_CPP11) && n_prims > c.opt.min_primitives_for_parallel_build) {
    orc_build_shallow_rec(&c, &st, &out, 0, n_prims, 0, c.opt.shallow_depth);
    /* sub-trees are independent (disjoint index ranges), so building them one
     * after the other gives the arrays the reference's worker threads produce;
     * the join below follows nanort.h:2041-2067. */
    for (size_t s = 0; s < c.n_deferred; s++) {
      node_vec sub = {NULL, 0, 0};
      orc_stats ls = {0, 0, 0};
      orc_build_rec(&c, &ls, &sub, c.deferred[s].l, c.deferred[s].r, c.opt.shallow_depth);
      uint32_t base = (uint32_t)out.n;
      for (size_t j = 0; j < sub.n; j++) {
        if (sub.v[j].flag == 0) {
          sub.v[j].data[0] += base - 1;
          sub.v[j].data[1] += base - 1;
        }
      }
      out.v[c.deferred[s].offset] = sub.v[0];
      for (size_t j = 1; j < sub.n; j++) nv_push(&out, &sub.v[j]);
      if (ls.max_tree_depth > st.max_tree_depth) st.max_tree_depth = ls.max_tree_depth;
      st.num_leaf_nodes += ls.num_leaf_nodes;
      st.num_branch_nodes += ls.num_branch_nodes;
      free(sub.v);
    }
  } else {
    orc_build_rec(&c, &st, &out, 0, n_prims, 0);
  }
  free(c.bins);
  free(c.deferred);
  *nodes_out = out.v;
  if (stats_out) *stats_out = st;
  return out.n;
}

size_t orc_build(const real *verts, size_t stride, const uint32_t *faces, uint32_t n_prims,
                 const orc_build_options *opts, uint32_t mode, orc_node **nodes_out,
                 uint32_t *indices_out, orc_stats *stats_out) {
  orc_mesh m = {(const unsigned char *)verts, stride, faces, NULL};
  return orc_build_core(&m, n_prims, opts, mode, nodes_out, indices_out, stats_out);
}

/* the same Build over axis-aligned boxes as primitives (Scene::Commit's top-level build with
 * NodeBBoxGeometry / NodeBBoxPred, examples/nanosg/nanosg.h:722-737) */
size_t orc_build_boxes(const real *boxes6, uint32_t n_prims, const orc_build_options *opts, uint32_t mode,
                       orc_node **nodes_out, uint32_t *indices_out, orc_stats *stats_out) {
  orc_mesh m = {NULL, 0, NULL, boxes6};
  return orc_build_core(&m, n_prims, opts, mode, nodes_out, indices_out, stats_out);
}

void orc_free(void *p) { free(p); }

/* ------------------------------------------------------------------ traversal */
typedef struct {
  uint64_t nodes_popped; /* nanort.h:2527 */
  uint64_t prims_tested; /* nanort.h:2397 */
  uint32_t max_stack;    /* deepest node_stack index reached */
} orc_counters;

typedef struct {
  real org[3];
  real inv[3];
  int sign[3];
  int kx, ky, kz;
  real Sx, Sy, Sz;
  real t_min;
  orc_trace_options opt;
  /* running best */
  real t, u, v;
  uint32_t prim;
} ray_state;

static inline real orc_safe_inverse(real d, int cpp11) {
  if (R_FABS(d) < R_EPS) {
    real sgn;
    if (cpp11)
      sgn = R_COPYSIGN(RC(1.0), d); /* -0.0 -> -inf */
    else
      sgn = (d < RC(0.0)) ? -RC(1.0) : RC(1.0); /* -0.0 -> +inf */
    return INFINITY * sgn;
  }
  return RC(1.0) / d;
}

static void orc_prepare(ray_state *s, const orc_ray *ray, const orc_trace_options *opt, int cpp11) {
  for (int k = 0; k < 3; k++) {
    s->org[k] = ray->org[k];
    s->sign[k] = ray->dir[k] < RC(0.0) ? 1 : 0;
    s->inv[k] = orc_safe_inverse(ray->dir[k], cpp11);
  }
  int kz = 0;
  real m = R_FABS(ray->dir[0]);
  if (m < R_FABS(ray->dir[1])) {
    kz = 1;
    m = R_FABS(ray->dir[1]);
  }
  if (m < R_FABS(ray->dir[2])) {
    kz = 2;
  }
  int kx = kz + 1 == 3 ? 0 : kz + 1;
  int ky = kx + 1 == 3 ? 0 : kx + 1;
  if (ray->dir[kz] < RC(0.0)) {
    int t = kx;
    kx = ky;
    ky = t;
  }
  s->kx = kx;
  s->ky = ky;
  s->kz = kz;
  s->Sx = ray->dir[kx] / ray->dir[kz];
  s->Sy = ray->dir[ky] / ray->dir[kz];
  s->Sz = RC(1.0) / ray->dir[kz];
  s->t_min = ray->min_t;
  s->opt = *opt;
  s->u = RC(0.0);
  s->v = RC(0.0);
}

/* (a > b) ? a : b and (a < b) ? a : b, the reference's safemax / safemin */
static inline real smax(real a, real b) { return (a > b) ? a : b; }
static inline real smin(real a, real b) { return (a < b) ? a : b; }

static inline int orc_slab(const ray_state *s, const orc_node *nd, real min_t, real max_t) {
  real tn[3], tf[3];
  for (int k = 0; k < 3; k++) {
    real nearp = s->sign[k] ? nd->bmax[k] : nd->bmin[k];
    real farp = s->sign[k] ? nd->bmin[k] : nd->bmax[k];
    tn[k] = (nearp - s->org[k]) * s->inv[k];
    tf[k] = ((farp - s->org[k]) * s->inv[k]) * R_MAXMULT;
  }
  real tmin = smax(tn[2], smax(tn[1], smax(tn[0], min_t)));
  real tmax = smin(tf[2], smin(tf[1], smin(tf[0], max_t)));
  return tmin <= tmax;
}

static inline int orc_tri(ray_state *s, const orc_mesh *m, uint32_t prim, real *t_inout) {
  if (prim < s->opt.prim_ids_range[0] || prim >= s->opt.prim_ids_range[1]) return 0;
  if (prim == s->opt.skip_prim_id) return 0;
  const real *p0 = vtx(m, m->faces[3 * (size_t)prim + 0]);
  const real *p1 = vtx(m, m->faces[3 * (size_t)prim + 1]);
  const real *p2 = vtx(m, m->faces[3 * (size_t)prim + 2]);
  real A[3], B[3], C[3];
  for (int k = 0; k < 3; k++) {
    A[k] = p0[k] - s->org[k];
    B[k] = p1[k] - s->org[k];
    C[k] = p2[k] - s->org[k];
  }
  const int kx = s->kx, ky = s->ky, kz = s->kz;
  const real Ax = A[kx] - s->Sx * A[kz], Ay = A[ky] - s->Sy * A[kz];
  const real Bx = B[kx] - s->Sx * B[kz], By = B[ky] - s->Sy * B[kz];
  const real Cx = C[kx] - s->Sx * C[kz], Cy = C[ky] - s->Sy * C[kz];
  real U = Cx * By - Cy * Bx;
  real V = Ax * Cy - Ay * Cx;
  real W = Bx * Ay - By * Ax;
  if (U == RC(0.0) || V == RC(0.0) || W == RC(0.0)) {
    U = (real)((double)Cx * (double)By - (double)Cy * (double)Bx);
    V = (real)((double)Ax * (double)Cy - (double)Ay * (double)Cx);
    W = (real)((double)Bx * (double)Ay - (double)By * (double)Ax);
  }
  if (U < RC(0.0) || V < RC(0.0) || W < RC(0.0)) {
    if (s->opt.cull_back_face || U > RC(0.0) || V > RC(0.0) || W > RC(0.0)) return 0;
  }
  real det = (U + V) + W;
  if (det == RC(0.0)) return 0;
  const real Az = s->Sz * A[kz], Bz = s->Sz * B[kz], Cz = s->Sz * C[kz];
  const real D = (U * Az + V * Bz) + W * Cz;
  const real rcp = RC(1.0) / det;
  const real tt = D * rcp;
  if (tt > *t_inout) return 0;
  if (tt < s->t_min) return 0;
  *t_inout = tt;
  s->u = V * rcp;
  s->v = W * rcp;
  return 1;
}

#define ORC_STACK 512

/* returns 1 on hit (hit written), 0 on miss (hit untouched) */
int orc_traverse_one(const orc_node *nodes, const uint32_t *indices, const real *verts,
                     size_t stride, const uint32_t *faces, const orc_ray *ray,
                     const orc_trace_options *topt, int cpp11, orc_hit *hit, orc_counters *ctr) {
  orc_mesh m = {(const unsigned char *)verts, stride, faces, NULL};
  orc_trace_options dflt;
  if (!topt) {
    orc_default_trace_options(&dflt);
    topt = &dflt;
  }
  ray_state s;
  real hit_t = ray->max_t;
  s.t = hit_t;
  s.prim = 0xFFFFFFFFu;
  orc_prepare(&s, ray, topt, cpp11);

  uint32_t stack[ORC_STACK];
  int sp = 0;
  stack[0] = 0;
  while (sp >= 0) {
    const orc_node *nd = &nodes[stack[sp]];
    sp--;
    if (ctr) ctr->nodes_popped++;
    if (!orc_slab(&s, nd, ray->min_t, hit_t)) continue;
    if (nd->flag == 0) {
      int nearc = s.sign[nd->axis];
      stack[++sp] = nd->data[1 - nearc];
      stack[++sp] = nd->data[nearc];
      if (ctr && (uint32_t)sp > ctr->max_stack) ctr->max_stack = (uint32_t)sp;
    } else {
      real t = s.t;
      int any = 0;
      for (uint32_t i = 0; i < nd->data[0]; i++) {
        uint32_t prim = indices[nd->data[1] + i];
        real lt = t;
        if (ctr) ctr->prims_tested++;
        if (orc_tri(&s, &m, prim, &lt)) {
          t = lt;
          s.t = t;
          s.prim = prim;
          any = 1;
        }
      }
      if (any) hit_t = s.t;
    }
  }
  int is_hit = s.t < ray->max_t;
  if (is_hit && hit) {
    hit->t = s.t;
    hit->u = s.u;
    hit->v = s.v;
    hit->prim_id = s.prim;
  }
  return is_hit;
}

typedef struct {
  const orc_node *nodes;
  const uint32_t *indices;
  const real *verts;
  size_t stride;
  const uint32_t *faces;
  const orc_ray *rays;
  size_t n_rays;
  orc_hit *hits;
  uint8_t *mask;
  const orc_trace_options *topt;
  int cpp11;
  int want_counters;
  size_t *next; /* shared chunk cursor */
  pthread_mutex_t *mu;
  size_t n_hits;
  orc_counters ctr;
} batch_job;

static void *batch_worker(void *arg) {
  batch_job *j = (batch_job *)arg;
  const size_t chunk = 1024;
  for (;;) {
    pthread_mutex_lock(j->mu);
    size_t b = *j->next;
    *j->next = b + chunk;
    pthread_mutex_unlock(j->mu);
    if (b >= j->n_rays) break;
    size_t e = b + chunk < j->n_rays ? b + chunk : j->n_rays;
    for (size_t i = b; i < e; i++) {
      int h = orc_traverse_one(j->nodes, j->indices, j->verts, j->stride, j->faces, &j->rays[i],
                               j->topt, j->cpp11, &j->hits[i], j->want_counters ? &j->ctr : NULL);
      if (j->mask) j->mask[i] = (uint8_t)h;
      j->n_hits += (size_t)h;
    }
  }
  return NULL;
}

/* hits[i] is written only where mask[i] == 1 (reference semantics, nanort.h:1205-1213) */
size_t orc_traverse_batch(const orc_node *nodes, const uint32_t *indices, const real *verts,
                          size_t stride, const uint32_t *faces, const orc_ray *rays, size_t n_rays,
                          orc_hit *hits, uint8_t *mask, const orc_trace_options *topt, int cpp11,
                          int n_threads, orc_counters *ctr_out) {
  if (n_threads < 1) n_threads = 1;
  if (n_threads > 256) n_threads = 256;
  size_t next = 0;
  pthread_mutex_t mu;
  pthread_mutex_init(&mu, NULL);
  batch_job *jobs = (batch_job *)calloc((size_t)n_threads, sizeof(batch_job));
  pthread_t *th = (pthread_t *)calloc((size_t)n_threads, sizeof(pthread_t));
  for (int t = 0; t < n_threads; t++) {
    batch_job *j = &jobs[t];
    j->nodes = nodes;
    j->indices = indices;
    j->verts = verts;
    j->stride = stride;
    j->faces = faces;
    j->rays = rays;
    j->n_rays = n_rays;
    j->hits = hits;
    j->mask = mask;
    j->topt = topt;
    j->cpp11 = cpp11;
    j->want_counters = ctr_out != NULL;
    j->next = &next;
    j->mu = &mu;
  }
  if (n_threads == 1) {
    batch_worker(&jobs[0]);
  } else {
    for (int t = 0; t < n_threads; t++) pthread_create(&th[t], NULL, batch_worker, &jobs[t]);
    for (int t = 0; t < n_threads; t++) pthread_join(th[t], NULL);
  }
  size_t total = 0;
  orc_counters c = {0, 0, 0};
  for (int t = 0; t < n_threads; t++) {
    total += jobs[t].n_hits;
    c.nodes_popped += jobs[t].ctr.nodes_popped;
    c.prims_tested += jobs[t].ctr.prims_tested;
    if (jobs[t].ctr.max_stack > c.max_stack) c.max_stack = jobs[t].ctr.max_stack;
  }
  if (ctr_out) *ctr_out = c;
  free(jobs);
  free(th);
  pthread_mutex_destroy(&mu);
  return total;
}

/* Re-tests ONE primitive for ONE ray with the reference arithmetic; used by the
 * parity checker to classify exact-t ties (SURVEY.md F3): returns 1 and the
 * (t,u,v) this primitive alone would report with t_inout = max_t. */
int orc_test_prim(const real *verts, size_t stride, const uint32_t *faces, const orc_ray *ray,
                  const orc_trace_options *topt, int cpp11, uint32_t prim, orc_hit *out) {
  orc_mesh m = {(const unsigned char *)verts, stride, faces, NULL};
  orc_trace_options dflt;
  if (!topt) {
    orc_default_trace_options(&dflt);
    topt = &dflt;
  }
  ray_state s;
  orc_prepare(&s, ray, topt, cpp11);
  real t = ray->max_t;
  if (!orc_tri(&s, &m, prim, &t)) return 0;
  out->t = t;
  out->u = s.u;
  out->v = s.v;
  out->prim_id = prim;
  return 1;
}

#ifndef ORC_DOUBLE /* the scene-graph example is float only (nanosg::Scene<float, M> in the reference's renderer) */
/* ====================================================================== two-level scene
 * Restatement of the reference's scene-graph example (examples/nanosg/nanosg.h) for the instancing row:
 *   orc_mat_inverse            Matrix::Inverse (Cramer's rule)          nanosg.h:92-184
 *   orc_mat_mult / orc_multv   Matrix::Mult / Matrix::MultV             nanosg.h:203-222
 *   orc_xform_bbox             XformBoundingBox                         nanosg.h:241-299
 *   orc_sg_node_update         Node::Update                             nanosg.h:400-445
 *   orc_build_boxes            Scene::Commit top-level Build            nanosg.h:722-737
 *   orc_sg_list                BVHAccel::ListNodeIntersections + TestLeafNodeIntersections with
 *                              NodeBBoxIntersector                      nanort.h:2558-2692, nanosg.h:592-660
 *   orc_sg_traverse_one        Scene::Traverse                          nanosg.h:779-875
 *   orc_sg_instance_hit        its per-instance body                    nanosg.h:831-850
 *   orc_sg_prim_hit            the same body on one triangle (tie re-tests, no reference counterpart)
 * Parity status: PINNED against oracle/_ref/libnanosg_ref*.so (tests/test_oracle_scene.py).
 *
 * Reference behaviours restated as they are (none is "fixed" here):
 *   S1  Matrix::Inverse's last cofactor reads tsrc[0] where Cramer's rule has tsrc[10] (nanosg.h:173);
 *       only m[3][3] is affected and MultV never reads it.
 *   S2  Scene::Traverse builds trace_options.cull_back_face but calls the instance's Traverse with the
 *       default options (nanosg.h:800-829): the flag has no effect.
 *   S3  at most kMaxIntersections = 64 instance boxes (the nearest by box entry t) are considered per ray.
 *   S4  the local ray is {min_t 0, max_t FLT_MAX}: the caller's min_t / max_t only gate the top-level walk.
 */
typedef struct {
  float xform[4][4];   /* parent x local; parent is the identity for scene roots */
  float inv[4][4];     /* world -> local */
  float inv33[4][4];   /* same with the translation cleared first (directions) */
  float invT33[4][4];  /* transpose of inv33 (normals) */
  float lbmin[3], lbmax[3];
  float xbmin[3], xbmax[3];
} orc_sg_node; /* 76 floats */

typedef struct {
  const orc_node *nodes;
  const uint32_t *indices;
  const float *verts;
  size_t stride;
  const uint32_t *faces;
} orc_sg_blas;

typedef struct {
  float u, v, t;
  uint32_t prim_id, node_id;
  float P[3];
} orc_sg_hit; /* 32 B */

/* pairs / cofactor tables of the Cramer's-rule inverse: every cofactor is
 * (p0*s0 + p1*s1 + p2*s2) - (q0*s0' + q1*s1' + q2*s2') with p/q from the pair table */
static const uint8_t kPairs[2][12][2] = {
    {{10, 15}, {11, 14}, {9, 15}, {11, 13}, {9, 14}, {10, 13}, {8, 15}, {11, 12}, {8, 14}, {10, 12}, {8, 13}, {9, 12}},
    {{2, 7}, {3, 6}, {1, 7}, {3, 5}, {1, 6}, {2, 5}, {0, 7}, {3, 4}, {0, 6}, {2, 4}, {0, 5}, {1, 4}}};
/* [element][plus/minus][term] = {pair index, source index} */
static const uint8_t kCof[16][2][3][2] = {
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
    {{{10, 10}, {4, 8}, {9, 9}}, {{8, 9}, {11, 0} /* S1 */, {5, 8}}}};

void orc_mat_inverse(float m[4][4]) {
  float src[16], pr[12], out[16];
  for (int i = 0; i < 4; i++)
    for (int c = 0; c < 4; c++) src[i + 4 * c] = m[i][c];
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
  for (int e = 0; e < 16; e++) m[e / 4][e % 4] = out[e] * det;
}

static void orc_mat_mult(float dst[4][4], const float m0[4][4], const float m1[4][4]) {
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) {
      float acc = 0.0f;
      for (int k = 0; k < 4; k++) acc += m0[k][j] * m1[i][k];
      dst[i][j] = acc;
    }
}

static void orc_multv(float dst[3], const float m[4][4], const float v[3]) {
  float t[3];
  for (int k = 0; k < 3; k++) t[k] = ((m[0][k] * v[0] + m[1][k] * v[1]) + m[2][k] * v[2]) + m[3][k];
  dst[0] = t[0];
  dst[1] = t[1];
  dst[2] = t[2];
}

static void orc_xform_bbox(float xbmin[3], float xbmax[3], const float bmin[3], const float bmax[3],
                           const float m[4][4]) {
  for (int i = 0; i < 8; i++) {
    float c[3] = {(i & 1) ? bmax[0] : bmin[0], (i & 2) ? bmax[1] : bmin[1], (i & 4) ? bmax[2] : bmin[2]};
    float x[3];
    orc_multv(x, m, c);
    for (int k = 0; k < 3; k++) {
      if (i == 0) {
        xbmin[k] = xbmax[k] = x[k];
      } else {
        xbmin[k] = stdmin(x[k], xbmin[k]);
        xbmax[k] = stdmax(x[k], xbmax[k]);
      }
    }
  }
}

/* Node::Update for a scene root: parent transform = identity */
void orc_sg_node_update(orc_sg_node *nd, const float local_xform[16], const float lbmin[3], const float lbmax[3]) {
  float ident[4][4], local[4][4];
  memset(ident, 0, sizeof(ident));
  for (int i = 0; i < 4; i++) ident[i][i] = 1.0f;
  memcpy(local, local_xform, sizeof(local));
  for (int k = 0; k < 3; k++) {
    nd->lbmin[k] = lbmin[k];
    nd->lbmax[k] = lbmax[k];
  }
  orc_mat_mult(nd->xform, ident, local);
  orc_xform_bbox(nd->xbmin, nd->xbmax, nd->lbmin, nd->lbmax, nd->xform);
  memcpy(nd->inv, nd->xform, sizeof(nd->inv));
  orc_mat_inverse(nd->inv);
  memcpy(nd->inv33, nd->xform, sizeof(nd->inv33));
  nd->inv33[3][0] = nd->inv33[3][1] = nd->inv33[3][2] = 0.0f;
  orc_mat_inverse(nd->inv33);
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) nd->invT33[j][i] = nd->inv33[i][j];
}

/* ---- std::priority_queue<NodeHit, vector, NodeHitComparator> as libstdc++ implements it
 * (bits/stl_heap.h __push_heap / __adjust_heap); comp(a, b) = a.t_min < b.t_min, so the top is the
 * farthest entry.  The order among equal t_min follows from these exact sift rules. */
typedef struct {
  float t_min, t_max;
  uint32_t id;
} sg_nodehit;

static void heap_sift_up(sg_nodehit *h, int hole, int top, sg_nodehit v) {
  int parent = (hole - 1) / 2;
  while (hole > top && h[parent].t_min < v.t_min) {
    h[hole] = h[parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  h[hole] = v;
}

static void heap_push(sg_nodehit *h, int *n, sg_nodehit v) {
  (*n)++;
  heap_sift_up(h, *n - 1, 0, v);
}

static void heap_pop(sg_nodehit *h, int *n) { /* moves the top to h[*n - 1] and shrinks */
  int len = *n - 1;
  sg_nodehit v = h[len];
  h[len] = h[0];
  int hole = 0, child = 0;
  while (child < (len - 1) / 2) {
    child = 2 * (child + 1);
    if (h[child].t_min < h[child - 1].t_min) child--;
    h[hole] = h[child];
    hole = child;
  }
  if ((len & 1) == 0 && child == (len - 2) / 2) {
    child = 2 * (child + 1);
    h[hole] = h[child - 1];
    hole = child - 1;
  }
  heap_sift_up(h, hole, 0, v);
  *n = len;
}

/* first stage of Scene::Traverse: the (at most max_hits <= 128) nearest instance boxes, nearest first */
int orc_sg_list(const orc_node *top, const uint32_t *top_idx, const orc_sg_node *sg, const orc_ray *ray,
                int max_hits, int cpp11, float *tmin_out, float *tmax_out, uint32_t *ids_out) {
  ray_state s;
  for (int k = 0; k < 3; k++) {
    s.org[k] = ray->org[k];
    s.sign[k] = ray->dir[k] < 0.0f ? 1 : 0;
    s.inv[k] = orc_safe_inverse(ray->dir[k], cpp11);
  }
  /* NodeBBoxIntersector::PrepareTraversal: plain reciprocal, no zero guard (nanosg.h:645-647) */
  const float rinv[3] = {1.0f / ray->dir[0], 1.0f / ray->dir[1], 1.0f / ray->dir[2]};
  sg_nodehit heap[129];
  int nh = 0;
  uint32_t stack[ORC_STACK];
  int sp = 0;
  stack[0] = 0;
  while (sp >= 0) {
    const orc_node *nd = &top[stack[sp]];
    sp--;
    if (!orc_slab(&s, nd, ray->min_t, ray->max_t)) continue; /* hit_t never shrinks here */
    if (nd->flag == 0) {
      int nearc = s.sign[nd->axis];
      stack[++sp] = nd->data[1 - nearc];
      stack[++sp] = nd->data[nearc];
      continue;
    }
    for (uint32_t i = 0; i < nd->data[0]; i++) {
      const uint32_t id = top_idx[nd->data[1] + i];
      const orc_sg_node *b = &sg[id];
      float tn[3], tf[3];
      for (int k = 0; k < 3; k++) {
        const float lo = s.sign[k] ? b->xbmax[k] : b->xbmin[k];
        const float hi = s.sign[k] ? b->xbmin[k] : b->xbmax[k];
        tn[k] = (lo - ray->org[k]) * rinv[k];
        tf[k] = (hi - ray->org[k]) * rinv[k];
      }
      const float tmin = smax(tn[2], smax(tn[1], tn[0]));
      const float tmax = smin(tf[2], smin(tf[1], tf[0]));
      if (!(tmin <= tmax)) continue;
      sg_nodehit v = {tmin, tmax, id};
      if (nh < max_hits) {
        heap_push(heap, &nh, v);
      } else if (tmin < heap[0].t_min) {
        heap_pop(heap, &nh);
        heap_push(heap, &nh, v);
      }
    }
  }
  const int n = nh;
  for (int i = 0; i < n; i++) { /* pop farthest first, store back to front */
    const sg_nodehit topv = heap[0];
    heap_pop(heap, &nh);
    tmin_out[n - i - 1] = topv.t_min;
    if (tmax_out) tmax_out[n - i - 1] = topv.t_max;
    ids_out[n - i - 1] = topv.id;
  }
  return n;
}

/* One instance of Scene::Traverse (nanosg.h:831-850): the world ray moved into instance `id` (MultV with inv and
 * inv33), the local ray {0, FLT_MAX} walked through the instance's tree -- or, for prim != 0xFFFFFFFF, tested against
 * that one triangle alone -- then the local hit point moved back to world space and its distance from the world
 * origin.  Returns 1 and the whole record on a hit. */
static int sg_local_hit(const orc_sg_node *sg, const orc_sg_blas *blas, const orc_ray *ray, uint32_t id, uint32_t prim,
                        int cpp11, orc_sg_hit *hit) {
  const orc_sg_node *nd = &sg[id];
  const orc_sg_blas *b = &blas[id];
  orc_ray lr;
  orc_multv(lr.org, nd->inv, ray->org);
  orc_multv(lr.dir, nd->inv33, ray->dir);
  lr.min_t = 0.0f;
  lr.max_t = FLT_MAX;
  lr.type = 0;
  orc_hit lh;
  if (prim == 0xFFFFFFFFu) {
    if (!orc_traverse_one(b->nodes, b->indices, b->verts, b->stride, b->faces, &lr, NULL, cpp11, &lh, NULL)) return 0;
  } else if (!orc_test_prim(b->verts, b->stride, b->faces, &lr, NULL, cpp11, prim, &lh)) {
    return 0;
  }
  float lp[3], wp[3];
  for (int k = 0; k < 3; k++) lp[k] = lr.org[k] + lh.t * lr.dir[k];
  orc_multv(wp, nd->xform, lp);
  const float px = wp[0] - ray->org[0], py = wp[1] - ray->org[1], pz = wp[2] - ray->org[2];
  hit->u = lh.u;
  hit->v = lh.v;
  hit->t = sqrtf((px * px + py * py) + pz * pz);
  hit->prim_id = lh.prim_id;
  hit->node_id = id;
  hit->P[0] = wp[0];
  hit->P[1] = wp[1];
  hit->P[2] = wp[2];
  return 1;
}

/* the nearest hit inside instance `id` alone, as Scene::Traverse records it */
int orc_sg_instance_hit(const orc_sg_node *sg, const orc_sg_blas *blas, const orc_ray *ray, uint32_t id, int cpp11,
                        orc_sg_hit *hit) {
  return sg_local_hit(sg, blas, ray, id, 0xFFFFFFFFu, cpp11, hit);
}

/* the record Scene::Traverse would write if triangle `prim` of instance `id` were its pick (tie re-tests) */
int orc_sg_prim_hit(const orc_sg_node *sg, const orc_sg_blas *blas, const orc_ray *ray, uint32_t id, uint32_t prim,
                    int cpp11, orc_sg_hit *hit) {
  return sg_local_hit(sg, blas, ray, id, prim, cpp11, hit);
}

/* orc_sg_instance_hit (prims == NULL) or orc_sg_prim_hit for rays[i] and ids[i] / prims[i]; ok[i] = hit */
void orc_sg_local_hit_batch(const orc_sg_node *sg, const orc_sg_blas *blas, const orc_ray *rays, size_t n,
                            const uint32_t *ids, const uint32_t *prims, int cpp11, orc_sg_hit *hits, uint8_t *ok) {
  for (size_t i = 0; i < n; i++)
    ok[i] = (uint8_t)sg_local_hit(sg, blas, &rays[i], ids[i], prims ? prims[i] : 0xFFFFFFFFu, cpp11, &hits[i]);
}

/* Scene::Traverse with the node-hit list cut at max_hits boxes (the reference's kMaxIntersections = 64; at most 128) */
int orc_sg_traverse_one(const orc_node *top, const uint32_t *top_idx, const orc_sg_node *sg,
                        const orc_sg_blas *blas, const orc_ray *ray, int max_hits, int cpp11, orc_sg_hit *hit) {
  float tmin[128];
  uint32_t ids[128];
  if (max_hits < 1) max_hits = 1;
  if (max_hits > 128) max_hits = 128;
  const int n = orc_sg_list(top, top_idx, sg, ray, max_hits, cpp11, tmin, NULL, ids);
  float t_nearest = FLT_MAX;
  int has_hit = 0;
  for (int i = 0; i < n; i++) {
    if (t_nearest < tmin[i]) continue;
    orc_sg_hit h;
    if (!sg_local_hit(sg, blas, ray, ids[i], 0xFFFFFFFFu, cpp11, &h)) continue;
    if (h.t < t_nearest) {
      t_nearest = h.t;
      has_hit = 1;
      *hit = h;
    }
  }
  return has_hit;
}

typedef struct {
  const orc_node *top;
  const uint32_t *top_idx;
  const orc_sg_node *sg;
  const orc_sg_blas *blas;
  const orc_ray *rays;
  size_t n_rays;
  orc_sg_hit *hits;
  uint8_t *mask;
  int max_hits;
  int cpp11;
  size_t *next;
  pthread_mutex_t *mu;
  size_t n_hits;
} sg_job;

static void *sg_worker(void *arg) {
  sg_job *j = (sg_job *)arg;
  for (;;) {
    pthread_mutex_lock(j->mu);
    size_t b = *j->next;
    *j->next = b + 256;
    pthread_mutex_unlock(j->mu);
    if (b >= j->n_rays) break;
    size_t e = b + 256 < j->n_rays ? b + 256 : j->n_rays;
    for (size_t i = b; i < e; i++) {
      orc_sg_hit h;
      int hit = orc_sg_traverse_one(j->top, j->top_idx, j->sg, j->blas, &j->rays[i], j->max_hits, j->cpp11, &h);
      if (hit) {
        j->hits[i] = h;
        j->n_hits++;
      }
      if (j->mask) j->mask[i] = (uint8_t)hit;
    }
  }
  return NULL;
}

/* Scene::Traverse over a batch; hits[i] is written only where mask[i] == 1 */
size_t orc_sg_traverse_batch(const orc_node *top, const uint32_t *top_idx, const orc_sg_node *sg,
                             const orc_sg_blas *blas, const orc_ray *rays, size_t n_rays, orc_sg_hit *hits,
                             uint8_t *mask, int max_hits, int cpp11, int n_threads) {
  if (n_threads < 1) n_threads = 1;
  if (n_threads > 256) n_threads = 256;
  pthread_mutex_t mu = PTHREAD_MUTEX_INITIALIZER;
  size_t next = 0, total = 0;
  sg_job jobs[256];
  pthread_t th[256];
  for (int t = 0; t < n_threads; t++) {
    sg_job j = {top, top_idx, sg, blas, rays, n_rays, hits, mask, max_hits, cpp11, &next, &mu, 0};
    jobs[t] = j;
  }
  if (n_threads == 1) {
    sg_worker(&jobs[0]);
  } else {
    for (int t = 0; t < n_threads; t++) pthread_create(&th[t], NULL, sg_worker, &jobs[t]);
    for (int t = 0; t < n_threads; t++) pthread_join(th[t], NULL);
  }
  for (int t = 0; t < n_threads; t++) total += jobs[t].n_hits;
  return total;
}
#endif /* !ORC_DOUBLE */
