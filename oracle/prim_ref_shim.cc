// TEST INFRASTRUCTURE ONLY -- the reference's own custom-primitive model behind a C interface.
//
// Compiles the UNMODIFIED $(NANORT_REF)/examples/particle_primitive/main.cc (its main() renamed away; nothing of it is
// copied into the repository) together with the unmodified nanort.h, and drives the example's SphereGeometry, SpherePred
// and SphereIntersector<SphereIntersection> (main.cc:80-291) through BVHAccel<float>::Build / Traverse exactly as the
// example's main() does (main.cc:338-401).  This is the oracle of the NRT_PRIM_SPHERES kind (csrc/prims.cu).
//
// Built twice by oracle/Makefile: _ref/libprim_ref.so with NANORT_USE_CPP11_FEATURE (copysign vsafe_inverse) and
// _ref/libprim_ref03.so without it (the C++03 vsafe_inverse, -0.0f -> +inf), the two conventions of
// NRT_TRAVERSE_CPP03_INVERSE.  refsph_adopt loads any (nodes, indices) pair -- the device's tree -- through the
// reference's own Load (nanort.h:2222-2275), so that its Traverse and SphereIntersector walk that tree.
#include <stdint.h>
#include <string.h>

#include <thread>
#include <vector>

#define NANORT_ENABLE_SERIALIZATION
#define main nanort_reference_particle_primitive_main
#include "main.cc"  // found through -I$(NANORT_REF)/examples/particle_primitive (oracle/Makefile)
#undef main

struct RefSpheres {
  std::vector<float> centers, radii;
  nanort::BVHAccel<float> accel;
};

namespace {

nanort::BVHTraceOptions trace_opts(const void *topts16) {
  nanort::BVHTraceOptions o;
  static_assert(sizeof(nanort::BVHTraceOptions) == 16, "BVHTraceOptions is 16 bytes");
  if (topts16) memcpy(&o, topts16, sizeof(o));
  return o;
}

RefSpheres *new_spheres(const float *centers, const float *radii, size_t n) {
  RefSpheres *s = new RefSpheres();
  s->centers.assign(centers, centers + 3 * n);
  s->radii.assign(radii, radii + n);
  return s;
}

}  // namespace

extern "C" {

// 1 when built with NANORT_USE_CPP11_FEATURE (copysign vsafe_inverse), 0 for the C++03 one
int refsph_mode_cpp11(void) {
#ifdef NANORT_USE_CPP11_FEATURE
  return 1;
#else
  return 0;
#endif
}

// build_opts28 == NULL: the default options, as the example
void *refsph_build_opts(const float *centers, const float *radii, size_t n, const void *build_opts28) {
  RefSpheres *s = new_spheres(centers, radii, n);
  nanort::BVHBuildOptions<float> options;
  static_assert(sizeof(options) == 28, "BVHBuildOptions<float> is 28 bytes");
  if (build_opts28) memcpy(&options, build_opts28, sizeof(options));
  SphereGeometry sphere_geom(&s->centers.at(0), &s->radii.at(0));
  SpherePred sphere_pred(&s->centers.at(0));
  if (!s->accel.Build(static_cast<unsigned int>(n), sphere_geom, sphere_pred, options)) {
    delete s;
    return NULL;
  }
  return s;
}

// the default options (the entry point of the first version of this shim, kept with its signature)
void *refsph_build(const float *centers, const float *radii, size_t n) { return refsph_build_opts(centers, radii, n, NULL); }

// An arbitrary (nodes, indices) pair -- e.g. the device's tree -- loaded through the reference's own Dump format:
// size_t n; nodes; size_t m; indices.
void *refsph_adopt(const void *nodes40, size_t n_nodes, const uint32_t *indices, size_t n_indices, const float *centers,
                   const float *radii, size_t n) {
  size_t bytes = 2 * sizeof(size_t) + n_nodes * sizeof(nanort::BVHNode<float>) + n_indices * sizeof(uint32_t);
  std::vector<unsigned char> buf(bytes);
  unsigned char *p = buf.data();
  memcpy(p, &n_nodes, sizeof(size_t));
  p += sizeof(size_t);
  memcpy(p, nodes40, n_nodes * sizeof(nanort::BVHNode<float>));
  p += n_nodes * sizeof(nanort::BVHNode<float>);
  memcpy(p, &n_indices, sizeof(size_t));
  p += sizeof(size_t);
  memcpy(p, indices, n_indices * sizeof(uint32_t));
  FILE *fp = fmemopen(buf.data(), bytes, "rb");
  if (!fp) return NULL;
  RefSpheres *s = new_spheres(centers, radii, n);
  const bool ok = s->accel.Load(fp);
  fclose(fp);
  if (!ok) {
    delete s;
    return NULL;
  }
  return s;
}

void refsph_free(void *h) { delete static_cast<RefSpheres *>(h); }

void refsph_bounding_box(const void *h, float bmin[3], float bmax[3]) {
  static_cast<const RefSpheres *>(h)->accel.BoundingBox(bmin, bmax);
}

size_t refsph_num_nodes(const void *h) { return static_cast<const RefSpheres *>(h)->accel.GetNodes().size(); }
size_t refsph_num_indices(const void *h) { return static_cast<const RefSpheres *>(h)->accel.GetIndices().size(); }
void refsph_copy_nodes(const void *h, void *out40) {
  const std::vector<nanort::BVHNode<float> > &v = static_cast<const RefSpheres *>(h)->accel.GetNodes();
  memcpy(out40, v.data(), v.size() * sizeof(nanort::BVHNode<float>));
}
void refsph_copy_indices(const void *h, uint32_t *out) {
  const std::vector<unsigned int> &v = static_cast<const RefSpheres *>(h)->accel.GetIndices();
  memcpy(out, v.data(), v.size() * sizeof(uint32_t));
}

// hits: {u, v, t, prim_id} per ray, untouched (zeroed by the caller) on a miss; trace_opts16 == NULL: the defaults
void refsph_traverse_opts(const void *h, const void *rays36, size_t n_rays, void *hits16, uint8_t *mask,
                          const void *trace_opts16, int threads) {
  const RefSpheres *s = static_cast<const RefSpheres *>(h);
  const nanort::Ray<float> *rays = static_cast<const nanort::Ray<float> *>(rays36);
  SphereIntersection *out = static_cast<SphereIntersection *>(hits16);
  static_assert(sizeof(SphereIntersection) == 16, "SphereIntersection is {u, v, t, prim_id}");
  const nanort::BVHTraceOptions opt = trace_opts(trace_opts16);
  if (threads < 1) threads = 1;
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; t++) {
    pool.emplace_back([=]() {
      for (size_t i = (size_t)t; i < n_rays; i += (size_t)threads) {
        SphereIntersector<SphereIntersection> isecter(&s->centers.at(0), &s->radii.at(0));
        SphereIntersection isect;
        memset(&isect, 0, sizeof(isect));
        const bool hit = s->accel.Traverse(rays[i], isecter, &isect, opt);
        mask[i] = hit ? 1 : 0;
        if (hit) out[i] = isect;
      }
    });
  }
  for (auto &th : pool) th.join();
}

// the default trace options with prim_ids_range = [prim_lo, prim_hi) (the first version's entry point and signature)
void refsph_traverse(const void *h, const void *rays36, size_t n_rays, void *hits16, uint8_t *mask, uint32_t prim_lo,
                     uint32_t prim_hi, int threads) {
  nanort::BVHTraceOptions opt;
  opt.prim_ids_range[0] = prim_lo;
  opt.prim_ids_range[1] = prim_hi;
  refsph_traverse_opts(h, rays36, n_rays, hits16, mask, &opt, threads);
}

// Per ray i: one SphereIntersector::Intersect(&t, prims[i]) after PrepareTraversal, starting from t = t_inout[i] (NULL:
// ray.max_t), then Update + PostTraversal(hit = true) -- the reference's full record {u, v, t, prim} had Traverse picked
// prims[i].  ok[i] = Intersect's return value; out[i] is written only where it is 1.
void refsph_test_prims(const void *h, const void *rays36, size_t n_rays, const uint32_t *prims, const float *t_inout,
                       const void *trace_opts16, void *hits16, uint8_t *ok) {
  const RefSpheres *s = static_cast<const RefSpheres *>(h);
  const nanort::Ray<float> *rays = static_cast<const nanort::Ray<float> *>(rays36);
  SphereIntersection *out = static_cast<SphereIntersection *>(hits16);
  const nanort::BVHTraceOptions opt = trace_opts(trace_opts16);
  for (size_t i = 0; i < n_rays; i++) {
    SphereIntersector<SphereIntersection> isecter(&s->centers.at(0), &s->radii.at(0));
    isecter.Update(rays[i].max_t, static_cast<unsigned int>(-1));
    isecter.PrepareTraversal(rays[i], opt);
    float t = t_inout ? t_inout[i] : rays[i].max_t;
    ok[i] = 0;
    if (prims[i] >= s->radii.size() || !isecter.Intersect(&t, prims[i])) continue;
    isecter.Update(t, prims[i]);
    SphereIntersection isect;
    memset(&isect, 0, sizeof(isect));
    isecter.PostTraversal(rays[i], true, &isect);
    out[i] = isect;
    ok[i] = 1;
  }
}

// Per ray: 1 when SphereIntersector::Intersect (t_inout = ray.max_t) yields a NaN t for some sphere of the scene inside
// the trace options' id range.  Such a t is accepted (`t > t_inout` is false) and replaced by the next accepted hit, so
// the reference's own answer then depends on its visiting order.  Brute force: small scenes only.
void refsph_nan_rays(const void *h, const void *rays36, size_t n_rays, const void *trace_opts16, uint8_t *out,
                     int threads) {
  const RefSpheres *s = static_cast<const RefSpheres *>(h);
  const nanort::Ray<float> *rays = static_cast<const nanort::Ray<float> *>(rays36);
  const nanort::BVHTraceOptions opt = trace_opts(trace_opts16);
  if (threads < 1) threads = 1;
  std::vector<std::thread> pool;
  for (int th = 0; th < threads; th++) {
    pool.emplace_back([=]() {
      for (size_t i = (size_t)th; i < n_rays; i += (size_t)threads) {
        SphereIntersector<SphereIntersection> isecter(&s->centers.at(0), &s->radii.at(0));
        isecter.PrepareTraversal(rays[i], opt);
        out[i] = 0;
        for (unsigned int p = 0; p < s->radii.size() && !out[i]; p++) {
          float t = rays[i].max_t;
          if (isecter.Intersect(&t, p) && t != t) out[i] = 1;
        }
      }
    });
  }
  for (auto &t : pool) t.join();
}

// 1 when the box of node `node` passes the reference's slab test IntersectRayAABB over the ray's [min_t, max_t] with the
// reference's own vsafe_inverse and direction signs (nanort.h:2505-2533); -1 when there is no such node.
int refsph_node_box_hit(const void *h, const void *ray36, size_t node) {
  const RefSpheres *s = static_cast<const RefSpheres *>(h);
  const nanort::Ray<float> &ray = *static_cast<const nanort::Ray<float> *>(ray36);
  const std::vector<nanort::BVHNode<float> > &nodes = s->accel.GetNodes();
  if (node >= nodes.size()) return -1;
  int dir_sign[3];
  nanort::real3<float> dir, org;
  for (int k = 0; k < 3; k++) {
    dir_sign[k] = ray.dir[k] < 0.0f ? 1 : 0;
    dir[k] = ray.dir[k];
    org[k] = ray.org[k];
  }
  const nanort::real3<float> inv = nanort::vsafe_inverse(dir);
  float tmin, tmax;
  return nanort::IntersectRayAABB(&tmin, &tmax, ray.min_t, ray.max_t, nodes[node].bmin, nodes[node].bmax, org, inv,
                                  dir_sign)
             ? 1
             : 0;
}

}  // extern "C"
