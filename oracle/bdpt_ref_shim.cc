// TEST INFRASTRUCTURE ONLY -- the reference bidirectional path tracer's own code behind a C interface.
//
// Compiles the UNMODIFIED $(NANORT_REF)/examples/bidir_path_tracer/main.cc into this translation unit (its main() is
// renamed away; nothing of it is copied into the repository), so that tests/test_gpu_bdpt.py checks the device pass
// against the reference's OWN functions:
//     Random (xorshift128)                          main.cc:132-157
//     LightSampler (constructor + sample)           main.cc:692-774
//     raytrace, eyeSubpath, lightSubpath            main.cc:898-1079
//     weightMIS, calcG, connectPath                 main.cc:1081-1289
// over the reference's own BVHAccel<float>, built as main() builds it (cache_bbox = false, main.cc:1333-1353).
//
// Built with -ftrivial-auto-var-init=zero (oracle/bdpt.mk): lightSubpath's `Vertex vertex;` leaves the light-origin
// vertex's material uninitialised and weightMIS reads its isDelta(); zeroed, that vertex is not delta, which is what
// the device defines.
//
// Vertices are exported in nrt_bdpt_vertex's layout (include/nanort_b200_bdpt.h).  The reference's Vertex keeps its
// material by value and not the face it lies on: the material index is the first material whose 16 floats equal the
// vertex's, and prim_id is recovered by tracing the reference's accel from the previous vertex along -wo (the same
// segment up to the rounding of the normalisation).
#include <stdint.h>
#include <string.h>

#include <vector>

#define main nanort_reference_bidir_main
#include "main.cc"  // found through -I$(NANORT_REF)/examples/bidir_path_tracer (oracle/bdpt.mk)
#undef main

namespace {

struct ExVertex {  // nrt_bdpt_vertex
  float position[3], original_norm[3], norm[3], beta[3], wo[3];
  float pdf_fwd, pdf_rev;
  uint32_t type, material, prim_id;
};
static_assert(sizeof(ExVertex) == 80, "nrt_bdpt_vertex");

struct BdptRefScene {
  Mesh mesh;
  std::vector<tinyobj::material_t> materials;
  Accel accel;
  LightSampler *lights = nullptr;
};

bool same_material(const tinyobj::material_t &a, const tinyobj::material_t &b) {
  for (int k = 0; k < 3; k++) {
    if (a.diffuse[k] != b.diffuse[k] || a.specular[k] != b.specular[k] || a.transmittance[k] != b.transmittance[k] ||
        a.emission[k] != b.emission[k])
      return false;
  }
  return a.ior == b.ior && a.dissolve == b.dissolve;
}

uint32_t material_index(const BdptRefScene &s, const Vertex &v) {
  if (v.type == Lens) return 0xFFFFFFFFu;
  for (size_t i = 0; i < s.materials.size(); i++)
    if (same_material(s.materials[i], v.mat)) return (uint32_t)i;
  return 0xFFFFFFFFu;
}

uint32_t trace_prim(const BdptRefScene &s, const float3 &org, const float3 &dir) {
  nanort::Ray<float> ray;
  for (int k = 0; k < 3; k++) {
    ray.org[k] = org[k];
    ray.dir[k] = dir[k];
  }
  ray.min_t = kEps;
  ray.max_t = kInf;
  nanort::TriangleIntersector<> ti(s.mesh.vertices, s.mesh.faces, sizeof(float) * 3);
  nanort::TriangleIntersection<> isect;
  return s.accel.Traverse(ray, ti, &isect) ? isect.prim_id : 0xFFFFFFFFu;
}

void export_path(const BdptRefScene &s, const std::vector<Vertex> &path, ExVertex *out) {
  for (size_t i = 0; i < path.size(); i++) {
    const Vertex &v = path[i];
    ExVertex &o = out[i];
    for (int k = 0; k < 3; k++) {
      o.position[k] = v.position[k];
      o.original_norm[k] = v.originalNorm[k];
      o.norm[k] = v.norm[k];
      o.beta[k] = v.beta[k];
      o.wo[k] = v.wo[k];
    }
    o.pdf_fwd = v.pdfFwd;
    o.pdf_rev = v.pdfRev;
    o.type = (uint32_t)v.type;
    const bool origin = i == 0;  // the lens vertex / the light-origin vertex
    o.material = origin ? 0xFFFFFFFFu : material_index(s, v);
    o.prim_id = origin ? 0xFFFFFFFFu : trace_prim(s, path[i - 1].position, -v.wo);
  }
}

Vertex import_vertex(const BdptRefScene &s, const ExVertex &e) {
  Vertex v = Vertex();
  for (int k = 0; k < 3; k++) {
    v.position[k] = e.position[k];
    v.originalNorm[k] = e.original_norm[k];
    v.norm[k] = e.norm[k];
    v.beta[k] = e.beta[k];
    v.wo[k] = e.wo[k];
  }
  v.pdfFwd = e.pdf_fwd;
  v.pdfRev = e.pdf_rev;
  v.type = (VertexType)e.type;
  if (e.material != 0xFFFFFFFFu) v.mat = s.materials[e.material];
  return v;
}

}  // namespace

extern "C" {

// The mesh over BORROWED arrays (the caller keeps them alive), the 16-float materials (csrc/wavefront.cuh:
// PathMaterial) as tinyobj::material_t, the reference's own BVH build and LightSampler.  NULL when no face emits
// (max(Le) > kEps): the reference would index cdf_[0] of an empty vector.
void *bdpt_ref_scene(const float *verts, size_t n_verts, const unsigned int *faces, size_t n_faces,
                     const unsigned int *material_ids, const float *facevarying_normals, const float *materials16,
                     size_t n_materials) {
  BdptRefScene *s = new BdptRefScene();
  memset(&s->mesh, 0, sizeof(Mesh));
  s->mesh.num_vertices = n_verts;
  s->mesh.num_faces = n_faces;
  s->mesh.vertices = const_cast<float *>(verts);
  s->mesh.faces = const_cast<unsigned int *>(faces);
  s->mesh.material_ids = const_cast<unsigned int *>(material_ids);
  s->mesh.facevarying_normals = const_cast<float *>(facevarying_normals);
  s->materials.resize(n_materials);
  for (size_t i = 0; i < n_materials; i++) {
    tinyobj::material_t &m = s->materials[i];
    const float *p = materials16 + 16 * i;
    for (int k = 0; k < 3; k++) {
      m.ambient[k] = 0.0f;
      m.diffuse[k] = p[k];
      m.specular[k] = p[3 + k];
      m.transmittance[k] = p[6 + k];
      m.emission[k] = p[9 + k];
    }
    m.shininess = 1.0f;
    m.ior = p[12];
    m.dissolve = p[13];
    m.illum = 0;
    m.dummy = 0;
  }
  size_t n_lights = 0;
  for (size_t i = 0; i < n_faces; i++) {
    const float *le = s->materials[material_ids[i]].emission;
    if (std::max(le[0], std::max(le[1], le[2])) > kEps) n_lights++;
  }
  nanort::BVHBuildOptions<float> build_options;
  build_options.cache_bbox = false;
  nanort::TriangleMesh<float> triangle_mesh(s->mesh.vertices, s->mesh.faces, sizeof(float) * 3);
  nanort::TriangleSAHPred<float> triangle_pred(s->mesh.vertices, s->mesh.faces, sizeof(float) * 3);
  if (n_lights == 0 || !s->accel.Build((unsigned int)n_faces, triangle_mesh, triangle_pred, build_options)) {
    delete s;
    return nullptr;
  }
  s->lights = new LightSampler(s->mesh, s->materials);
  return s;
}

void bdpt_ref_scene_free(void *h) {
  BdptRefScene *s = static_cast<BdptRefScene *>(h);
  if (!s) return;
  delete s->lights;
  delete s;
}

// The body of main()'s sample loop (main.cc:1383-1392) for loop pixel (x, y) and `seed`: both subpaths (each at most
// uMaxBounces + 1 vertices) and connectPath's colour.  A sample whose eye subpath is the lens alone has no light
// subpath and colour 0.
void bdpt_ref_sample(void *h, int x, int y, int width, int height, unsigned int seed, void *eye_out,
                     unsigned int *n_eye, void *light_out, unsigned int *n_light, float *rgb) {
  BdptRefScene *s = static_cast<BdptRefScene *>(h);
  Random rng(seed);
  std::vector<Vertex> eyeVert;
  eyeSubpath(x, y, width, height, s->mesh, s->materials, s->accel, rng, &eyeVert);
  export_path(*s, eyeVert, static_cast<ExVertex *>(eye_out));
  *n_eye = (unsigned int)eyeVert.size();
  rgb[0] = rgb[1] = rgb[2] = 0.0f;
  *n_light = 0;
  if (eyeVert.size() <= 1) return;
  std::vector<Vertex> lightVert;
  lightSubpath(s->mesh, s->materials, s->accel, rng, *s->lights, &lightVert);
  export_path(*s, lightVert, static_cast<ExVertex *>(light_out));
  *n_light = (unsigned int)lightVert.size();
  const float3 c = connectPath(eyeVert, lightVert, s->mesh, s->accel, *s->lights);
  rgb[0] = c[0];
  rgb[1] = c[1];
  rgb[2] = c[2];
}

// connectPath over the caller's vertices (nrt_bdpt_vertex records; mat looked up from the material index, a zeroed
// material for 0xFFFFFFFF), with the reference's accel for calcG
void bdpt_ref_connect(void *h, const void *eye, unsigned int n_eye, const void *light, unsigned int n_light,
                      float *rgb) {
  BdptRefScene *s = static_cast<BdptRefScene *>(h);
  const ExVertex *e = static_cast<const ExVertex *>(eye), *l = static_cast<const ExVertex *>(light);
  std::vector<Vertex> eyeVert, lightVert;
  for (unsigned int i = 0; i < n_eye; i++) eyeVert.push_back(import_vertex(*s, e[i]));
  for (unsigned int i = 0; i < n_light; i++) lightVert.push_back(import_vertex(*s, l[i]));
  const float3 c = connectPath(eyeVert, lightVert, s->mesh, s->accel, *s->lights);
  rgb[0] = c[0];
  rgb[1] = c[1];
  rgb[2] = c[2];
}

// n draws of Random(seed).nextReal()
void bdpt_ref_random(unsigned int seed, size_t n, float *out) {
  Random rng(seed);
  for (size_t i = 0; i < n; i++) out[i] = rng.nextReal();
}

}  // extern "C"
