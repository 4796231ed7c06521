// Device-side pieces of the two-level scene shared by scene.cu's passes, bdpt.cu's scene pass and scene_bake.cu's
// bakes: the instance record, the scene walk's hit record, Matrix::MultV, world-space triangles, normals and light
// records, the rule that lifts spawned rays off a surface, and the host entry points the other files walk the scene
// and run the path pass's stages through.
#pragma once

#include "../../include/nanort_b200_scene_path.h"
#include "common.cuh"

namespace nrt {

// the scene walk's hit record and one instance's shading inputs (named outside the anonymous namespace below, so
// that ScenePathCall can hold them typed)
struct SceneHit32 {
  float u, v, t;
  uint32_t prim_id, node_id;
  float P[3];
};
static_assert(sizeof(SceneHit32) == 32, "nrt_scene_hit");

struct SceneShadingDev {  // nrt_scene_shading
  const uint32_t *mat_ids;
  const float *fvn;
};
static_assert(sizeof(SceneShadingDev) == sizeof(nrt_scene_shading), "nrt_scene_shading");

namespace {

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

// Spawned rays start lift = ray_min_t above P along the unit geometric normal g, on the side the ray leaves.
struct SceneSpawn {
  float gx, gy, gz;
  __device__ __forceinline__ void lifted(float lift, float Px, float Py, float Pz, float dx, float dy, float dz,
                                          float &x, float &y, float &z) const {
    float nx = gx, ny = gy, nz = gz;
    const float c = nx * dx + ny * dy + nz * dz;
    if (c < 0.0f) nx = -nx, ny = -ny, nz = -nz;
    x = Px + nx * lift;
    y = Py + ny * lift;
    z = Pz + nz * lift;
  }
  __device__ __forceinline__ void continuation(const nrt_path_params &p, float Px, float Py, float Pz, float ox,
                                               float oy, float oz, float4 &co, float4 &cd) const {
    float x, y, z;
    lifted(p.ray_min_t, Px, Py, Pz, ox, oy, oz, x, y, z);
    co = make_float4(x, y, z, p.ray_min_t);
    cd = make_float4(ox, oy, oz, p.ray_max_t);
    if (ox == 0.0f && oy == 0.0f && oz == 0.0f) {  // total internal reflection: a radiance ray that misses at the root
      co.w = 0.0f;
      cd.w = -1.0f;
    }
  }
  // Direction and dist come from the unlifted P.  The lifted ray meets the light triangle's plane (unit normal ln) at
  // dist - ray_min_t (ln . g') / (ln . l) rather than at dist (g' = the lift's direction), so that is where max_t is put,
  // less 1e-5: with dist - 1e-5 the light would occlude its own sample.  A light seen edge-on (ln . l = 0) adds nothing.
  __device__ __forceinline__ void shadow(const nrt_path_params &p, float Px, float Py, float Pz, float lx, float ly,
                                         float lz, float dist, float lnx, float lny, float lnz, float4 &so,
                                         float4 &sd) const {
    float x, y, z;
    lifted(p.ray_min_t, Px, Py, Pz, lx, ly, lz, x, y, z);
    so = make_float4(x, y, z, 0.00001f);
    sd = make_float4(lx, ly, lz, plane_max_t(Px, Py, Pz, x, y, z, lx, ly, lz, dist, lnx, lny, lnz));
  }
  // max_t of a ray from (x, y, z), P lifted, along the unit direction l towards a point at dist from P on a plane of
  // unit normal ln: where the ray meets that plane, less 1e-5
  __device__ __forceinline__ static float plane_max_t(float Px, float Py, float Pz, float x, float y, float z, float lx,
                                                      float ly, float lz, float dist, float lnx, float lny, float lnz) {
    const float ndl = lnx * lx + lny * ly + lnz * lz;
    const float ndo = lnx * (x - Px) + lny * (y - Py) + lnz * (z - Pz);  // lift (ln . g')
    return (ndl != 0.0f ? dist - ndo / ndl : dist) - 0.00001f;
  }
};

// t[k] = ((m[0][k] v0 + m[1][k] v1) + m[2][k] v2) + m[3][k] over a full row-major 4x4 (Matrix::MultV)
__device__ __forceinline__ void multv16(const float *m, float x, float y, float z, float &ox, float &oy, float &oz) {
  ox = ((m[0] * x + m[4] * y) + m[8] * z) + m[12];
  oy = ((m[1] * x + m[5] * y) + m[9] * z) + m[13];
  oz = ((m[2] * x + m[6] * y) + m[10] * z) + m[14];
}

__device__ __forceinline__ void world_triangle(const InstanceDev *I, uint32_t prim, float w[9]) {
  const Mat43 xf = load_mat(&I->xf);
  const uint32_t *f = I->faces + 3 * (size_t)prim;
  for (int k = 0; k < 3; k++) {
    const float *v = I->verts + 3 * (size_t)f[k];
    multv(xf, v[0], v[1], v[2], w[3 * k], w[3 * k + 1], w[3 * k + 2]);
  }
}

// unit cross(e1, e2) of a world triangle and the length of the cross product (geometric_normal's arithmetic)
__device__ __forceinline__ void world_normal(const float w[9], float &nx, float &ny, float &nz, float &area2) {
  const float e1x = w[3] - w[0], e1y = w[4] - w[1], e1z = w[5] - w[2];
  const float e2x = w[6] - w[0], e2y = w[7] - w[1], e2z = w[8] - w[2];
  nx = e1y * e2z - e1z * e2y;
  ny = e1z * e2x - e1x * e2z;
  nz = e1x * e2y - e1y * e2x;
  area2 = sqrtf(nx * nx + ny * ny + nz * nz);
  const float il = area2 > 0.0f ? 1.0f / area2 : 0.0f;
  nx *= il;
  ny *= il;
  nz *= il;
}

// One emissive pair in world space, 64 bytes: v0.xyz v1.x | v1.yz v2.xy | v2.z n.xyz | area e.xyz (n: unit
// cross(e1, e2), area: half its length before normalisation -- geometric_normal() of the world triangle)
struct SceneLights {
  const float4 *rec;
  __device__ __forceinline__ void sample(uint32_t k, float c0, float c1, float c2, float Px, float Py, float Pz,
                                         float &lx, float &ly, float &lz, float &lnx, float &lny, float &lnz,
                                         float &area, float &ex, float &ey, float &ez) const {
    const float4 a = __ldg(rec + 4 * (size_t)k), b = __ldg(rec + 4 * (size_t)k + 1), c = __ldg(rec + 4 * (size_t)k + 2),
                 d = __ldg(rec + 4 * (size_t)k + 3);
    lx = c0 * a.x + c1 * a.w + c2 * b.z - Px;
    ly = c0 * a.y + c1 * b.x + c2 * b.w - Py;
    lz = c0 * a.z + c1 * b.y + c2 * c.x - Pz;
    lnx = c.y;
    lny = c.z;
    lnz = c.w;
    area = d.x;
    ex = d.y;
    ey = d.z;
    ez = d.w;
  }
};

}  // namespace

// What a pass outside scene.cu reads of a committed scene.  (The types in the signatures below are not the anonymous
// ones above, so that every file that includes this header names the same functions.)
struct SceneView {
  int device;
  uint32_t n;                // instances
  const uint32_t *n_faces;   // per instance: triangles of its accel (0: not a triangle accel)
  const void *inst;          // DEVICE InstanceDev per instance
  const float *state76;      // DEVICE, nrt_scene_instance_state's 76 floats per instance
};
SceneView scene_view(const nrt_scene *s);
// the scene walk of n rays into SceneHit32 records (nrt_scene_traverse_device), ordered on the device after the
// earlier walks of the scene that used the same scratch
int scene_walk(const nrt_scene *s, const Ray36 *d_rays, size_t n, void *d_hits, uint8_t *d_mask, uint32_t flags,
               cudaStream_t st);

class CallMemory;  // pass_host.cuh

// What one scene path or lightmap call keeps on the device, in its CallMemory: the per-instance shading table, the
// world-space light records (SceneLights) and the walk's buffers.
struct ScenePathCall {
  const nrt_scene *s = nullptr;
  nrt_path_params p{};
  uint32_t trav_flags = 0;
  SceneShadingDev *shading = nullptr;
  float4 *lights = nullptr;
  Ray36 *rays = nullptr;
  SceneHit32 *hits = nullptr;
  uint8_t *mask = nullptr;
  unsigned long long *ctr = nullptr;  // [0] continuation rays, [1] shadow rays, [2] camera rays
  uint32_t launches = 0, trav_launches = 0;
};
// The set-up both scene.cu's path pass and the scene lightmap bake start with, after their own parameter checks:
// refuses a NULL shading array, material ids or normals in p, ANY_HIT, a non-triangle instance and an emissive pair
// that is no {instance, face} of the scene (read back once); then allocates the call's buffers for `cap` rays in mem
// and writes the shading table and the light records.
int scene_path_setup(const char *name, const nrt_scene *s, const nrt_path_params &p, const nrt_scene_shading *shading,
                     size_t cap, cudaStream_t st, CallMemory &mem, ScenePathCall &c);

}  // namespace nrt
