// The reference's bidirectional path tracer (examples/bidir_path_tracer/main.cc) as a wavefront pass.  Per wave of
// whole tiles: eye starts, max_bounces eye bounces, light starts, max_bounces light bounces, the connection records
// (count, scan, write), one traversal launch over all calcG rays, then the per-sample and per-pixel sums.  The bounce
// and connection rays are traced by the persistent traversal kernel with the retire steps of wavefront.cuh
// (bd::BounceEpilogue, bd::ConnEpilogue) or, under NRT_TRAVERSE_CONFORMANCE, by the reference-order walk with the same
// retire steps.  What is here: argument checks, the light table, the stage kernels and the launch bookkeeping.
#include <algorithm>
#include <mutex>
#include <string>

#include "../../include/nanort_b200_scene_bdpt.h"
#include "common.cuh"
#include "radix_sort.cuh"
#include "scan.cuh"
#include "scene.cuh"
#include "wavefront.cuh"
#include "pass_host.cuh"

namespace nrt {

int launch_traverse_bdpt_bounce(const Accel *a, const bd::BounceRays &rays, const bd::BounceEpilogue &epi,
                                const unsigned long long *d_count, size_t capacity, uint32_t flags, cudaStream_t s);
int launch_traverse_bdpt_connect(const Accel *a, const bd::ConnRays &rays, const bd::ConnEpilogue &epi,
                                 const unsigned long long *d_count, size_t capacity, uint32_t flags, cudaStream_t s);

namespace {

using namespace bd;

// Scratch of one wave is bounded by this (tiles per wave = what fits; at least one tile)
constexpr size_t kWaveBudget = (size_t)512 << 20;

// ---- light table (LightSampler's constructor, main.cc:694-729)
// *flag = 1 iff material `id` emits (max(Le) > kEps); an id out of range sets info[1] and *flag = 0
__device__ __forceinline__ void emissive_flag(const Scene &sc, uint32_t id, uint32_t *flag, unsigned long long *info) {
  if (id >= sc.n_materials) {
    info[1] = 1ull;
    *flag = 0u;
    return;
  }
  const float *le = sc.mats[id].emission;
  const float mx = le[0] < (le[1] < le[2] ? le[2] : le[1]) ? (le[1] < le[2] ? le[2] : le[1]) : le[0];  // std::max
  *flag = mx <= kEps ? 0u : 1u;
}

// a light triangle's area (main.cc:707-712)
__device__ __forceinline__ float light_area(float3 v0, float3 v1, float3 v2) {
  return 0.5f * length(cross(sub(v2, v0), sub(v1, v0)));
}

// flags[i] = face i emits (max(Le) > kEps); info[1] = some material id is out of range
__global__ void __launch_bounds__(256)
    light_flags_kernel(Scene sc, uint32_t n, uint32_t *__restrict__ flags, unsigned long long *info) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  emissive_flag(sc, sc.mat_ids[i], flags + i, info);
}

// emissive faces in face order: ids and the bits of their areas; info[0] = their count
__global__ void __launch_bounds__(256)
    light_compact_kernel(Scene sc, uint32_t n, const uint32_t *__restrict__ flags, const uint32_t *__restrict__ offs,
                         uint32_t *__restrict__ ids, uint32_t *__restrict__ area_bits, unsigned long long *info) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (flags[i]) {
    float3 v[3];
    for (int k = 0; k < 3; k++) v[k] = f3(sc.verts + 3 * (size_t)sc.faces[3 * (size_t)i + k]);
    const float area = light_area(v[0], v[1], v[2]);
    ids[offs[i]] = i;
    area_bits[offs[i]] = __float_as_uint(area);
  }
  if (i == n - 1) info[0] = (unsigned long long)offs[i] + flags[i];
}

// totalArea_, summed in face order (one thread: the reference's sequential sum)
__global__ void light_total_kernel(const uint32_t *__restrict__ area_bits, uint32_t n, float *total) {
  float t = 0.0f;
  for (uint32_t i = 0; i < n; i++) t += __uint_as_float(area_bits[i]);
  *total = t;
}

// cdf_ over the (area, face) order, one sequential float sum
__global__ void light_cdf_kernel(const uint32_t *__restrict__ area_bits, uint32_t n, const float *total,
                                 float *__restrict__ cdf) {
  const float T = *total;
  float c = __uint_as_float(area_bits[0]) / T;
  cdf[0] = c;
  for (uint32_t i = 1; i < n; i++) {
    c = c + __uint_as_float(area_bits[i]) / T;
    cdf[i] = c;
  }
}

// ---- per-wave stages
struct BdptWave {
  TileMap tm;
  uint32_t spp_total;
  float cam[12];
  unsigned long long s0;  // the wave's first slot (of the call)
  uint32_t count;         // slots in the wave
};

// eyeSubpath (main.cc:1015-1043) of every slot: seed, jitter, camera ray, lens vertex; the slot joins queue 0
__global__ void __launch_bounds__(256)
    eye_start_kernel(BdptWave w, Subpaths sp, PathState *__restrict__ st, uint32_t *__restrict__ queue,
                     unsigned long long *count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t pix = 0, smp = 0;
  const bool valid = i < w.count && slot_to_pixel(w.tm, w.s0 + i, pix, smp);
  if (i < w.count) {
    sp.n_eye[i] = valid ? 1u : 0u;
    sp.n_light[i] = 0u;
  }
  if (valid) {
    const uint32_t W = w.tm.width, H = w.tm.height;
    const uint32_t x = pix % W, y = H - 1u - pix / W;  // the reference's loop row
    Random rng;
    rng.seed((y * W + x) * w.spp_total + (w.tm.sample0 + smp));
    const float px = (float)x + (rng.real() - 0.5f);
    const float py = (float)y + (rng.real() - 0.5f);
    const float sx = px / (float)W - 0.5f, sy = py / (float)H - 0.5f;
    const float *c = w.cam;
    const float3 dir = normalize(f3(sx * c[3] + sy * c[6] + c[9], sx * c[4] + sy * c[7] + c[10],
                                    sx * c[5] + sy * c[8] + c[11]));
    const float3 org = f3(c[0], c[1], c[2]), z = f3(0.0f, 0.0f, 0.0f);
    vstore(sp.eye[(size_t)i * sp.stride], org, z, dir, f3(1.0f, 1.0f, 1.0f), z, 1.0f, 0.0f, NRT_BDPT_LENS, kNone,
           kNone);
    PathState s;
    s.org_pdf = make_float4(org.x, org.y, org.z, 1.0f);
    s.dir = make_float4(dir.x, dir.y, dir.z, 0.0f);
    s.beta = make_float4(1.0f, 1.0f, 1.0f, 0.0f);
    s.rng = make_uint4(rng.s[0], rng.s[1], rng.s[2], rng.s[3]);
    st[i] = s;
  }
  queue_append(queue, count, valid, i);
}

// LightSampler::sample (main.cc:731-765) and lightSubpath's start (main.cc:1045-1075) of slot i: picks
// ids_[lower_bound(cdf_, u)]; light.fetch(id, v, n, mid) gives that light's vertices, face-varying normals and material,
// light.origin(P, dir) where its first ray starts.
template <class Light>
__device__ __forceinline__ void light_start_slot(const Scene &sc, uint32_t i, Subpaths sp, PathState *__restrict__ st,
                                                 Light &lt) {
  PathState s = st[i];
  Random rng;
  rng.s[0] = s.rng.x, rng.s[1] = s.rng.y, rng.s[2] = s.rng.z, rng.s[3] = s.rng.w;
  const float rnd = rng.real();
  uint32_t lo = 0, hi = sc.n_lights;  // std::lower_bound
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (sc.cdf[mid] < rnd)
      lo = mid + 1;
    else
      hi = mid;
  }
  const uint32_t light = sc.light_ids[min(lo, sc.n_lights - 1u)];
  float u1 = rng.real();
  float u2 = rng.real();
  if (u1 + u2 >= 1.0f) {
    u1 = 1.0f - u1;
    u2 = 1.0f - u2;
  }
  float3 v[3], fn[3];
  uint32_t mid;
  lt.fetch(light, v, fn, mid);
  const float b0 = 1.0f - u1 - u2;
  const float3 pos = add(add(mul(v[0], b0), mul(v[1], u1)), mul(v[2], u2));
  const float3 nrm = add(add(mul(fn[0], b0), mul(fn[1], u1)), mul(fn[2], u2));
  const float pdf_pos = 1.0f / *sc.total_area;
  const float3 le = f3(sc.mats[mid].emission);
  // directionCosTheta(norm, rng.nextReal(), rng.nextReal(), &pdfDir): arguments drawn right to left; the light's
  // interpolated normal goes in un-normalised
  const float d2 = rng.real();
  const float d1 = rng.real();
  float pdf_dir;
  const float3 dir = direction_cos_theta(nrm, d1, d2, pdf_dir);
  const float3 beta = div(le, pdf_pos), z = f3(0.0f, 0.0f, 0.0f);
  vstore(sp.light[(size_t)i * sp.stride], pos, z, normalize(nrm), beta, z, pdf_pos, 0.0f, NRT_BDPT_LIGHT, kNone,
         kNone);
  sp.n_light[i] = 1u;
  const float3 o = lt.origin(pos, dir);
  s.org_pdf = make_float4(o.x, o.y, o.z, pdf_dir);
  s.dir = make_float4(dir.x, dir.y, dir.z, 0.0f);
  s.beta = make_float4(beta.x, beta.y, beta.z, 0.0f);
  s.rng = make_uint4(rng.s[0], rng.s[1], rng.s[2], rng.s[3]);
  st[i] = s;
}

// the flat mesh's face `id`; the first ray starts at the light
struct FlatLight {
  const Scene &sc;
  __device__ __forceinline__ void fetch(uint32_t id, float3 v[3], float3 fn[3], uint32_t &mid) const {
    const uint32_t *f = sc.faces + 3 * (size_t)id;
    const float *n = sc.fv_normals + 9 * (size_t)id;
    for (int k = 0; k < 3; k++) {
      v[k] = f3(sc.verts + 3 * (size_t)f[k]);
      fn[k] = f3(n + 3 * k);
    }
    mid = sc.mat_ids[id];
  }
  __device__ __forceinline__ float3 origin(float3 p, float3) const { return p; }
};

// lightSubpath's start for every slot whose eye subpath has a vertex beyond the lens
__global__ void __launch_bounds__(256)
    light_start_kernel(Scene sc, uint32_t count_slots, Subpaths sp, PathState *__restrict__ st,
                       uint32_t *__restrict__ queue, unsigned long long *count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < count_slots && sp.n_eye[i] > 1u;
  if (live) {
    FlatLight lt{sc};
    light_start_slot(sc, i, sp, st, lt);
  }
  queue_append(queue, count, live, i);
}

// counters: [0] rays of the launch about to run, [1] rays appended by it; totals [0] eye [1] light [2] connection
__global__ void begin_launch_kernel(unsigned long long *ctr, unsigned long long *total) {
  ctr[0] = ctr[1];
  ctr[1] = 0;
  *total += ctr[0];
}

// weightMIS (main.cc:1081-1211) of eye vertices E[0..ne) and light vertices Lv[0..nl)
__device__ float weight_mis(const Scene &sc, const nrt_bdpt_vertex *E, const nrt_bdpt_vertex *Lv, int ne, int nl) {
  if (ne <= 2 && nl == 0) return 1.0f;
  const int len = ne + nl;
  // the four entries of path[].second weightMIS overrides (indices ne - 1, ne, ne - 2, ne + 1)
  float o_e1 = 0.0f, o_e = 0.0f, o_e2 = 0.0f, o_e_1 = 0.0f;
  const nrt_bdpt_vertex *ve = &E[ne - 1];
  const nrt_bdpt_vertex *vl = nl >= 1 ? &Lv[nl - 1] : nullptr;
  const nrt_bdpt_vertex *vem = ne >= 2 ? &E[ne - 2] : nullptr;
  const nrt_bdpt_vertex *vlm = nl >= 2 ? &Lv[nl - 2] : nullptr;
  if (nl == 0) {
    o_e1 = 1.0f / *sc.total_area;
  } else if (nl == 1) {
    float3 to = sub(f3(ve->position), f3(vl->position));
    const float dist = length(to);
    to = div(to, dist);
    const float pdf_dir = fmax0(dot(f3(vl->norm), to));
    const float d = dot(f3(vl->norm), to);
    o_e1 = pdf_dir * d / (dist * dist);
  } else {
    float3 wi = sub(f3(vlm->position), f3(vl->position));
    float3 wo = sub(f3(ve->position), f3(vl->position));
    const float dist = length(wo);
    wi = normalize(wi);
    wo = normalize(wo);
    const float po = pdf_brdf(sc.mat(vl->material), wi, wo, f3(vl->original_norm), f3(vl->norm));
    o_e1 = po * fabsf(dot(f3(vl->norm), wo)) / (dist * dist);
  }
  if (vl) {
    float3 wi = sub(f3(vem->position), f3(ve->position));
    float3 wo = sub(f3(vl->position), f3(ve->position));
    const float dist = length(wo);
    wi = normalize(wi);
    wo = normalize(wo);
    const float po = pdf_brdf(sc.mat(ve->material), wi, wo, f3(ve->original_norm), f3(ve->norm));
    o_e = po * fabsf(dot(f3(ve->norm), wo)) / (dist * dist);
  }
  if (vem) {
    if (nl == 0) {
      float3 to = sub(f3(vem->position), f3(ve->position));
      const float dist = length(to);
      to = div(to, dist);
      const float pdf_dir = fmax0(dot(f3(ve->norm), to));
      const float d = dot(f3(ve->norm), to);
      o_e2 = pdf_dir * d / (dist * dist);
    } else {
      float3 wi = sub(f3(vl->position), f3(ve->position));
      float3 wo = sub(f3(vem->position), f3(ve->position));
      const float dist = length(wo);
      wi = normalize(wi);
      wo = normalize(wo);
      const float po = pdf_brdf(sc.mat(ve->material), wi, wo, f3(ve->original_norm), f3(ve->norm));
      o_e2 = po * fabsf(dot(f3(ve->norm), wo)) / (dist * dist);
    }
  }
  if (vlm) {
    float3 wi = sub(f3(ve->position), f3(vl->position));
    float3 wo = sub(f3(vlm->position), f3(vl->position));
    const float dist = length(wo);
    wi = normalize(wi);
    wo = normalize(wo);
    const float po = pdf_brdf(sc.mat(vl->material), wi, wo, f3(vl->original_norm), f3(vl->norm));
    o_e_1 = po * fabsf(dot(f3(vl->norm), wo)) / (dist * dist);
  }
  // path[i] = (pdfFwd, pdfRev) of eye vertex i, then of the light vertices in reverse, with the overrides
  auto entry = [&](int i, float &fwd, float &rev) {
    const nrt_bdpt_vertex &v = i < ne ? E[i] : Lv[len - 1 - i];
    fwd = v.pdf_fwd;
    rev = v.pdf_rev;
    if (i == ne - 1) rev = o_e1;
    if (vl && i == ne) rev = o_e;
    if (vem && i == ne - 2) rev = o_e2;
    if (vlm && i == ne + 1) rev = o_e_1;
  };
  float mis = 0.0f, prob = 1.0f;
  for (int i = ne - 1; i >= 2; i--) {
    float fwd, rev;
    entry(i, fwd, rev);
    fwd = fwd == 0.0f ? 1.0f : fwd;
    rev = rev == 0.0f ? 1.0f : rev;
    prob *= rev / fwd;
    if (is_delta(sc.mat(E[i].material)) || is_delta(sc.mat(E[i - 1].material))) continue;
    mis += prob * prob;
  }
  prob = 1.0f;
  for (int i = ne; i < len; i++) {
    float fwd, rev;
    entry(i, fwd, rev);
    fwd = fwd == 0.0f ? 1.0f : fwd;
    rev = rev == 0.0f ? 1.0f : rev;
    prob *= rev / fwd;
    if (is_delta(sc.mat(Lv[len - i - 1].material)) ||
        (i + 1 < len && is_delta(sc.mat(Lv[len - i - 2].material))))
      continue;
    mis += prob * prob;
  }
  return 1.0f / (1.0f + mis);
}

// connectPath's unshadowed L for (e, l) (main.cc:1269-1277)
__device__ __forceinline__ float3 conn_L(const Scene &sc, const nrt_bdpt_vertex &ev, const nrt_bdpt_vertex &lv,
                                         int l) {
  const float3 fe = vertex_f(ev, sc.mat(ev.material), f3(lv.position));
  if (l == 1) {
    float3 to = sub(f3(lv.position), f3(ev.position));
    const float dist = length(to);
    to = div(to, dist);
    return mul(mul(mul(f3(ev.beta), fe), f3(lv.beta)), fabsf(dot(f3(lv.norm), neg(to))));
  }
  return mul(mul(mul(f3(ev.beta), fe), vertex_f(lv, sc.mat(lv.material), f3(ev.position))), f3(lv.beta));
}

// connectPath's enumeration (main.cc:1257-1285) of one sample; write == false only counts the connections to trace.
// The emission term's mis * ev.beta goes to *emit.
__device__ uint32_t connect_sample(const Scene &sc, uint32_t max_bounces, const nrt_bdpt_vertex *E, int ne,
                                   const nrt_bdpt_vertex *Lv, int nl, uint32_t slot, Conn *out, float3 *emit) {
  uint32_t k = 0;
  if (out && E[ne - 1].type == NRT_BDPT_LIGHT) *emit = mul(f3(E[ne - 1].beta), weight_mis(sc, E, Lv, ne, 0));
  for (int e = 2; e <= ne; e++) {
    const nrt_bdpt_vertex &ev = E[e - 1];
    if (is_delta(sc.mat(ev.material)) || ev.type == NRT_BDPT_LIGHT) continue;
    for (int l = 1; l <= nl; l++) {
      if (e + l - 2 > (int)max_bounces) continue;
      const nrt_bdpt_vertex &lv = Lv[l - 1];
      if (l != 1 && is_delta(sc.mat(lv.material))) continue;
      const float3 L = conn_L(sc, ev, lv, l);
      if (L.x == 0.0f && L.y == 0.0f && L.z == 0.0f) continue;
      if (out) {
        Conn c;
        c.slot = slot;
        c.el = (uint32_t)e | ((uint32_t)l << 16);
        c.L[0] = L.x;
        c.L[1] = L.y;
        c.L[2] = L.z;
        c.mis = weight_mis(sc, E, Lv, e, l);
        out[k] = c;
      }
      k++;
    }
  }
  return k;
}

__global__ void __launch_bounds__(128)
    conn_count_kernel(Scene sc, uint32_t max_bounces, uint32_t n, Subpaths sp, uint32_t *__restrict__ cnt) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t ne = sp.n_eye[i];
  cnt[i] = ne > 1u ? connect_sample(sc, max_bounces, sp.eye + (size_t)i * sp.stride, (int)ne,
                                    sp.light + (size_t)i * sp.stride, (int)sp.n_light[i], i, nullptr, nullptr)
                   : 0u;
}

// slot-major records at offs[i]; emit[i] = the emission term (0 without one); *total = the record count
__global__ void __launch_bounds__(128)
    conn_write_kernel(Scene sc, uint32_t max_bounces, uint32_t n, Subpaths sp, const uint32_t *__restrict__ cnt,
                      const uint32_t *__restrict__ offs, Conn *__restrict__ conns, float3 *__restrict__ emit,
                      unsigned long long *total) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (i == n - 1) *total = (unsigned long long)offs[i] + cnt[i];
  float3 em = f3(0.0f, 0.0f, 0.0f);
  const uint32_t ne = sp.n_eye[i];
  if (ne > 1u)
    connect_sample(sc, max_bounces, sp.eye + (size_t)i * sp.stride, (int)ne, sp.light + (size_t)i * sp.stride,
                   (int)sp.n_light[i], i, conns + offs[i], &em);
  emit[i] = em;
}

// connectPath's colour: the emission term, then the connections in record order
__global__ void __launch_bounds__(256)
    sample_sum_kernel(uint32_t n, Subpaths sp, const uint32_t *__restrict__ cnt, const uint32_t *__restrict__ offs,
                      const Conn *__restrict__ conns, const float3 *__restrict__ emit, float *__restrict__ rgb) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float3 c = f3(0.0f, 0.0f, 0.0f);
  if (sp.n_eye[i] > 1u) {
    c = add(c, emit[i]);
    const Conn *r = conns + offs[i];
    for (uint32_t k = 0; k < cnt[i]; k++) c = add(c, f3(r[k].L));
  }
  rgb[3 * (size_t)i + 0] = c.x;
  rgb[3 * (size_t)i + 1] = c.y;
  rgb[3 * (size_t)i + 2] = c.z;
}

// each pixel of the wave's tiles adds its samples' colours in ascending sample order
__global__ void __launch_bounds__(256)
    pixel_sum_kernel(BdptWave w, uint32_t n_pix, Subpaths sp, const float *__restrict__ rgb, float *__restrict__ accum) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_pix) return;
  const uint32_t tile_pix = w.tm.tile_w * w.tm.tile_h;
  const uint32_t k = j / tile_pix, q = j % tile_pix;
  const unsigned long long base = (unsigned long long)k * tile_pix * w.tm.spp + q;  // slot of sample 0
  uint32_t pix, smp;
  if (!slot_to_pixel(w.tm, w.s0 + base, pix, smp)) return;
  float *a = accum + 3 * (size_t)pix;
  float r = a[0], g = a[1], b = a[2];
  for (uint32_t s = 0; s < w.tm.spp; s++) {
    const size_t slot = base + (size_t)s * tile_pix;
    if (sp.n_eye[slot] <= 1u) continue;
    r += rgb[3 * slot + 0];
    g += rgb[3 * slot + 1];
    b += rgb[3 * slot + 2];
  }
  a[0] = r;
  a[1] = g;
  a[2] = b;
}

// ---- the scene pass's stage kernels: world-space geometry from the instance records (scene.cuh)
struct SceneGeo {
  const InstanceDev *inst;
  const float *state76;
  const SceneShadingDev *shading;  // per instance: material ids and LOCAL face-varying normals
  const uint32_t *face_offs;       // pair index of each instance's face 0; face_offs[n] = the pair count
  uint32_t n;                      // instances
  // the instance of pair `k` (flattened order: face_offs[instance] + face)
  __device__ __forceinline__ uint32_t instance(uint32_t k) const {
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) / 2;
      if (face_offs[mid] <= k)
        lo = mid;
      else
        hi = mid;
    }
    return lo;
  }
  // unit world geometric normal of face `face` of instance I (cross(e1, e2) of the world triangle)
  __device__ __forceinline__ float3 geo_normal(uint32_t I, uint32_t face) const {
    float w[9], a2;
    float3 g;
    world_triangle(inst + I, face, w);
    world_normal(w, g.x, g.y, g.z, a2);
    return g;
  }
  // the face's three face-varying normals moved to world space by the instance's inverse_transpose33
  __device__ __forceinline__ void world_normals(uint32_t I, uint32_t face, float wn[9]) const {
    const float *T = state76 + 76 * (size_t)I + 48;
    const float *n0 = shading[I].fvn + 9 * (size_t)face;
    for (int k = 0; k < 3; k++) multv16(T, n0[3 * k], n0[3 * k + 1], n0[3 * k + 2], wn[3 * k], wn[3 * k + 1], wn[3 * k + 2]);
  }
};

// Per vertex record: the instance of its face (0xFFFFFFFF where prim_id is); per slot: the sampled {instance, face}
struct SceneVerts {
  uint32_t *eye_inst, *light_inst, *light_pair;
};

// A scene ray spawned at a vertex starts kEps above it along the unit world geometric normal g, on the side it leaves
struct LiftedOrigin {
  float3 g;
  __device__ __forceinline__ float3 operator()(float3 p, float3 d) const {
    float x, y, z;
    SceneSpawn{g.x, g.y, g.z}.lifted(kEps, p.x, p.y, p.z, d.x, d.y, d.z, x, y, z);
    return f3(x, y, z);
  }
};

// light_flags_kernel over the {instance, face} pairs
__global__ void __launch_bounds__(256)
    pair_flags_kernel(Scene sc, SceneGeo g, uint32_t n, uint32_t *__restrict__ flags, unsigned long long *info) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t I = g.instance(i);
  emissive_flag(sc, g.shading[I].mat_ids[i - g.face_offs[I]], flags + i, info);
}

// light_compact_kernel over the pairs: the world triangle's area
__global__ void __launch_bounds__(256)
    pair_compact_kernel(SceneGeo g, uint32_t n, const uint32_t *__restrict__ flags, const uint32_t *__restrict__ offs,
                        uint32_t *__restrict__ ids, uint32_t *__restrict__ area_bits, unsigned long long *info) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (flags[i]) {
    const uint32_t I = g.instance(i);
    float w[9];
    world_triangle(g.inst + I, i - g.face_offs[I], w);
    ids[offs[i]] = i;
    area_bits[offs[i]] = __float_as_uint(light_area(f3(w), f3(w + 3), f3(w + 6)));
  }
  if (i == n - 1) info[0] = (unsigned long long)offs[i] + flags[i];
}

// the sampled pair in world space; the first ray is lifted off the light
struct SceneLight {
  const SceneGeo &g;
  uint32_t *pair;
  float3 gn;
  __device__ __forceinline__ void fetch(uint32_t id, float3 v[3], float3 fn[3], uint32_t &mid) {
    const uint32_t I = g.instance(id), face = id - g.face_offs[I];
    float w[9], wn[9], a2;
    world_triangle(g.inst + I, face, w);
    g.world_normals(I, face, wn);
    for (int k = 0; k < 3; k++) {
      v[k] = f3(w + 3 * k);
      fn[k] = f3(wn + 3 * k);
    }
    world_normal(w, gn.x, gn.y, gn.z, a2);
    mid = g.shading[I].mat_ids[face];
    pair[0] = I;
    pair[1] = face;
  }
  __device__ __forceinline__ float3 origin(float3 p, float3 d) const { return LiftedOrigin{gn}(p, d); }
};

__global__ void __launch_bounds__(256)
    scene_light_start_kernel(Scene sc, SceneGeo g, uint32_t count_slots, Subpaths sp, SceneVerts sv,
                             PathState *__restrict__ st, uint32_t *__restrict__ queue, unsigned long long *count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < count_slots && sp.n_eye[i] > 1u;
  if (i < count_slots) {
    if (sp.n_eye[i] > 0u) sv.eye_inst[(size_t)i * sp.stride] = kNone;  // the lens vertex
    sv.light_pair[2 * (size_t)i] = sv.light_pair[2 * (size_t)i + 1] = kNone;
  }
  if (live) {
    SceneLight lt{g, sv.light_pair + 2 * (size_t)i, f3(0.0f, 0.0f, 0.0f)};
    light_start_slot(sc, i, sp, st, lt);
    sv.light_inst[(size_t)i * sp.stride] = kNone;
  }
  queue_append(queue, count, live, i);
}

// the walk's rays of a bounce, in queue order
__global__ void __launch_bounds__(256)
    scene_bounce_rays_kernel(BounceRays q, uint32_t n, Ray36 *__restrict__ rays) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Ray36 r;
  q.load(i, r.org[0], r.org[1], r.org[2], r.dir[0], r.dir[1], r.dir[2], r.min_t, r.max_t);
  r.type = 0;
  rays[i] = r;
}

// raytrace's per-hit block from the scene walk's records: P = org + t dir of the world ray, the instance's
// face-varying normals in world space, its material ids; the next ray is lifted
__global__ void __launch_bounds__(256)
    scene_bounce_kernel(Scene sc, SceneGeo g, Subpaths sp, uint32_t *__restrict__ vinst, PathState *__restrict__ st,
                        const uint32_t *__restrict__ queue_in, uint32_t n_rays, const SceneHit32 *__restrict__ hits,
                        const uint8_t *__restrict__ mask, uint32_t *__restrict__ queue_out,
                        unsigned long long *count_out, uint32_t max_bounces, int eye) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool cont = false;
  uint32_t slot = 0;
  if (i < n_rays && mask[i]) {
    slot = queue_in[i];
    const SceneHit32 h = hits[i];
    PathState s = st[slot];
    float w[9], wn[9], a2;
    float3 gn;
    world_triangle(g.inst + h.node_id, h.prim_id, w);
    world_normal(w, gn.x, gn.y, gn.z, a2);
    g.world_normals(h.node_id, h.prim_id, wn);
    uint32_t *np = (eye ? sp.n_eye : sp.n_light) + slot;
    const uint32_t n0 = *np;
    // the walk reports a world distance; the light's first ray is the one whose direction is not unit length
    // (directionCosTheta of the un-normalised light normal), so its distance becomes the ray parameter
    const float3 dir = f3(s.dir.x, s.dir.y, s.dir.z);
    const float t = !eye && n0 == 1u ? h.t / length(dir) : h.t;
    const float3 next = add(f3(s.org_pdf.x, s.org_pdf.y, s.org_pdf.z), mul(dir, t));
    uint32_t n = n0;
    cont = subpath_vertex(sc, eye != 0, max_bounces, s, (eye ? sp.eye : sp.light) + (size_t)slot * sp.stride, n, next,
                          hit_normal(wn, h.u, h.v), g.shading[h.node_id].mat_ids[h.prim_id], h.prim_id,
                          LiftedOrigin{gn});
    if (n != n0) vinst[(size_t)slot * sp.stride + n0] = h.node_id;
    *np = n;
    st[slot] = s;
  }
  queue_append(queue_out, count_out, cont, slot);
}

// calcG's rays over the scene: direction and dist from the unlifted vertices, the origin lifted along the eye vertex's
// geometric normal, max_t where the ray meets the light vertex's plane less 1e-5 (SceneSpawn::shadow's rule)
__global__ void __launch_bounds__(256)
    scene_conn_rays_kernel(SceneGeo g, const Conn *__restrict__ conns, uint32_t n, Subpaths sp, SceneVerts sv,
                           Ray36 *__restrict__ rays) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t slot = conns[i].slot, el = conns[i].el, l = el >> 16;
  const size_t ie = (size_t)slot * sp.stride + (el & 0xFFFFu) - 1, il = (size_t)slot * sp.stride + l - 1;
  const float3 pe = f3(sp.eye[ie].position), pl = f3(sp.light[il].position);
  float3 to;
  float dist;
  conn_ray(pe, pl, to, dist);
  const float3 ge = g.geo_normal(sv.eye_inst[ie], sp.eye[ie].prim_id);
  const float3 gl = l == 1 ? g.geo_normal(sv.light_pair[2 * (size_t)slot], sv.light_pair[2 * (size_t)slot + 1])
                           : g.geo_normal(sv.light_inst[il], sp.light[il].prim_id);
  const float3 o = LiftedOrigin{ge}(pe, to);
  Ray36 r;
  r.org[0] = o.x, r.org[1] = o.y, r.org[2] = o.z;
  r.dir[0] = to.x, r.dir[1] = to.y, r.dir[2] = to.z;
  r.min_t = kEps;
  r.max_t = SceneSpawn::plane_max_t(pe.x, pe.y, pe.z, o.x, o.y, o.z, to.x, to.y, to.z, dist, gl.x, gl.y, gl.z);
  r.type = 0;
  rays[i] = r;
}

// visible iff the walk reports no hit nearer than max_t; G from the unlifted geometry
__global__ void __launch_bounds__(256)
    scene_conn_g_kernel(Conn *__restrict__ conns, uint32_t n, Subpaths sp, const Ray36 *__restrict__ rays,
                        const SceneHit32 *__restrict__ hits, const uint8_t *__restrict__ mask) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Conn &c = conns[i];
  const uint32_t slot = c.slot, el = c.el;
  const nrt_bdpt_vertex &ev = sp.eye[(size_t)slot * sp.stride + (el & 0xFFFFu) - 1];
  const nrt_bdpt_vertex &lv = sp.light[(size_t)slot * sp.stride + (el >> 16) - 1];
  float3 to;
  float dist;
  conn_ray(f3(ev.position), f3(lv.position), to, dist);
  const bool blocked = mask[i] && hits[i].t < rays[i].max_t;
  conn_finish(c, blocked ? 0.0f : g_term(to, dist, f3(ev.norm), f3(lv.norm)));
}

uint32_t scan_launches(uint32_t n) {
  const uint32_t tiles = (n + kScanTile - 1) / kScanTile;
  return n == 0 ? 0u : tiles > 1 ? 2u + scan_launches(tiles) : 1u;
}

// upper bound of connectPath's connections of one sample: e - 2 in [0, B), l in [1, B - (e - 2)]
uint32_t max_conns(uint32_t B) { return B * (B + 1) / 2; }

struct Out {  // export buffers (nullptr: render into accum)
  nrt_bdpt_vertex *eye, *light;
  uint32_t *n_eye, *n_light;
  float *rgb;
  uint32_t *eye_inst, *light_inst, *light_pair;  // the scene pass's
};

// the rules both passes share
int check_common(const nrt_bdpt_params &p, const char *who) {
  if (p.flags & ~(uint32_t)NRT_TRAVERSE_CONFORMANCE)
    return refuse(who,
                  "flags other than NRT_TRAVERSE_CONFORMANCE (calcG needs the nearest distance: no ANY_HIT)");
  if (p.width == 0 || p.height == 0 || p.spp == 0 || p.n_shards == 0 || p.shard >= p.n_shards || p.tile_w == 0 ||
      p.tile_h == 0 || (p.tile_w % 8) != 0 || (p.tile_h % 4) != 0)
    return refuse(who, "bad image, sample or tile parameters");
  if ((uint64_t)p.sample0 + p.spp > p.spp_total) return refuse(who, "sample0 + spp > spp_total");
  if (p.max_bounces == 0 || p.max_bounces > 64) return refuse(who, "max_bounces must lie in [1, 64]");
  return NRT_OK;
}

int check_params(const Accel *a, const nrt_bdpt_params *pp, const char *who) {
  if (!a || !pp) return refuse(who, "NULL argument");
  const nrt_bdpt_params &p = *pp;
  if (!p.d_materials || !p.d_material_ids || !p.d_facevarying_normals || p.n_materials == 0)
    return refuse(who, "materials, material ids and face-varying normals are required");
  if (const int rc = check_common(p, who)) return rc;
  if (a->prim_kind != 0 || a->d_prim_boxes || !a->d_faces || !a->d_verts || !a->d_pair || !a->d_tris_cm)
    return refuse(who, "the accel must be a triangle accel");
  return NRT_OK;
}

// Sizes of one call: this shard's slots, the wave capacity and the light table's capacity.
// extra_per_slot: what a pass keeps per slot beyond the flat pass's records.
struct Layout {
  TileMap tm;
  unsigned long long total_slots, cap;
  uint32_t B, stride, mc, n_lights_max;  // n_lights_max: faces (flat) or pairs (scene)
  bool exported;
};

int make_layout(const nrt_bdpt_params &p, bool exported, uint32_t nf, size_t extra_per_slot, const char *who,
                Layout &L) {
  L.tm = TileMap{p.width, p.height, p.spp, p.sample0, p.tile_w, p.tile_h, p.shard, p.n_shards, 0u};
  const ShardSlots sh = shard_slots(p.width, p.height, p.tile_w, p.tile_h, p.spp, p.shard, p.n_shards);
  L.total_slots = sh.total;
  L.B = p.max_bounces;
  L.stride = L.B + 1;
  L.mc = max_conns(L.B);
  L.exported = exported;
  const uint32_t stride = L.stride, mc = L.mc;
  // per slot: state, two subpaths (unless exported), queues, counts, offsets, emission, colour, records
  const size_t per_slot = sizeof(PathState) + (exported ? 0 : 2 * (size_t)stride * sizeof(nrt_bdpt_vertex) + 8 + 12) +
                          2 * 4 + 4 + 4 + 12 + (size_t)mc * sizeof(Conn) + 8 + extra_per_slot;
  L.cap = sh.wave(kWaveBudget / per_slot);
  if (L.cap > 0xFFFFFFFFull / mc) {
    set_error(std::string(who) + ": a tile holds too many samples");
    return NRT_ERR_INVALID;
  }
  L.n_lights_max = nf;
  return NRT_OK;
}

// The scratch of one pass: the light table, then the buffers of one wave
struct Scratch {
  uint32_t *l_flags, *l_offs, *l_ids, *l_keys, *l_keys_tmp, *l_table, *l_scratch;
  float *l_total;
  PathState *st;
  nrt_bdpt_vertex *w_eye, *w_light;  // the wave's subpaths, their lengths and the sample colours (not exported)
  uint32_t *w_ne, *w_nl;
  float *w_rgb;
  uint32_t *queue[2], *cnt, *offs;
  float3 *emit;
  Conn *conns;
  uint32_t *scan_scratch;
};

Scratch carve_scratch(Carver &c, const Layout &L) {
  const uint32_t nf = L.n_lights_max, sort_tiles = (nf + kSortTile - 1) / kSortTile;
  const size_t cap = L.cap;
  Scratch m = {};
  m.l_flags = c.take<uint32_t>(nf);
  m.l_offs = c.take<uint32_t>(nf);
  m.l_ids = c.take<uint32_t>(nf);
  m.l_keys = c.take<uint32_t>(nf);
  m.l_keys_tmp = c.take<uint32_t>(nf);
  m.l_table = c.take<uint32_t>(16 * (size_t)sort_tiles + 1);
  m.l_scratch = c.take<uint32_t>(std::max(scan_scratch_words(nf), scan_scratch_words(16 * sort_tiles)));
  m.l_total = c.take<float>(4);
  m.st = c.take<PathState>(cap);
  if (!L.exported) {
    m.w_eye = c.take<nrt_bdpt_vertex>(cap * L.stride);
    m.w_light = c.take<nrt_bdpt_vertex>(cap * L.stride);
    m.w_ne = c.take<uint32_t>(cap);
    m.w_nl = c.take<uint32_t>(cap);
    m.w_rgb = c.take<float>(3 * cap);
  }
  m.queue[0] = c.take<uint32_t>(cap);
  m.queue[1] = c.take<uint32_t>(cap);
  m.cnt = c.take<uint32_t>(cap);
  m.offs = c.take<uint32_t>(cap);
  m.emit = c.take<float3>(cap);
  m.conns = c.take<Conn>(cap * L.mc);
  m.scan_scratch = c.take<uint32_t>(scan_scratch_words((uint32_t)cap));
  return m;
}

// The flat mesh: the light table over its faces, the accel's traversal launches with the retire steps
struct FlatWalk {
  const Accel *a;
  uint32_t flags;
  int light_candidates(const Scene &sc, uint32_t n, uint32_t *l_flags, uint32_t *l_offs, uint32_t *l_ids,
                       uint32_t *l_keys, uint32_t *l_scratch, unsigned long long *info, cudaStream_t s) {
    const unsigned gf = (n + 255) / 256;
    light_flags_kernel<<<gf, 256, 0, s>>>(sc, n, l_flags, info);
    NRT_CUDA(cudaGetLastError());
    if (const int rc = exclusive_scan_u32_async(l_flags, l_offs, n, l_scratch, s)) return rc;
    light_compact_kernel<<<gf, 256, 0, s>>>(sc, n, l_flags, l_offs, l_ids, l_keys, info);
    NRT_CUDA(cudaGetLastError());
    return NRT_OK;
  }
  void wave(unsigned long long) {}
  void light_start(const Scene &sc, uint32_t count, const Subpaths &sp, PathState *st, uint32_t *queue,
                   unsigned long long *ctr1, cudaStream_t s) {
    light_start_kernel<<<(count + 255) / 256, 256, 0, s>>>(sc, count, sp, st, queue, ctr1);
  }
  // ctr[0]: the launch's rays (device); ctr[1] receives the continuing ones.  The count stays on the device, so
  // *empty (no ray left: the later bounces of this subpath can be skipped) is never known here.
  int bounce(const Scene &sc, const Subpaths &sp, PathState *st, const uint32_t *q_in, uint32_t *q_out,
             unsigned long long *ctr, uint32_t count, uint32_t B, int eye, PassClock &tm, uint32_t &launches,
             uint32_t &trav_launches, bool *empty, cudaStream_t s) {
    *empty = false;
    if (const int rc = tm.begin(s)) return rc;
    const BounceRays rays{q_in, st};
    const BounceEpilogue epi{sc, sp, st, q_in, q_out, ctr + 1, B, eye};
    if (const int rc = launch_traverse_bdpt_bounce(a, rays, epi, ctr, count, flags, s)) return rc;
    if (const int rc = tm.end(s)) return rc;
    launches++;
    trav_launches++;
    return NRT_OK;
  }
  int connect(Conn *conns, const Subpaths &sp, unsigned long long *ctr, size_t capacity, PassClock &tm,
              uint32_t &launches, uint32_t &trav_launches, cudaStream_t s) {
    if (const int rc = tm.begin(s)) return rc;
    if (const int rc = launch_traverse_bdpt_connect(a, ConnRays{conns, sp}, ConnEpilogue{conns, sp}, ctr, capacity,
                                                    flags, s))
      return rc;
    if (const int rc = tm.end(s)) return rc;
    launches++;
    trav_launches++;
    return NRT_OK;
  }
};

// One pass over L's slots on the scratch m: the light table, then per wave eye starts, eye bounces, light starts,
// light bounces, the connection records, the connection walk and the sums.  `cnt64` holds the pass's counters
// ([0, 2) light table info, [2, 4) queue counts, [4, 7) ray totals).
template <class Walk>
int run_pass(Walk &wk, const nrt_bdpt_params &p, const Layout &L, Scene sc, const Scratch &m, unsigned long long *info,
             unsigned long long *ctr, unsigned long long *totals, float *d_accum, const Out *out, nrt_bdpt_result *res,
             cudaStream_t s, const char *who) {
  const TileMap tm = L.tm;
  const unsigned long long total_slots = L.total_slots, cap = L.cap;
  const uint32_t B = L.B, stride = L.stride, mc = L.mc, nf = L.n_lights_max;
  // light table (the sort swaps its key and id buffers)
  uint32_t *l_ids = m.l_ids, *l_keys = m.l_keys, *l_ids_tmp = m.l_flags, *l_keys_tmp = m.l_keys_tmp;
  float *l_cdf = reinterpret_cast<float *>(m.l_offs);  // the offsets are dead once the ids are compacted
  sc.cdf = l_cdf;
  sc.light_ids = l_ids;
  sc.total_area = m.l_total;
  sc.n_lights = 0;

  PassClock clock(res != nullptr);
  if (const int rc = clock.start(s)) return rc;
  uint32_t launches = 0, trav_launches = 0;
  NRT_CUDA(cudaMemsetAsync(info, 0, 2 * sizeof(unsigned long long), s));
  NRT_CUDA(cudaMemsetAsync(totals, 0, 3 * sizeof(unsigned long long), s));
  if (const int rc = wk.light_candidates(sc, nf, m.l_flags, m.l_offs, l_ids, l_keys, m.l_scratch, info, s)) return rc;
  launches += 2 + scan_launches(nf);
  unsigned long long hinfo[2] = {0, 0};
  NRT_CUDA(cudaMemcpyAsync(hinfo, info, sizeof(hinfo), cudaMemcpyDeviceToHost, s));
  NRT_CUDA(cudaStreamSynchronize(s));
  if (hinfo[1]) {
    set_error(std::string(who) + ": a material id is not below n_materials");
    return NRT_ERR_INVALID;
  }
  if (hinfo[0] == 0) {
    set_error(std::string(who) + ": the mesh has no emissive face (max(Le) > 0.001)");
    return NRT_ERR_INVALID;
  }
  sc.n_lights = (uint32_t)hinfo[0];
  light_total_kernel<<<1, 1, 0, s>>>(l_keys, sc.n_lights, m.l_total);
  NRT_CUDA(cudaGetLastError());
  // (area, face) order: a stable sort on the area bits of the face-ordered ids (areas are >= 0)
  if (const int rc = radix_sort_pairs(l_keys, l_ids, l_keys_tmp, l_ids_tmp, sc.n_lights, 0, 32, m.l_table, m.l_scratch, s))
    return rc;
  sc.light_ids = l_ids;
  light_cdf_kernel<<<1, 1, 0, s>>>(l_keys, sc.n_lights, m.l_total, l_cdf);
  NRT_CUDA(cudaGetLastError());
  launches += 2 + 8 * (2 + scan_launches(16 * ((sc.n_lights + kSortTile - 1) / kSortTile)));

  // wave scratch
  PathState *st = m.st;
  uint32_t *const *queue = m.queue;
  Subpaths sp;
  sp.stride = stride;

  for (unsigned long long s0 = 0; s0 < total_slots; s0 += cap) {
    const uint32_t count = (uint32_t)std::min<unsigned long long>(cap, total_slots - s0);
    BdptWave w;
    w.tm = tm;
    w.spp_total = p.spp_total;
    for (int k = 0; k < 12; k++) w.cam[k] = p.cam[k];
    w.s0 = s0;
    w.count = count;
    if (out) {
      sp.eye = out->eye + s0 * stride;
      sp.light = out->light + s0 * stride;
      sp.n_eye = out->n_eye + s0;
      sp.n_light = out->n_light + s0;
    } else {
      sp.eye = m.w_eye;
      sp.light = m.w_light;
      sp.n_eye = m.w_ne;
      sp.n_light = m.w_nl;
    }
    wk.wave(s0);
    float *rgb = out ? out->rgb + 3 * s0 : m.w_rgb;
    const unsigned g = (count + 255) / 256;
    for (int eye = 1; eye >= 0; eye--) {
      NRT_CUDA(cudaMemsetAsync(ctr, 0, 2 * sizeof(unsigned long long), s));
      if (eye)
        eye_start_kernel<<<g, 256, 0, s>>>(w, sp, st, queue[0], ctr + 1);
      else
        wk.light_start(sc, count, sp, st, queue[0], ctr + 1, s);
      NRT_CUDA(cudaGetLastError());
      launches++;
      int in = 0;
      for (uint32_t bounce = 0; bounce < B; bounce++) {
        begin_launch_kernel<<<1, 1, 0, s>>>(ctr, totals + (eye ? 0 : 1));
        NRT_CUDA(cudaGetLastError());
        launches++;
        bool empty = false;
        if (const int rc = wk.bounce(sc, sp, st, queue[in], queue[in ^ 1], ctr, count, B, eye, clock, launches,
                                     trav_launches, &empty, s))
          return rc;
        if (empty) break;
        in ^= 1;
      }
    }
    conn_count_kernel<<<(count + 127) / 128, 128, 0, s>>>(sc, B, count, sp, m.cnt);
    NRT_CUDA(cudaGetLastError());
    if (const int rc = exclusive_scan_u32_async(m.cnt, m.offs, count, m.scan_scratch, s)) return rc;
    conn_write_kernel<<<(count + 127) / 128, 128, 0, s>>>(sc, B, count, sp, m.cnt, m.offs, m.conns, m.emit, ctr + 1);
    NRT_CUDA(cudaGetLastError());
    begin_launch_kernel<<<1, 1, 0, s>>>(ctr, totals + 2);
    NRT_CUDA(cudaGetLastError());
    launches += 3 + scan_launches(count);
    if (const int rc = wk.connect(m.conns, sp, ctr, (size_t)count * mc, clock, launches, trav_launches, s)) return rc;
    sample_sum_kernel<<<g, 256, 0, s>>>(count, sp, m.cnt, m.offs, m.conns, m.emit, rgb);
    NRT_CUDA(cudaGetLastError());
    launches++;
    if (!out) {
      pixel_sum_kernel<<<g, 256, 0, s>>>(w, count / p.spp, sp, rgb, d_accum);
      NRT_CUDA(cudaGetLastError());
      launches++;
    }
  }
  if (res) {
    unsigned long long ht[3] = {0, 0, 0};
    if (const int rc = clock.stop(s)) return rc;
    NRT_CUDA(cudaMemcpyAsync(ht, totals, sizeof(ht), cudaMemcpyDeviceToHost, s));
    NRT_CUDA(cudaStreamSynchronize(s));
    float total_ms = 0.0f, span[2];
    if (const int rc = clock.read(&total_ms, span)) return rc;
    res->eye_rays = ht[0];
    res->light_rays = ht[1];
    res->connection_rays = ht[2];
    res->traverse_ms = span[0];
    res->total_ms = total_ms;
    res->launches = launches;
    res->traverse_launches = trav_launches;
  }
  return NRT_OK;
}

int run_bdpt(const nrt_accel *h, const nrt_bdpt_params *pp, float *d_accum, const Out *out, nrt_bdpt_result *res,
             void *stream, const char *who) {
  Accel *a = const_cast<Accel *>(reinterpret_cast<const Accel *>(h));
  if (const int rc = check_params(a, pp, who)) return rc;
  const nrt_bdpt_params p = *pp;
  Layout L;
  if (const int rc = make_layout(p, out != nullptr, a->n_prims, 0, who, L)) return rc;

  NRT_DEVICE(a->device);
  std::lock_guard<std::mutex> lock(a->host_mu);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (const int rc = wait_previous_pass(a, s)) return rc;
  const RecordOnExit pass_done{a->pass_done, s};
  Scratch m;
  if (const int rc = carve_pass_scratch(a, [&](Carver &c) { m = carve_scratch(c, L); })) return rc;
  Scene sc;
  sc.mats = static_cast<const PathMaterial *>(p.d_materials);
  sc.mat_ids = static_cast<const uint32_t *>(p.d_material_ids);
  sc.fv_normals = static_cast<const float *>(p.d_facevarying_normals);
  sc.verts = a->d_verts;
  sc.faces = a->d_faces;
  sc.n_materials = p.n_materials;
  FlatWalk wk{a, p.flags};
  // d_counters: [2, 3] lights, bad id; [48, 49] queue counts; [52..54] ray totals
  return run_pass(wk, p, L, sc, m, pass_counters(a, kWaveCounters), pass_counters(a, kPathCounters),
                  pass_counters(a, kPathTotals), d_accum, out, res, s, who);
}

// ---- the scene pass
// A two-level scene: the light table over {instance, face} pairs, per bounce the scene walk between a packing kernel
// and a stage kernel (the walk takes its ray count from the host: one read-back per walk)
struct SceneWalk {
  const nrt_scene *scene;
  SceneGeo g;
  uint32_t flags;
  uint32_t stride;
  const Out *out;
  Ray36 *rays;  // cap * max_conns records, shared by the bounce and connection walks
  SceneHit32 *hits;
  uint8_t *mask;
  SceneVerts w_sv;  // the render's own instance arrays
  SceneVerts sv;    // the wave's
  unsigned long long h_count;
  int light_candidates(const Scene &sc, uint32_t n, uint32_t *l_flags, uint32_t *l_offs, uint32_t *l_ids,
                       uint32_t *l_keys, uint32_t *l_scratch, unsigned long long *info, cudaStream_t s) {
    const unsigned gf = (n + 255) / 256;
    pair_flags_kernel<<<gf, 256, 0, s>>>(sc, g, n, l_flags, info);
    NRT_CUDA(cudaGetLastError());
    if (const int rc = exclusive_scan_u32_async(l_flags, l_offs, n, l_scratch, s)) return rc;
    pair_compact_kernel<<<gf, 256, 0, s>>>(g, n, l_flags, l_offs, l_ids, l_keys, info);
    NRT_CUDA(cudaGetLastError());
    return NRT_OK;
  }
  void wave(unsigned long long s0) {
    if (out)
      sv = SceneVerts{out->eye_inst + s0 * stride, out->light_inst + s0 * stride, out->light_pair + 2 * s0};
    else
      sv = w_sv;
  }
  void light_start(const Scene &sc, uint32_t count, const Subpaths &sp, PathState *st, uint32_t *queue,
                   unsigned long long *ctr1, cudaStream_t s) {
    scene_light_start_kernel<<<(count + 255) / 256, 256, 0, s>>>(sc, g, count, sp, sv, st, queue, ctr1);
  }
  int read_count(const unsigned long long *d, uint32_t &n, cudaStream_t s) {
    NRT_CUDA(cudaMemcpyAsync(&h_count, d, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    NRT_CUDA(cudaStreamSynchronize(s));
    n = (uint32_t)h_count;
    return NRT_OK;
  }
  int bounce(const Scene &sc, const Subpaths &sp, PathState *st, const uint32_t *q_in, uint32_t *q_out,
             unsigned long long *ctr, uint32_t, uint32_t B, int eye, PassClock &tm, uint32_t &launches,
             uint32_t &trav_launches, bool *empty, cudaStream_t s) {
    uint32_t n = 0;
    if (const int rc = read_count(ctr, n, s)) return rc;
    *empty = n == 0;
    if (n == 0) return NRT_OK;
    const unsigned blocks = (n + 255) / 256;
    scene_bounce_rays_kernel<<<blocks, 256, 0, s>>>(BounceRays{q_in, st}, n, rays);
    NRT_CUDA(cudaGetLastError());
    if (const int rc = tm.begin(s)) return rc;
    if (const int rc = scene_walk(scene, rays, n, hits, mask, flags, s)) return rc;
    if (const int rc = tm.end(s)) return rc;
    scene_bounce_kernel<<<blocks, 256, 0, s>>>(sc, g, sp, eye ? sv.eye_inst : sv.light_inst, st, q_in, n, hits, mask,
                                               q_out, ctr + 1, B, eye);
    NRT_CUDA(cudaGetLastError());
    launches += 3;
    trav_launches++;
    return NRT_OK;
  }
  int connect(Conn *conns, const Subpaths &sp, unsigned long long *ctr, size_t, PassClock &tm, uint32_t &launches,
              uint32_t &trav_launches, cudaStream_t s) {
    uint32_t n = 0;
    if (const int rc = read_count(ctr, n, s)) return rc;
    if (n == 0) return NRT_OK;
    const unsigned blocks = (n + 255) / 256;
    scene_conn_rays_kernel<<<blocks, 256, 0, s>>>(g, conns, n, sp, sv, rays);
    NRT_CUDA(cudaGetLastError());
    if (const int rc = tm.begin(s)) return rc;
    if (const int rc = scene_walk(scene, rays, n, hits, mask, flags, s)) return rc;
    if (const int rc = tm.end(s)) return rc;
    scene_conn_g_kernel<<<blocks, 256, 0, s>>>(conns, n, sp, rays, hits, mask);
    NRT_CUDA(cudaGetLastError());
    launches += 3;
    trav_launches++;
    return NRT_OK;
  }
};

int run_scene_bdpt(const nrt_scene *scn, const nrt_bdpt_params *pp, const nrt_scene_shading *shading, float *d_accum,
                   const Out *out, nrt_bdpt_result *res, void *stream, const char *who) {
  if (!scn || !pp) return refuse(who, "NULL argument");
  if (!shading) return refuse(who, "NULL shading array (one nrt_scene_shading per instance)");
  const nrt_bdpt_params p = *pp;
  if (!p.d_materials || p.n_materials == 0) return refuse(who, "materials are required");
  if (p.d_material_ids || p.d_facevarying_normals)
    return refuse(who,
                  "material ids and face-varying normals are given per instance (nrt_scene_shading), not in the params");
  if (const int rc = check_common(p, who)) return rc;
  const SceneView view = scene_view(scn);
  std::vector<uint32_t> face_offs(view.n + 1, 0u);
  for (uint32_t i = 0; i < view.n; i++) {
    if (view.n_faces[i] == 0) return refuse(who, "triangle instances only");
    if (!shading[i].d_material_ids || !shading[i].d_facevarying_normals)
      return refuse(who, "instance " + std::to_string(i) + " has no material ids or face-varying normals");
    const uint64_t next = (uint64_t)face_offs[i] + view.n_faces[i];
    if (next > 0xFFFFFFFFull) return refuse(who, "more than 2^32 - 1 {instance, face} pairs");
    face_offs[i + 1] = (uint32_t)next;
  }
  const uint32_t n_pairs = face_offs[view.n];
  Layout L;
  const size_t per_conn = sizeof(Ray36) + sizeof(SceneHit32) + 1;
  const size_t extra = (out ? 0 : 2 * (size_t)(p.max_bounces + 1) * 4 + 8) + (size_t)max_conns(p.max_bounces) * per_conn;
  if (const int rc = make_layout(p, out != nullptr, n_pairs, extra, who, L)) return rc;
  const size_t n_rec = (size_t)L.cap * L.mc;

  NRT_DEVICE(view.device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  SceneWalk wk;
  wk.scene = scn;
  wk.flags = p.flags;
  wk.stride = L.stride;
  wk.out = out;
  wk.w_sv = SceneVerts{nullptr, nullptr, nullptr};
  Scratch m;
  SceneShadingDev *d_shading = nullptr;
  uint32_t *d_offs = nullptr;
  unsigned long long *c = nullptr;
  CallMemory mem(s);
  if (const int rc = mem.alloc([&](Carver &k) {
        m = carve_scratch(k, L);
        wk.rays = k.take<Ray36>(n_rec);
        wk.hits = k.take<SceneHit32>(n_rec);
        wk.mask = k.take<uint8_t>(n_rec);
        if (!out) {
          wk.w_sv.eye_inst = k.take<uint32_t>(L.cap * L.stride);
          wk.w_sv.light_inst = k.take<uint32_t>(L.cap * L.stride);
          wk.w_sv.light_pair = k.take<uint32_t>(2 * L.cap);
        }
        d_shading = k.take<SceneShadingDev>(view.n);
        d_offs = k.take<uint32_t>((size_t)view.n + 1);
        c = k.take<unsigned long long>(8);
      }))
    return rc;
  NRT_CUDA(cudaMemcpyAsync(d_shading, shading, sizeof(SceneShadingDev) * view.n, cudaMemcpyHostToDevice, s));
  NRT_CUDA(cudaMemcpyAsync(d_offs, face_offs.data(), 4 * face_offs.size(), cudaMemcpyHostToDevice, s));
  wk.g = SceneGeo{static_cast<const InstanceDev *>(view.inst), view.state76, d_shading, d_offs, view.n};
  Scene sc{};
  sc.mats = static_cast<const PathMaterial *>(p.d_materials);
  sc.n_materials = p.n_materials;
  // c: [0, 1] lights, bad id; [2, 3] queue counts; [4..6] ray totals
  if (const int rc = run_pass(wk, p, L, sc, m, c, c + 2, c + 4, d_accum, out, res, s, who)) return rc;
  return mem.drain();
}

}  // namespace
}  // namespace nrt

using namespace nrt;

extern "C" int nrt_render_bdpt_device(const nrt_accel *h, const nrt_bdpt_params *p, float *d_accum_rgb,
                                      nrt_bdpt_result *res, void *stream) {
  if (!d_accum_rgb) {
    set_error("nrt_render_bdpt_device: NULL argument");
    return NRT_ERR_INVALID;
  }
  return run_bdpt(h, p, d_accum_rgb, nullptr, res, stream, "nrt_render_bdpt_device");
}

extern "C" int nrt_bdpt_export_device(const nrt_accel *h, const nrt_bdpt_params *p, nrt_bdpt_vertex *d_eye,
                                      nrt_bdpt_vertex *d_light, uint32_t *d_n_eye, uint32_t *d_n_light,
                                      float *d_sample_rgb, nrt_bdpt_result *res, void *stream) {
  if (!d_eye || !d_light || !d_n_eye || !d_n_light || !d_sample_rgb) {
    set_error("nrt_bdpt_export_device: NULL argument");
    return NRT_ERR_INVALID;
  }
  const Out out{d_eye, d_light, d_n_eye, d_n_light, d_sample_rgb, nullptr, nullptr, nullptr};
  return run_bdpt(h, p, nullptr, &out, res, stream, "nrt_bdpt_export_device");
}

extern "C" int nrt_scene_render_bdpt_device(const nrt_scene *s, const nrt_bdpt_params *p,
                                            const nrt_scene_shading *shading, float *d_accum_rgb,
                                            nrt_bdpt_result *res, void *stream) {
  if (!d_accum_rgb) {
    set_error("nrt_scene_render_bdpt_device: NULL argument");
    return NRT_ERR_INVALID;
  }
  return run_scene_bdpt(s, p, shading, d_accum_rgb, nullptr, res, stream, "nrt_scene_render_bdpt_device");
}

extern "C" int nrt_scene_bdpt_export_device(const nrt_scene *s, const nrt_bdpt_params *p,
                                            const nrt_scene_shading *shading, nrt_bdpt_vertex *d_eye,
                                            nrt_bdpt_vertex *d_light, uint32_t *d_eye_inst, uint32_t *d_light_inst,
                                            uint32_t *d_light_pair, uint32_t *d_n_eye, uint32_t *d_n_light,
                                            float *d_sample_rgb, nrt_bdpt_result *res, void *stream) {
  if (!d_eye || !d_light || !d_eye_inst || !d_light_inst || !d_light_pair || !d_n_eye || !d_n_light ||
      !d_sample_rgb) {
    set_error("nrt_scene_bdpt_export_device: NULL argument");
    return NRT_ERR_INVALID;
  }
  const Out out{d_eye, d_light, d_n_eye, d_n_light, d_sample_rgb, d_eye_inst, d_light_inst, d_light_pair};
  return run_scene_bdpt(s, p, shading, nullptr, &out, res, stream, "nrt_scene_bdpt_export_device");
}
