// The reference's bidirectional path tracer (examples/bidir_path_tracer/main.cc) as a wavefront pass.  Per wave of
// whole tiles: eye starts, max_bounces eye bounces, light starts, max_bounces light bounces, the connection records
// (count, scan, write), one traversal launch over all calcG rays, then the per-sample and per-pixel sums.  The bounce
// and connection rays are traced by the persistent traversal kernel with the retire steps of wavefront.cuh
// (bd::BounceEpilogue, bd::ConnEpilogue) or, under NRT_TRAVERSE_CONFORMANCE, by the reference-order walk with the same
// retire steps.  What is here: argument checks, the light table, the stage kernels and the launch bookkeeping.
#include <algorithm>
#include <mutex>
#include <string>

#include "../../include/nanort_b200_bdpt.h"
#include "common.cuh"
#include "radix_sort.cuh"
#include "scan.cuh"
#include "wavefront.cuh"

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
// flags[i] = face i emits (max(Le) > kEps); info[1] = some material id is out of range
__global__ void __launch_bounds__(256)
    light_flags_kernel(Scene sc, uint32_t n, uint32_t *__restrict__ flags, unsigned long long *info) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t id = sc.mat_ids[i];
  if (id >= sc.n_materials) {
    info[1] = 1ull;
    flags[i] = 0u;
    return;
  }
  const float *le = sc.mats[id].emission;
  const float mx = le[0] < (le[1] < le[2] ? le[2] : le[1]) ? (le[1] < le[2] ? le[2] : le[1]) : le[0];  // std::max
  flags[i] = mx <= kEps ? 0u : 1u;
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
    const float area = 0.5f * length(cross(sub(v[2], v[0]), sub(v[1], v[0])));
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

// lightSubpath's start (main.cc:1045-1075) for every slot whose eye subpath has a vertex beyond the lens
__global__ void __launch_bounds__(256)
    light_start_kernel(Scene sc, uint32_t count_slots, Subpaths sp, PathState *__restrict__ st,
                       uint32_t *__restrict__ queue, unsigned long long *count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < count_slots && sp.n_eye[i] > 1u;
  if (live) {
    PathState s = st[i];
    Random rng;
    rng.s[0] = s.rng.x, rng.s[1] = s.rng.y, rng.s[2] = s.rng.z, rng.s[3] = s.rng.w;
    // LightSampler::sample (main.cc:731-765)
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
    const uint32_t *f = sc.faces + 3 * (size_t)light;
    const float *fn = sc.fv_normals + 9 * (size_t)light;
    const float b0 = 1.0f - u1 - u2;
    const float3 pos = add(add(mul(f3(sc.verts + 3 * (size_t)f[0]), b0), mul(f3(sc.verts + 3 * (size_t)f[1]), u1)),
                           mul(f3(sc.verts + 3 * (size_t)f[2]), u2));
    const float3 nrm = add(add(mul(f3(fn), b0), mul(f3(fn + 3), u1)), mul(f3(fn + 6), u2));
    const float pdf_pos = 1.0f / *sc.total_area;
    const float3 le = f3(sc.mats[sc.mat_ids[light]].emission);
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
    s.org_pdf = make_float4(pos.x, pos.y, pos.z, pdf_dir);
    s.dir = make_float4(dir.x, dir.y, dir.z, 0.0f);
    s.beta = make_float4(beta.x, beta.y, beta.z, 0.0f);
    s.rng = make_uint4(rng.s[0], rng.s[1], rng.s[2], rng.s[3]);
    st[i] = s;
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
};

int check_params(const Accel *a, const nrt_bdpt_params *pp, const char *who) {
  auto bad = [&](const char *why) {
    set_error(std::string(who) + ": " + why);
    return NRT_ERR_INVALID;
  };
  if (!a || !pp) return bad("NULL argument");
  const nrt_bdpt_params &p = *pp;
  if (!p.d_materials || !p.d_material_ids || !p.d_facevarying_normals || p.n_materials == 0)
    return bad("materials, material ids and face-varying normals are required");
  if (p.flags & ~(uint32_t)NRT_TRAVERSE_CONFORMANCE)
    return bad("flags other than NRT_TRAVERSE_CONFORMANCE (calcG needs the nearest distance: no ANY_HIT)");
  if (p.width == 0 || p.height == 0 || p.spp == 0 || p.n_shards == 0 || p.shard >= p.n_shards || p.tile_w == 0 ||
      p.tile_h == 0 || (p.tile_w % 8) != 0 || (p.tile_h % 4) != 0)
    return bad("bad image, sample or tile parameters");
  if ((uint64_t)p.sample0 + p.spp > p.spp_total) return bad("sample0 + spp > spp_total");
  if (p.max_bounces == 0 || p.max_bounces > 64) return bad("max_bounces must lie in [1, 64]");
  if (a->prim_kind != 0 || a->d_prim_boxes || !a->d_faces || !a->d_verts || !a->d_pair || !a->d_tris_cm)
    return bad("the accel must be a triangle accel");
  return NRT_OK;
}

int run_bdpt(const nrt_accel *h, const nrt_bdpt_params *pp, float *d_accum, const Out *out, nrt_bdpt_result *res,
             void *stream, const char *who) {
  Accel *a = const_cast<Accel *>(reinterpret_cast<const Accel *>(h));
  if (const int rc = check_params(a, pp, who)) return rc;
  const nrt_bdpt_params p = *pp;
  const TileMap tm{p.width, p.height, p.spp, p.sample0, p.tile_w, p.tile_h, p.shard, p.n_shards, 0u};
  const uint32_t tiles_x = (p.width + p.tile_w - 1) / p.tile_w, tiles_y = (p.height + p.tile_h - 1) / p.tile_h;
  const uint32_t n_tiles = tiles_x * tiles_y;
  const uint32_t my_tiles = n_tiles > p.shard ? (n_tiles - p.shard + p.n_shards - 1) / p.n_shards : 0;
  const unsigned long long per_tile = (unsigned long long)p.tile_w * p.tile_h * p.spp;
  const unsigned long long total_slots = (unsigned long long)my_tiles * per_tile;
  const uint32_t B = p.max_bounces, stride = B + 1, mc = max_conns(B);
  // per slot: state, two subpaths (unless exported), queues, counts, offsets, emission, colour, records
  const size_t per_slot = sizeof(PathState) + (out ? 0 : 2 * (size_t)stride * sizeof(nrt_bdpt_vertex) + 8 + 12) +
                          2 * 4 + 4 + 4 + 12 + (size_t)mc * sizeof(Conn) + 8;
  unsigned long long tiles_per_wave = kWaveBudget / (per_slot * per_tile);
  if (tiles_per_wave == 0) tiles_per_wave = 1;
  const unsigned long long cap = std::min<unsigned long long>(total_slots, tiles_per_wave * per_tile);
  if (cap > 0xFFFFFFFFull / mc) {
    set_error(std::string(who) + ": a tile holds too many samples");
    return NRT_ERR_INVALID;
  }
  const uint32_t nf = a->n_prims;
  const uint32_t sort_tiles = (nf + kSortTile - 1) / kSortTile;
  auto rnd = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t light_bytes = 5 * rnd(4 * (size_t)nf) + rnd(4 * (16 * (size_t)sort_tiles + 1)) +
                             rnd(4 * std::max(scan_scratch_words(nf), scan_scratch_words(16 * sort_tiles))) + rnd(16);
  const size_t wave_bytes = rnd(cap * sizeof(PathState)) +
                            (out ? 0 : 2 * rnd(cap * stride * sizeof(nrt_bdpt_vertex)) + 2 * rnd(cap * 4) + rnd(cap * 12)) +
                            4 * rnd(cap * 4) + rnd(cap * 12) + rnd(cap * mc * sizeof(Conn)) +
                            rnd(scan_scratch_words((uint32_t)cap) * 4);

  NRT_DEVICE(a->device);
  std::lock_guard<std::mutex> lock(a->host_mu);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (const int rc = wait_previous_pass(a, s)) return rc;
  const RecordOnExit pass_done{a->pass_done, s};
  if (const int rc = grow_wave(a, light_bytes + wave_bytes)) return rc;
  char *b = static_cast<char *>(a->d_wave);
  auto take = [&](size_t bytes) {
    char *r = b;
    b += rnd(bytes);
    return r;
  };
  // light table
  uint32_t *l_flags = reinterpret_cast<uint32_t *>(take(4 * (size_t)nf));
  uint32_t *l_offs = reinterpret_cast<uint32_t *>(take(4 * (size_t)nf));
  uint32_t *l_ids = reinterpret_cast<uint32_t *>(take(4 * (size_t)nf));
  uint32_t *l_keys = reinterpret_cast<uint32_t *>(take(4 * (size_t)nf));
  uint32_t *l_ids_tmp = l_flags, *l_keys_tmp = reinterpret_cast<uint32_t *>(take(4 * (size_t)nf));
  uint32_t *l_table = reinterpret_cast<uint32_t *>(take(4 * (16 * (size_t)sort_tiles + 1)));
  uint32_t *l_scratch = reinterpret_cast<uint32_t *>(
      take(4 * std::max(scan_scratch_words(nf), scan_scratch_words(16 * sort_tiles))));
  float *l_cdf = reinterpret_cast<float *>(l_offs);  // the offsets are dead once the ids are compacted
  float *l_total = reinterpret_cast<float *>(take(16));
  unsigned long long *info = reinterpret_cast<unsigned long long *>(a->d_counters) + 2;  // [2] lights, [3] bad id
  unsigned long long *ctr = reinterpret_cast<unsigned long long *>(a->d_counters) + 48;  // [48, 49] queue counts
  unsigned long long *totals = reinterpret_cast<unsigned long long *>(a->d_counters) + 52;  // [52..54]

  Scene sc;
  sc.mats = static_cast<const PathMaterial *>(p.d_materials);
  sc.mat_ids = static_cast<const uint32_t *>(p.d_material_ids);
  sc.fv_normals = static_cast<const float *>(p.d_facevarying_normals);
  sc.verts = a->d_verts;
  sc.faces = a->d_faces;
  sc.cdf = l_cdf;
  sc.light_ids = l_ids;
  sc.total_area = l_total;
  sc.n_materials = p.n_materials;
  sc.n_lights = 0;

  cudaEvent_t e_begin = nullptr, e_end = nullptr;
  std::vector<cudaEvent_t> ev;
  struct Events {  // destroyed on every exit
    std::vector<cudaEvent_t> &v;
    ~Events() {
      for (cudaEvent_t e : v)
        if (e) cudaEventDestroy(e);
    }
  } events{ev};
  if (res) {
    NRT_CUDA(cudaEventCreate(&e_begin));
    ev.push_back(e_begin);
    NRT_CUDA(cudaEventCreate(&e_end));
    ev.push_back(e_end);
    NRT_CUDA(cudaEventRecord(e_begin, s));
  }
  uint32_t launches = 0, trav_launches = 0;
  NRT_CUDA(cudaMemsetAsync(info, 0, 2 * sizeof(unsigned long long), s));
  NRT_CUDA(cudaMemsetAsync(totals, 0, 3 * sizeof(unsigned long long), s));
  const unsigned gf = (nf + 255) / 256;
  light_flags_kernel<<<gf, 256, 0, s>>>(sc, nf, l_flags, info);
  NRT_CUDA(cudaGetLastError());
  if (const int rc = exclusive_scan_u32_async(l_flags, l_offs, nf, l_scratch, s)) return rc;
  light_compact_kernel<<<gf, 256, 0, s>>>(sc, nf, l_flags, l_offs, l_ids, l_keys, info);
  NRT_CUDA(cudaGetLastError());
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
  light_total_kernel<<<1, 1, 0, s>>>(l_keys, sc.n_lights, l_total);
  NRT_CUDA(cudaGetLastError());
  // (area, face) order: a stable sort on the area bits of the face-ordered ids (areas are >= 0)
  if (const int rc = radix_sort_pairs(l_keys, l_ids, l_keys_tmp, l_ids_tmp, sc.n_lights, 0, 32, l_table, l_scratch, s))
    return rc;
  sc.light_ids = l_ids;
  light_cdf_kernel<<<1, 1, 0, s>>>(l_keys, sc.n_lights, l_total, l_cdf);
  NRT_CUDA(cudaGetLastError());
  launches += 2 + 8 * (2 + scan_launches(16 * ((sc.n_lights + kSortTile - 1) / kSortTile)));

  // wave scratch
  PathState *st = reinterpret_cast<PathState *>(take(cap * sizeof(PathState)));
  Subpaths sp;
  sp.stride = stride;
  nrt_bdpt_vertex *w_eye = nullptr, *w_light = nullptr;
  uint32_t *w_ne = nullptr, *w_nl = nullptr;
  float *w_rgb = nullptr;
  if (!out) {
    w_eye = reinterpret_cast<nrt_bdpt_vertex *>(take(cap * stride * sizeof(nrt_bdpt_vertex)));
    w_light = reinterpret_cast<nrt_bdpt_vertex *>(take(cap * stride * sizeof(nrt_bdpt_vertex)));
    w_ne = reinterpret_cast<uint32_t *>(take(cap * 4));
    w_nl = reinterpret_cast<uint32_t *>(take(cap * 4));
    w_rgb = reinterpret_cast<float *>(take(cap * 12));
  }
  uint32_t *queue[2] = {reinterpret_cast<uint32_t *>(take(cap * 4)), reinterpret_cast<uint32_t *>(take(cap * 4))};
  uint32_t *cnt = reinterpret_cast<uint32_t *>(take(cap * 4));
  uint32_t *offs = reinterpret_cast<uint32_t *>(take(cap * 4));
  float3 *emit = reinterpret_cast<float3 *>(take(cap * 12));
  Conn *conns = reinterpret_cast<Conn *>(take(cap * mc * sizeof(Conn)));
  uint32_t *scan_scratch = reinterpret_cast<uint32_t *>(take(scan_scratch_words((uint32_t)cap) * 4));

  const uint32_t flags = p.flags;
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
      sp.eye = w_eye;
      sp.light = w_light;
      sp.n_eye = w_ne;
      sp.n_light = w_nl;
    }
    float *rgb = out ? out->rgb + 3 * s0 : w_rgb;
    const unsigned g = (count + 255) / 256;
    for (int eye = 1; eye >= 0; eye--) {
      NRT_CUDA(cudaMemsetAsync(ctr, 0, 2 * sizeof(unsigned long long), s));
      if (eye)
        eye_start_kernel<<<g, 256, 0, s>>>(w, sp, st, queue[0], ctr + 1);
      else
        light_start_kernel<<<g, 256, 0, s>>>(sc, count, sp, st, queue[0], ctr + 1);
      NRT_CUDA(cudaGetLastError());
      launches++;
      int in = 0;
      for (uint32_t bounce = 0; bounce < B; bounce++) {
        begin_launch_kernel<<<1, 1, 0, s>>>(ctr, totals + (eye ? 0 : 1));
        NRT_CUDA(cudaGetLastError());
        cudaEvent_t t0 = nullptr, t1 = nullptr;
        if (res) {
          NRT_CUDA(cudaEventCreate(&t0));
          ev.push_back(t0);
          NRT_CUDA(cudaEventCreate(&t1));
          ev.push_back(t1);
          NRT_CUDA(cudaEventRecord(t0, s));
        }
        const BounceRays rays{queue[in], st};
        const BounceEpilogue epi{sc, sp, st, queue[in], queue[in ^ 1], ctr + 1, B, eye};
        if (const int rc = launch_traverse_bdpt_bounce(a, rays, epi, ctr, count, flags, s)) return rc;
        if (res) NRT_CUDA(cudaEventRecord(t1, s));
        launches += 2;
        trav_launches++;
        in ^= 1;
      }
    }
    conn_count_kernel<<<(count + 127) / 128, 128, 0, s>>>(sc, B, count, sp, cnt);
    NRT_CUDA(cudaGetLastError());
    if (const int rc = exclusive_scan_u32_async(cnt, offs, count, scan_scratch, s)) return rc;
    conn_write_kernel<<<(count + 127) / 128, 128, 0, s>>>(sc, B, count, sp, cnt, offs, conns, emit, ctr + 1);
    NRT_CUDA(cudaGetLastError());
    begin_launch_kernel<<<1, 1, 0, s>>>(ctr, totals + 2);
    NRT_CUDA(cudaGetLastError());
    launches += 3 + scan_launches(count);
    {
      cudaEvent_t t0 = nullptr, t1 = nullptr;
      if (res) {
        NRT_CUDA(cudaEventCreate(&t0));
        ev.push_back(t0);
        NRT_CUDA(cudaEventCreate(&t1));
        ev.push_back(t1);
        NRT_CUDA(cudaEventRecord(t0, s));
      }
      if (const int rc = launch_traverse_bdpt_connect(a, ConnRays{conns, sp}, ConnEpilogue{conns, sp}, ctr,
                                                      (size_t)count * mc, flags, s))
        return rc;
      if (res) NRT_CUDA(cudaEventRecord(t1, s));
      launches++;
      trav_launches++;
    }
    sample_sum_kernel<<<g, 256, 0, s>>>(count, sp, cnt, offs, conns, emit, rgb);
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
    NRT_CUDA(cudaEventRecord(e_end, s));
    NRT_CUDA(cudaMemcpyAsync(ht, totals, sizeof(ht), cudaMemcpyDeviceToHost, s));
    NRT_CUDA(cudaStreamSynchronize(s));
    float tms = 0.0f, total_ms = 0.0f;
    for (size_t i = 2; i + 1 < ev.size(); i += 2) {
      float m = 0.0f;
      NRT_CUDA(cudaEventElapsedTime(&m, ev[i], ev[i + 1]));
      tms += m;
    }
    NRT_CUDA(cudaEventElapsedTime(&total_ms, e_begin, e_end));
    res->eye_rays = ht[0];
    res->light_rays = ht[1];
    res->connection_rays = ht[2];
    res->traverse_ms = tms;
    res->total_ms = total_ms;
    res->launches = launches;
    res->traverse_launches = trav_launches;
  }
  return NRT_OK;
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
  const Out out{d_eye, d_light, d_n_eye, d_n_light, d_sample_rgb};
  return run_bdpt(h, p, nullptr, &out, res, stream, "nrt_bdpt_export_device");
}
