// Path-traced lightmaps: the path tracer's bounces started from every covered texel of a UV atlas.  Bounce 0 is the
// texel vertex (wavefront.cuh: lightmap_texel_vertex), a stage kernel that traces nothing and feeds the queues; bounces
// 1 and up are the path pass's radiance launch with the texel slot map (LightmapShadeEpilogue) and its shadow launch.
// What is here: argument checks, the covered-texel compaction (bake.cu: bake_prepare), the wave and bounce loop, and
// the one-bounce entry.
#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/nanort_b200_lightmap.h"
#include "common.cuh"
#include "scan.cuh"
#include "wavefront.cuh"
#include "pass_host.cuh"

namespace nrt {

bool is_triangle_accel(const Accel *a);
int bake_prepare(Accel *a, const void *d_records, uint32_t n, const char *who, cudaStream_t s, uint32_t **list,
                 uint32_t *n_cov, uint32_t *launches);
int launch_traverse_lightmap_radiance(const Accel *a, const LightmapShadeEpilogue &epi,
                                      const unsigned long long *d_count, size_t capacity, const TraceOptions16 &opt,
                                      uint32_t flags, cudaStream_t s);
int launch_traverse_path_shadow(const Accel *a, const PathQueues &q, const unsigned long long *d_count,
                                size_t capacity, float *d_accum, const TraceOptions16 &opt, uint32_t flags,
                                cudaStream_t s);

// the path pass's parameters of a bake: what path_shade_hit and the slot maps read (also the scene bake's,
// scene_bake.cu)
nrt_path_params path_params(const nrt_lightmap_params &lp) {
  nrt_path_params p = {};
  p.width = lp.width;
  p.height = lp.height;
  p.spp = lp.spp;
  p.sample0 = lp.sample0;
  p.seed = lp.seed;
  p.tile_w = 8;
  p.tile_h = 4;
  p.n_shards = 1;
  p.max_bounces = lp.max_bounces;
  p.ray_min_t = lp.ray_min_t;
  p.ray_max_t = lp.ray_max_t;
  p.n_materials = lp.n_materials;
  p.n_emissive = lp.n_emissive;
  p.d_materials = lp.d_materials;
  p.d_material_ids = lp.d_material_ids;
  p.d_emissive_faces = lp.d_emissive_faces;
  p.d_facevarying_normals = lp.d_facevarying_normals;
  p.flags = lp.flags;
  return p;
}

namespace {

// bounce 0 of paths [0, count): continuations to queue `out`, light samples to the shadow queue
__global__ void __launch_bounds__(256)
    texel_vertex_kernel(nrt_path_params p, TexelSlots slots, uint32_t count, const float4 *__restrict__ records,
                        const float *__restrict__ verts, const uint32_t *__restrict__ faces,
                        const float4 *__restrict__ face_n, PathQueues q, int out, float *accum,
                        unsigned long long *counters /* [0] continuations, [1] shadow rays */) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool cont = false, shadow = false;
  float4 co = make_float4(0, 0, 0, 0), cd = co, so = co, sd = co, sc = co;
  if (i < count)
    lightmap_texel_vertex(p, slots, i, records, verts, faces, face_n, q.weight + i, accum, cont, shadow, co, cd, so, sd,
                          sc);
  path_append(q, out, counters, cont, shadow, i, co, cd, so, sd, sc);
}

// after each bounce's shadow launch: counters [0] continuations of the bounce, [1] its shadow rays, [3] rays of the
// next radiance launch; totals [0] radiance rays, [1] shadow rays
__global__ void next_bounce_kernel(unsigned long long *counters, unsigned long long *totals) {
  totals[0] += counters[0];
  totals[1] += counters[1];
  counters[3] = counters[0];
  counters[0] = 0;
  counters[1] = 0;
}

int lightmap_check(const Accel *a, const void *d_records, const nrt_lightmap_params *p, const float *d_accum,
                   const char *who) {
  if (!a || !d_records || !p || !d_accum) {
    set_error(std::string(who) + ": NULL argument");
    return NRT_ERR_INVALID;
  }
  if (const int rc = check_lightmap_params(*p, who)) return rc;
  if (p->flags & ~(uint32_t)(NRT_TRAVERSE_ANY_HIT | NRT_TRAVERSE_CPP03_INVERSE)) {
    set_error(std::string(who) + ": flags other than NRT_TRAVERSE_ANY_HIT / NRT_TRAVERSE_CPP03_INVERSE");
    return NRT_ERR_INVALID;
  }
  if (!is_triangle_accel(a)) {
    set_error(std::string(who) + ": the world accel must be a triangle accel");
    return NRT_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(d_records) & 15u) != 0) {
    set_error(std::string(who) + ": the record buffer must be 16-byte aligned");
    return NRT_ERR_INVALID;
  }
  return NRT_OK;
}

}  // namespace
}  // namespace nrt

using namespace nrt;

extern "C" int nrt_bake_lightmap_device(const nrt_accel *world, const void *d_records_16B,
                                        const nrt_lightmap_params *pp, float *d_accum_rgb, nrt_lightmap_result *res,
                                        void *stream) {
  static const char *who = "nrt_bake_lightmap_device";
  Accel *a = const_cast<Accel *>(reinterpret_cast<const Accel *>(world));
  if (const int rc = lightmap_check(a, d_records_16B, pp, d_accum_rgb, who)) return rc;
  const nrt_lightmap_params lp = *pp;
  const nrt_path_params p = path_params(lp);
  const uint32_t n = lp.width * lp.height;
  NRT_DEVICE(a->device);
  // the compacted list and the queues (d_wave) and d_counters[2..3], [48..53] are the accel's pass scratch
  std::lock_guard<std::mutex> lock(a->host_mu);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (const int rc = wait_previous_pass(a, s)) return rc;
  const RecordOnExit pass_done{a->pass_done, s};
  // the paths of one wave: at most 8 Mi, as in the path pass
  const unsigned long long kMaxWave = 8ull << 20;
  const unsigned long long cap_max = std::min<unsigned long long>(kMaxWave, (unsigned long long)n * lp.spp);
  // the compaction's scratch (bake_prepare), then the queues
  PathQueues q;
  const auto scratch = [&](Carver &c, unsigned long long cap) {
    carve_compaction(c, n);
    q = carve_path_queues(c, cap);
  };
  if (const int rc = carve_pass_scratch(a, [&](Carver &c) { scratch(c, cap_max); })) return rc;
  uint32_t launches = a->d_face_n ? 0u : 1u;
  if (const int rc = ensure_face_normals(a, s)) return rc;

  PassClock clock(res != nullptr);
  if (const int rc = clock.start(s)) return rc;
  uint32_t *list = nullptr, n_cov = 0;
  if (const int rc = bake_prepare(a, d_records_16B, n, who, s, &list, &n_cov, &launches)) return rc;
  const unsigned long long total = (unsigned long long)n_cov * lp.spp;
  const unsigned long long cap = std::min(total, kMaxWave);
  Carver c(a->d_wave);
  scratch(c, cap);
  unsigned long long *ctr = pass_counters(a, kPathCounters);   // [48..51]
  unsigned long long *totals = pass_counters(a, kPathTotals);  // [52..53]
  NRT_CUDA(cudaMemsetAsync(ctr, 0, 6 * sizeof(unsigned long long), s));
  const TraceOptions16 opt = default_trace_options();
  const float4 *records = static_cast<const float4 *>(d_records_16B);
  const FastDiv n_cov_div(n_cov);
  uint32_t trav_launches = 0;
  for (unsigned long long s0 = 0; s0 < total; s0 += cap) {
    const uint32_t count = (uint32_t)std::min(cap, total - s0);
    const TexelSlots slots{list, n_cov_div, (uint32_t)(s0 % n_cov), (uint32_t)(s0 / n_cov)};
    // bounce 0: the texel vertex writes continuations to queue 1; bounce b >= 1 reads queue b & 1
    texel_vertex_kernel<<<(count + 255) / 256, 256, 0, s>>>(p, slots, count, records, a->d_verts, a->d_faces,
                                                             a->d_face_n, q, 1, d_accum_rgb, ctr);
    NRT_CUDA(cudaGetLastError());
    launches++;
    for (uint32_t b = 0; b < lp.max_bounces; b++) {
      if (const int rc = clock.begin(s)) return rc;
      if (b > 0) {
        const LightmapShadeEpilogue epi{p, slots, (int)(b & 1u), b, q, a->d_verts, a->d_faces, d_accum_rgb, ctr};
        if (const int rc = launch_traverse_lightmap_radiance(a, epi, ctr + 3, count, opt, lp.flags, s)) return rc;
        launches++;
        trav_launches++;
      }
      if (const int rc = launch_traverse_path_shadow(a, q, ctr + 1, count, d_accum_rgb, opt, lp.flags, s)) return rc;
      launches++;
      trav_launches++;
      if (const int rc = clock.end(s)) return rc;
      next_bounce_kernel<<<1, 1, 0, s>>>(ctr, totals);
      NRT_CUDA(cudaGetLastError());
      launches++;
    }
  }
  if (res) {
    if (const int rc = clock.stop(s)) return rc;
    unsigned long long ht[2] = {0, 0};
    NRT_CUDA(cudaMemcpyAsync(ht, totals, sizeof(ht), cudaMemcpyDeviceToHost, s));
    NRT_CUDA(cudaStreamSynchronize(s));
    float total_ms = 0.0f, span[2];
    if (const int rc = clock.read(&total_ms, span)) return rc;
    res->texels = n_cov;
    res->paths = total;
    res->radiance_rays = ht[0];
    res->shadow_rays = ht[1];
    res->traverse_ms = span[0];
    res->total_ms = total_ms;
    res->launches = launches;
    res->traverse_launches = trav_launches;
  }
  return NRT_OK;
}

// One bounce of the bake on caller-owned queues (nrt_path_bounce_device's unit, with the texel slot map)
extern "C" int nrt_bake_lightmap_bounce_device(const nrt_accel *world, const void *d_records_16B,
                                               const nrt_lightmap_params *pp, uint32_t bounce, uint64_t n_rays,
                                               const void *d_org_tmin, const void *d_dir_tmax,
                                               const uint32_t *d_path_id, void *d_weight, void *d_out_org_tmin,
                                               void *d_out_dir_tmax, uint32_t *d_out_path_id, void *d_sh_org_tmin,
                                               void *d_sh_dir_tmax, void *d_sh_contrib_pix, float *d_accum_rgb,
                                               uint64_t *n_continue, uint64_t *n_shadow, int skip_shadow_pass,
                                               void *stream) {
  static const char *who = "nrt_bake_lightmap_bounce_device";
  Accel *a = const_cast<Accel *>(reinterpret_cast<const Accel *>(world));
  if (const int rc = lightmap_check(a, d_records_16B, pp, d_accum_rgb, who)) return rc;
  if (!d_weight || !d_out_org_tmin || !d_out_dir_tmax || !d_out_path_id || !d_sh_org_tmin || !d_sh_dir_tmax ||
      !d_sh_contrib_pix || (bounce > 0 && (!d_org_tmin || !d_dir_tmax || !d_path_id))) {
    set_error(std::string(who) + ": NULL argument");
    return NRT_ERR_INVALID;
  }
  if (n_rays >= (1ull << 32)) {
    set_error(std::string(who) + ": n_rays must be below 2^32");
    return NRT_ERR_INVALID;
  }
  if (n_continue) *n_continue = 0;
  if (n_shadow) *n_shadow = 0;
  if (n_rays == 0) return NRT_OK;
  const nrt_lightmap_params lp = *pp;
  const nrt_path_params p = path_params(lp);
  const uint32_t n = lp.width * lp.height;
  NRT_DEVICE(a->device);
  std::lock_guard<std::mutex> lock(a->host_mu);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (const int rc = wait_previous_pass(a, s)) return rc;
  const RecordOnExit pass_done{a->pass_done, s};
  if (const int rc = carve_pass_scratch(a, [&](Carver &c) { carve_compaction(c, n); })) return rc;
  if (const int rc = ensure_face_normals(a, s)) return rc;
  uint32_t *list = nullptr, n_cov = 0, launches = 0;
  if (const int rc = bake_prepare(a, d_records_16B, n, who, s, &list, &n_cov, &launches)) return rc;
  if (bounce == 0 && n_rays > (uint64_t)n_cov * lp.spp) {
    set_error(std::string(who) + ": bounce 0 of more paths than covered texels x spp");
    return NRT_ERR_INVALID;
  }
  if (n_cov == 0) {
    set_error(std::string(who) + ": the records cover no texel");
    return NRT_ERR_INVALID;
  }
  const PathQueues q = caller_path_queues(d_org_tmin, d_dir_tmax, d_path_id, d_weight, d_out_org_tmin, d_out_dir_tmax,
                                         d_out_path_id, d_sh_org_tmin, d_sh_dir_tmax, d_sh_contrib_pix);
  unsigned long long *ctr = pass_counters(a, kPathCounters);  // [0] cont, [1] shadow, [3] n
  const unsigned long long init[4] = {0ull, 0ull, 0ull, (unsigned long long)n_rays};
  NRT_CUDA(cudaMemcpyAsync(ctr, init, sizeof(init), cudaMemcpyHostToDevice, s));
  const TraceOptions16 opt = default_trace_options();
  const TexelSlots slots{list, FastDiv(n_cov), 0u, 0u};
  if (bounce == 0) {
    texel_vertex_kernel<<<(unsigned)((n_rays + 255) / 256), 256, 0, s>>>(
        p, slots, (uint32_t)n_rays, static_cast<const float4 *>(d_records_16B), a->d_verts, a->d_faces, a->d_face_n, q,
        1, d_accum_rgb, ctr);
    NRT_CUDA(cudaGetLastError());
  } else {
    const LightmapShadeEpilogue epi{p, slots, 0, bounce, q, a->d_verts, a->d_faces, d_accum_rgb, ctr};
    if (const int rc = launch_traverse_lightmap_radiance(a, epi, ctr + 3, (size_t)n_rays, opt, lp.flags, s)) return rc;
  }
  if (!skip_shadow_pass) {
    if (const int rc = launch_traverse_path_shadow(a, q, ctr + 1, (size_t)n_rays, d_accum_rgb, opt, lp.flags, s))
      return rc;
  }
  unsigned long long counts[2] = {0, 0};
  return finish_bounce(ctr, counts, n_continue, n_shadow, s);
}
