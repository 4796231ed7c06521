// Texture-space baking: the reference's uv_raster texel cast (examples/uv_raster/main.cc:687-836) and a cosine AO
// bake from the texels it covers.  The rays of both are generated at fetch by the persistent traversal kernel
// (wavefront.cuh: TexelRays, BakeAoRays); what is here is argument checking, the compaction of covered texels, the
// conformance walk's scatter step and the launch bookkeeping.
#include <algorithm>
#include <mutex>
#include <string>

#include "../../include/nanort_b200_bake.h"
#include "common.cuh"
#include "scan.cuh"
#include "wavefront.cuh"
#include "pass_host.cuh"

namespace nrt {

int launch_traverse_texels(const Accel *a, const TexelRays &rays, size_t n, const TexelStore &store, Hit16 *d_by_ray,
                           uint32_t flags, cudaStream_t s);
int launch_traverse_bake(const Accel *a, const BakeAoRays &rays, size_t n, float *d_accum, unsigned long long *d_occluded,
                         uint32_t flags, cudaStream_t s);

namespace {

// the conformance walk's records, written by ray index, moved to their (flipped) texels with their AOVs
__global__ void __launch_bounds__(256)
    scatter_texels_kernel(const Hit16 *__restrict__ by_ray, uint32_t n, TexelRays rays, TexelStore store) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = i < n;
  Hit16 h = {0.0f, 0.0f, 1.0e30f, 0xFFFFFFFFu};
  uint32_t texel = 0;
  if (active) {
    h = by_ray[i];
    texel = rays.dest(i % rays.width.d, i / rays.width.d);
  }
  store(active, texel, h.t, h.u, h.v, h.prim_id, 1.0e30f);
}

// 1 per covered texel; a prim_id that is neither a miss nor a face of the world accel sets info[1]
__global__ void __launch_bounds__(256)
    covered_flags_kernel(const Hit16 *__restrict__ rec, uint32_t n, uint32_t n_prims, uint32_t *__restrict__ flags,
                         unsigned long long *info) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t p = rec[i].prim_id;
  flags[i] = p != 0xFFFFFFFFu ? 1u : 0u;
  if (p != 0xFFFFFFFFu && p >= n_prims) info[1] = 1ull;
}

// stable compaction: covered texel i goes to list[offs[i]]; info[0] = the covered count
__global__ void __launch_bounds__(256)
    compact_texels_kernel(const Hit16 *__restrict__ rec, uint32_t n, const uint32_t *__restrict__ offs,
                          uint32_t *__restrict__ list, unsigned long long *info) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool covered = rec[i].prim_id != 0xFFFFFFFFu;
  if (covered) list[offs[i]] = i;
  if (i == n - 1) info[0] = (unsigned long long)offs[i] + (covered ? 1ull : 0ull);
}

// the bake's AO rays of one launch as nanort::Ray records, through the traversal's own loader
__global__ void __launch_bounds__(256) bake_rays_kernel(BakeAoRays rays, uint32_t n, Ray36 *__restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Ray36 r;
  uint32_t texel;
  rays.load(i, r.org[0], r.org[1], r.org[2], r.dir[0], r.dir[1], r.dir[2], r.min_t, r.max_t, &texel);
  r.type = 0;
  out[i] = r;
}

// kernels exclusive_scan_u32_async launches for n items
uint32_t scan_launches(uint32_t n) {
  const uint32_t tiles = (n + kScanTile - 1) / kScanTile;
  return n == 0 ? 0u : tiles > 1 ? 2u + scan_launches(tiles) : 1u;
}

}  // namespace

bool is_triangle_accel(const Accel *a) {
  return a->prim_kind == 0 && !a->d_prim_boxes && a->d_faces && a->d_verts && a->d_pair && a->d_tris_cm;
}

// The covered-texel compaction of n records: flags, then offsets, the list of covered texels and the scan's scratch.
// The flat bakes keep it at the start of the accel's pass scratch, the scene bakes in their call's memory.
Compaction carve_compaction(Carver &c, uint32_t n) {
  Compaction r;
  r.offs = c.take<uint32_t>(n);
  r.list = c.take<uint32_t>(n);
  r.scratch = c.take<uint32_t>(scan_scratch_words(n));
  return r;
}

// Compacts the covered texels of the n records into `list` and reads their count back, under the world accel's pass
// ordering, which the caller holds; d_wave starts with carve_compaction(n).  Refuses (after the compaction's launches,
// before any traversal) records whose prim_id is neither a miss nor a face of `a`.  The AO bake and the lightmap bake
// (lightmap.cu) start here.
int bake_prepare(Accel *a, const void *d_records, uint32_t n, const char *who, cudaStream_t s, uint32_t **list,
                 uint32_t *n_cov, uint32_t *launches) {
  Carver c(a->d_wave);
  const Compaction cp = carve_compaction(c, n);
  uint32_t *offs = cp.offs, *scratch = cp.scratch;
  *list = cp.list;
  unsigned long long *info = pass_counters(a, kWaveCounters);  // [2] covered, [3] bad record
  const Hit16 *rec = static_cast<const Hit16 *>(d_records);
  NRT_CUDA(cudaMemsetAsync(info, 0, 2 * sizeof(unsigned long long), s));
  covered_flags_kernel<<<(n + 255) / 256, 256, 0, s>>>(rec, n, a->n_prims, offs, info);
  NRT_CUDA(cudaGetLastError());
  if (const int rc = exclusive_scan_u32_async(offs, offs, n, scratch, s)) return rc;
  compact_texels_kernel<<<(n + 255) / 256, 256, 0, s>>>(rec, n, offs, *list, info);
  NRT_CUDA(cudaGetLastError());
  *launches += 2 + scan_launches(n);
  unsigned long long h[2] = {0, 0};
  NRT_CUDA(cudaMemcpyAsync(h, info, sizeof(h), cudaMemcpyDeviceToHost, s));
  NRT_CUDA(cudaStreamSynchronize(s));
  if (h[1]) {
    set_error(std::string(who) + ": a record's prim_id is not a face of the world accel");
    return NRT_ERR_INVALID;
  }
  *n_cov = (uint32_t)h[0];
  return NRT_OK;
}

}  // namespace nrt

using namespace nrt;

extern "C" int nrt_uv_raster_device(const nrt_accel *uv_h, const nrt_accel *world_h, const nrt_uv_raster_params *pp,
                                    void *d_records_16B, float *d_position_3f, float *d_normal_3f,
                                    const float *d_facevarying_normals, uint64_t *n_covered, void *stream) {
  if (!uv_h || !pp || !d_records_16B) {
    set_error("nrt_uv_raster_device: NULL argument");
    return NRT_ERR_INVALID;
  }
  Accel *a = const_cast<Accel *>(reinterpret_cast<const Accel *>(uv_h));
  const Accel *world = reinterpret_cast<const Accel *>(world_h);
  const nrt_uv_raster_params p = *pp;
  const uint64_t n = (uint64_t)p.width * p.height;
  if (n == 0 || n > kMaxTexels) {
    set_error("nrt_uv_raster_device: width * height must lie in [1, 2^31]");
    return NRT_ERR_INVALID;
  }
  if (p.flags & ~(uint32_t)(NRT_TRAVERSE_CONFORMANCE | NRT_TRAVERSE_CPP03_INVERSE)) {
    set_error("nrt_uv_raster_device: flags other than NRT_TRAVERSE_CONFORMANCE / NRT_TRAVERSE_CPP03_INVERSE");
    return NRT_ERR_INVALID;
  }
  if (!is_triangle_accel(a) || (world && !is_triangle_accel(world))) {
    set_error("nrt_uv_raster_device: the UV and world accels must be triangle accels");
    return NRT_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(d_records_16B) & 15u) != 0) {
    set_error("nrt_uv_raster_device: the record buffer must be 16-byte aligned");
    return NRT_ERR_INVALID;
  }
  if ((d_position_3f || d_normal_3f) && !world) {
    set_error("nrt_uv_raster_device: position and normal AOVs need the world accel");
    return NRT_ERR_INVALID;
  }
  if (d_normal_3f && !d_facevarying_normals) {
    set_error("nrt_uv_raster_device: the normal AOV needs face-varying normals");
    return NRT_ERR_INVALID;
  }
  if (world && (world->n_prims != a->n_prims || world->device != a->device)) {
    set_error("nrt_uv_raster_device: the world accel must have the UV accel's face count, on the same device");
    return NRT_ERR_INVALID;
  }
  NRT_DEVICE(a->device);
  // the covered counter (d_counters[2]) and the conformance walk's records (d_wave) are the accel's pass scratch
  std::lock_guard<std::mutex> lock(a->host_mu);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (const int rc = wait_previous_pass(a, s)) return rc;
  const RecordOnExit pass_done{a->pass_done, s};
  const bool conf = (p.flags & NRT_TRAVERSE_CONFORMANCE) != 0;
  if (conf) {
    if (const int rc = grow_wave(a, (size_t)n * sizeof(Hit16))) return rc;
  }
  unsigned long long *covered = pass_counters(a, kWaveCounters);
  NRT_CUDA(cudaMemsetAsync(covered, 0, sizeof(unsigned long long), s));

  TexelRays rays;
  rays.width = FastDiv(p.width);
  rays.height = p.height;
  rays.flip_x = p.flip_x ? 1u : 0u;
  rays.flip_y = p.flip_y ? 1u : 0u;
  rays.r0 = p.uv_region[0];
  rays.r2 = p.uv_region[2];
  rays.usize = p.uv_region[1] - p.uv_region[0];
  rays.vsize = p.uv_region[3] - p.uv_region[2];
  rays.off0 = p.texel_offset[0];
  rays.off1 = p.texel_offset[1];
  rays.fw = (float)p.width;
  rays.fh = (float)p.height;
  const bool aov = d_position_3f || d_normal_3f;
  const TexelStore store{static_cast<Hit16 *>(d_records_16B), d_position_3f, d_normal_3f,
                         aov ? world->d_verts : nullptr,   aov ? world->d_faces : nullptr,
                         d_facevarying_normals,            covered};
  Hit16 *by_ray = conf ? static_cast<Hit16 *>(a->d_wave) : nullptr;
  if (const int rc = launch_traverse_texels(a, rays, (size_t)n, store, by_ray, p.flags, s)) return rc;
  if (conf) {
    scatter_texels_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(by_ray, (uint32_t)n, rays, store);
    NRT_CUDA(cudaGetLastError());
  }
  if (n_covered) {
    unsigned long long c = 0;
    NRT_CUDA(cudaMemcpyAsync(&c, covered, sizeof(c), cudaMemcpyDeviceToHost, s));
    NRT_CUDA(cudaStreamSynchronize(s));
    *n_covered = c;
  }
  return NRT_OK;
}

static int bake_check(const Accel *a, const void *d_records, const nrt_bake_params *p, const char *who) {
  if (!a || !d_records || !p) {
    set_error(std::string(who) + ": NULL argument");
    return NRT_ERR_INVALID;
  }
  if (const int rc = check_bake_params(*p, who)) return rc;
  if (p->flags & ~(uint32_t)(NRT_TRAVERSE_ANY_HIT | NRT_TRAVERSE_CPP03_INVERSE)) {
    set_error(std::string(who) + ": flags other than NRT_TRAVERSE_ANY_HIT / NRT_TRAVERSE_CPP03_INVERSE "
                                 "(the conformance walk is not offered: export the rays and trace them with it)");
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

static BakeAoRays bake_rays(const Accel *a, const void *d_records, const nrt_bake_params &p, const uint32_t *list,
                            uint32_t n_cov) {
  BakeAoRays r;
  r.texels = list;
  r.records = static_cast<const float4 *>(d_records);
  r.verts = a->d_verts;
  r.faces = a->d_faces;
  r.face_n = a->d_face_n;
  r.fv_normals = static_cast<const float *>(p.d_facevarying_normals);
  r.n_cov = FastDiv(n_cov);
  r.sample0 = p.sample0;
  r.seed = p.seed;
  r.min_t = p.ao_min_t;
  r.max_t = p.ao_max_t;
  return r;
}

// dump != nullptr: write the rays (capacity records) instead of tracing them
static int run_bake(const nrt_accel *h, const void *d_records, const nrt_bake_params *pp, float *d_accum,
                    nrt_bake_result *res, Ray36 *dump, uint64_t capacity, uint64_t *n_rays, void *stream,
                    const char *who) {
  Accel *a = const_cast<Accel *>(reinterpret_cast<const Accel *>(h));
  if (const int rc = bake_check(a, d_records, pp, who)) return rc;
  if (!dump && !d_accum) {
    set_error(std::string(who) + ": NULL argument");
    return NRT_ERR_INVALID;
  }
  const nrt_bake_params p = *pp;
  const uint32_t n = p.width * p.height;
  NRT_DEVICE(a->device);
  // the compacted list (d_wave) and the counters d_counters[2..4] are the accel's pass scratch, as in run_ao_pass
  std::lock_guard<std::mutex> lock(a->host_mu);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (const int rc = wait_previous_pass(a, s)) return rc;
  const RecordOnExit pass_done{a->pass_done, s};
  if (const int rc = carve_pass_scratch(a, [&](Carver &c) { carve_compaction(c, n); })) return rc;
  uint32_t launches = a->d_face_n ? 0u : 1u;
  if (const int rc = ensure_face_normals(a, s)) return rc;

  PassClock clock(res != nullptr);
  if (const int rc = clock.start(s)) return rc;
  uint32_t *list = nullptr, n_cov = 0;
  if (const int rc = bake_prepare(a, d_records, n, who, s, &list, &n_cov, &launches)) return rc;
  const uint64_t total = (uint64_t)n_cov * p.spp;
  if (n_rays) *n_rays = total;
  if (dump && total > capacity) {
    set_error(std::string(who) + ": the ray buffer holds fewer records than covered texels x spp");
    return NRT_ERR_INVALID;
  }
  unsigned long long *occluded = pass_counters(a, kPassTotals);
  NRT_CUDA(cudaMemsetAsync(occluded, 0, sizeof(unsigned long long), s));
  uint32_t trav_launches = 0;
  if (n_cov > 0) {
    // whole samples per launch, so that a launch's slot indices fit the loader's 32-bit FastDiv
    const uint32_t per_launch = 0xFFFFFFFFu / n_cov;
    BakeAoRays rays = bake_rays(a, d_records, p, list, n_cov);
    for (uint32_t s0 = 0; s0 < p.spp; s0 += std::min(per_launch, p.spp - s0)) {
      const uint32_t count = std::min(per_launch, p.spp - s0) * n_cov;
      rays.sample0 = p.sample0 + s0;
      if (dump) {
        bake_rays_kernel<<<(count + 255) / 256, 256, 0, s>>>(rays, count, dump + (size_t)s0 * n_cov);
        NRT_CUDA(cudaGetLastError());
        launches++;
        continue;
      }
      if (const int rc = clock.begin(s)) return rc;
      if (const int rc = launch_traverse_bake(a, rays, count, d_accum, occluded, p.flags, s)) return rc;
      if (const int rc = clock.end(s)) return rc;
      launches++;
      trav_launches++;
    }
  }
  if (res) {
    unsigned long long hits = 0;
    if (const int rc = clock.stop(s)) return rc;
    NRT_CUDA(cudaMemcpyAsync(&hits, occluded, sizeof(hits), cudaMemcpyDeviceToHost, s));
    NRT_CUDA(cudaStreamSynchronize(s));
    float total_ms = 0.0f, span[2];
    if (const int rc = clock.read(&total_ms, span)) return rc;
    res->texels = n_cov;
    res->ao_rays = total;
    res->ao_hits = hits;
    res->traverse_ms = span[0];
    res->total_ms = total_ms;
    res->launches = launches;
    res->traverse_launches = trav_launches;
  }
  return NRT_OK;
}

extern "C" int nrt_bake_ao_device(const nrt_accel *world, const void *d_records_16B, const nrt_bake_params *p,
                                  float *d_accum, nrt_bake_result *res, void *stream) {
  return run_bake(world, d_records_16B, p, d_accum, res, nullptr, 0, nullptr, stream, "nrt_bake_ao_device");
}

extern "C" int nrt_bake_ao_rays_device(const nrt_accel *world, const void *d_records_16B, const nrt_bake_params *p,
                                       void *d_rays_36B, uint64_t capacity, uint64_t *n_rays, void *stream) {
  if (!d_rays_36B) {
    set_error("nrt_bake_ao_rays_device: NULL argument");
    return NRT_ERR_INVALID;
  }
  return run_bake(world, d_records_16B, p, nullptr, nullptr, static_cast<Ray36 *>(d_rays_36B), capacity, n_rays,
                  stream, "nrt_bake_ao_rays_device");
}
