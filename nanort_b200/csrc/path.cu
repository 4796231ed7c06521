// Wavefront form of the reference path tracer's pixel -> sample -> bounce loop
// (examples/path_tracer/main.cc:804-991), diffuse + emissive materials.  The shading of a
// bounce lives in the retire step of the traversal kernel (wavefront.cuh: PathShadeEpilogue,
// ShadowAccumulateEpilogue); this file owns the queues and the bounce loop: per wave and bounce exactly two
// traversal launches (radiance rays, shadow rays) -- the two Traverse calls per bounce of the reference
// (main.cc:854 and :696).
#include <algorithm>
#include <mutex>

#include "common.cuh"
#include "wavefront.cuh"
#include "pass_host.cuh"

namespace nrt {

int launch_traverse_path_radiance(const Accel *a, const PathShadeEpilogue &epi, const unsigned long long *d_count,
                                  size_t capacity, const TraceOptions16 &opt, uint32_t flags, cudaStream_t s);
int launch_traverse_path_shadow(const Accel *a, const PathQueues &q, const unsigned long long *d_count,
                                size_t capacity, float *d_accum, const TraceOptions16 &opt, uint32_t flags,
                                cudaStream_t s);

namespace {

// bounce 0: camera rays (main.cc:809-817, 839-849); every path starts with weight 1
__global__ void __launch_bounds__(256)
    gen_camera_kernel(nrt_path_params p, unsigned long long slot0, uint32_t count, PathQueues q,
                      unsigned long long *counters /* [2] valid camera rays */) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false;
  if (i < count) {
    uint32_t pix, smp;
    q.path_id[0][i] = i;
    q.weight[i] = make_float4(1.0f, 1.0f, 1.0f, 1.0f);  // weight 1, do_emission = true (main.cc:820-824)
    if (!slot_to_pixel(tile_map(p), slot0 + i, pix, smp)) {
      q.org_tmin[0][i] = make_float4(0.f, 0.f, 0.f, 0.f);
      q.dir_tmax[0][i] = make_float4(0.f, 0.f, -1.f, -1.f);  // retires at the root as a miss
    } else {
      valid = true;
      smp += p.sample0;
      const float jx = rand_ps(pix, smp, 0, p.seed), jy = rand_ps(pix, smp, 1, p.seed);
      const float px = (float)(pix % p.width), py = (float)(pix / p.width);
      const float sx = (px + jx) / (float)p.width - 0.5f;
      const float sy = 0.5f - (py + jy) / (float)p.height;
      const float dx = p.cam[3] * sx + p.cam[6] * sy + p.cam[9];
      const float dy = p.cam[4] * sx + p.cam[7] * sy + p.cam[10];
      const float dz = p.cam[5] * sx + p.cam[8] * sy + p.cam[11];
      const float inv = 1.0f / sqrtf(dx * dx + dy * dy + dz * dz);
      q.org_tmin[0][i] = make_float4(p.cam[0], p.cam[1], p.cam[2], p.ray_min_t);
      q.dir_tmax[0][i] = make_float4(dx * inv, dy * inv, dz * inv, p.ray_max_t);
    }
  }
  const unsigned m = __ballot_sync(0xFFFFFFFFu, valid);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(counters + 2, (unsigned long long)__popc(m));
}

// counters: [0] continuation rays written by the bounce just traced, [1] its shadow rays, [2] camera rays,
//           [3] rays of the bounce about to be traced.  totals: [0] radiance, [1] shadow, [2] camera.
__global__ void begin_bounce_kernel(unsigned long long *counters, unsigned long long *totals, uint32_t first_count,
                                    int first) {
  if (first) {
    counters[3] = first_count;
    totals[2] += counters[2];
    totals[0] += counters[2];  // camera rays are radiance Traverse calls too (slots outside the image are not)
  } else {
    counters[3] = counters[0];
    totals[0] += counters[0];
  }
  counters[0] = 0;
  counters[1] = 0;
}
__global__ void end_bounce_kernel(const unsigned long long *counters, unsigned long long *totals) {
  totals[1] += counters[1];
}

}  // namespace

// the camera stage on its own, for the two-level scene's path pass (scene.cu)
void launch_path_camera(const nrt_path_params &p, unsigned long long slot0, uint32_t count, const PathQueues &q,
                        unsigned long long *counters, cudaStream_t s) {
  gen_camera_kernel<<<(count + 255) / 256, 256, 0, s>>>(p, slot0, count, q, counters);
}

}  // namespace nrt

using namespace nrt;

extern "C" int nrt_render_path_device(const nrt_accel *h, const nrt_path_params *pp, float *d_accum_rgb,
                                      nrt_path_result *res, void *stream) {
  if (!h || !pp || !d_accum_rgb) {
    set_error("nrt_render_path_device: NULL argument");
    return NRT_ERR_INVALID;
  }
  Accel *a = const_cast<Accel *>(reinterpret_cast<const Accel *>(h));
  const nrt_path_params p = *pp;
  if (const int rc = check_path_params(p, "nrt_render_path_device")) return rc;
  NRT_DEVICE(a->device);
  // d_wave / d_counters[48..54] are per-accel scratch, shared with AO passes and path bounces: the pass waits on the
  // device for the previous pass on this accel (render.cu)
  std::lock_guard<std::mutex> lock(a->host_mu);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (const int rc = wait_previous_pass(a, s)) return rc;
  const RecordOnExit pass_done{a->pass_done, s};
  const ShardSlots sh = shard_slots(p.width, p.height, p.tile_w, p.tile_h, p.spp, p.shard, p.n_shards);
  const unsigned long long total_slots = sh.total;
  const unsigned long long cap = sh.wave(8ull << 20);
  PathQueues q;
  if (const int rc = carve_pass_scratch(a, [&](Carver &c) { q = carve_path_queues(c, cap); })) return rc;
  unsigned long long *ctr = pass_counters(a, kPathCounters);   // [48..51]
  unsigned long long *totals = pass_counters(a, kPathTotals);  // [52..54]
  NRT_CUDA(cudaMemsetAsync(ctr, 0, 8 * sizeof(unsigned long long), s));

  const TraceOptions16 opt = default_trace_options();
  const uint32_t trav_flags = p.flags & 0xFFFFu;
  PassClock clock(res != nullptr);
  if (const int rc = clock.start(s)) return rc;
  uint32_t launches = 0, trav_launches = 0;
  for (unsigned long long s0 = 0; s0 < total_slots; s0 += cap) {
    const uint32_t count = (uint32_t)std::min<unsigned long long>(cap, total_slots - s0);
    NRT_CUDA(cudaMemsetAsync(ctr, 0, 4 * sizeof(unsigned long long), s));
    gen_camera_kernel<<<(count + 255) / 256, 256, 0, s>>>(p, s0, count, q, ctr);
    launches++;
    int in = 0;
    for (uint32_t b = 0; b < p.max_bounces; b++) {
      begin_bounce_kernel<<<1, 1, 0, s>>>(ctr, totals, count, b == 0 ? 1 : 0);
      if (const int rc = clock.begin(s)) return rc;
      PathShadeEpilogue epi{p, TileSlots{s0}, in, b, q, a->d_verts, a->d_faces, d_accum_rgb, ctr};
      if (const int rc = launch_traverse_path_radiance(a, epi, ctr + 3, count, opt, trav_flags, s)) return rc;
      if (const int rc = launch_traverse_path_shadow(a, q, ctr + 1, count, d_accum_rgb, opt, trav_flags, s)) return rc;
      if (const int rc = clock.end(s)) return rc;
      end_bounce_kernel<<<1, 1, 0, s>>>(ctr, totals);
      launches += 4;
      trav_launches += 2;
      in ^= 1;
    }
    NRT_CUDA(cudaGetLastError());
  }
  if (res) {
    unsigned long long ht[3] = {0, 0, 0};
    if (const int rc = clock.stop(s)) return rc;
    NRT_CUDA(cudaMemcpyAsync(ht, totals, sizeof(ht), cudaMemcpyDeviceToHost, s));
    NRT_CUDA(cudaStreamSynchronize(s));
    float total_ms = 0.0f, span[2];
    if (const int rc = clock.read(&total_ms, span)) return rc;
    res->radiance_rays = ht[0];
    res->shadow_rays = ht[1];
    res->camera_rays = ht[2];
    res->traverse_ms = span[0];
    res->total_ms = total_ms;
    res->launches = launches;
    res->traverse_launches = trav_launches;
  }
  return NRT_OK;
}

// One bounce of the wavefront path tracer on caller-owned queues: traverses the n radiance rays, runs the reference's
// per-hit shading block in the retire step (PathShadeEpilogue), appends the continuation rays and the shadow (next-event)
// rays to the caller's output queues, then -- unless skip_shadow_pass -- traverses the shadow rays and accumulates the
// light samples that are not occluded.  This is the unit nrt_render_path_device repeats; it is exported for renderers
// that own the bounce loop, and it is what tests/test_gpu_path.py checks bounce by bounce against the reference's own
// functions (oracle/pt_ref_shim.cc).
extern "C" int nrt_path_bounce_device(const nrt_accel *h, const nrt_path_params *pp, uint32_t bounce, uint64_t n_rays,
                                      const void *d_org_tmin, const void *d_dir_tmax, const uint32_t *d_path_id,
                                      void *d_weight, void *d_out_org_tmin, void *d_out_dir_tmax, uint32_t *d_out_path_id,
                                      void *d_sh_org_tmin, void *d_sh_dir_tmax, void *d_sh_contrib_pix, float *d_accum_rgb,
                                      uint64_t *n_continue, uint64_t *n_shadow, int skip_shadow_pass, void *stream) {
  if (!h || !pp || !d_org_tmin || !d_dir_tmax || !d_path_id || !d_weight || !d_out_org_tmin || !d_out_dir_tmax ||
      !d_out_path_id || !d_sh_org_tmin || !d_sh_dir_tmax || !d_sh_contrib_pix || !d_accum_rgb) {
    set_error("nrt_path_bounce_device: NULL argument");
    return NRT_ERR_INVALID;
  }
  Accel *a = const_cast<Accel *>(reinterpret_cast<const Accel *>(h));
  const nrt_path_params p = *pp;
  if (const int rc = check_path_params(p, "nrt_path_bounce_device")) return rc;
  if (n_continue) *n_continue = 0;
  if (n_shadow) *n_shadow = 0;
  if (n_rays == 0) return NRT_OK;
  NRT_DEVICE(a->device);
  // d_counters[48..51] are the pass scratch of nrt_render_path_device too: ordered like a pass
  std::lock_guard<std::mutex> lock(a->host_mu);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (const int rc = wait_previous_pass(a, s)) return rc;
  const RecordOnExit pass_done{a->pass_done, s};
  const PathQueues q = caller_path_queues(d_org_tmin, d_dir_tmax, d_path_id, d_weight, d_out_org_tmin, d_out_dir_tmax,
                                         d_out_path_id, d_sh_org_tmin, d_sh_dir_tmax, d_sh_contrib_pix);
  unsigned long long *ctr = pass_counters(a, kPathCounters);  // [0] cont, [1] shadow, [3] n
  const unsigned long long init[4] = {0ull, 0ull, 0ull, (unsigned long long)n_rays};
  NRT_CUDA(cudaMemcpyAsync(ctr, init, sizeof(init), cudaMemcpyHostToDevice, s));
  const TraceOptions16 opt = default_trace_options();
  const uint32_t trav_flags = p.flags & 0xFFFFu;
  PathShadeEpilogue epi{p, TileSlots{0ull}, 0, bounce, q, a->d_verts, a->d_faces, d_accum_rgb, ctr};
  int rc = launch_traverse_path_radiance(a, epi, ctr + 3, (size_t)n_rays, opt, trav_flags, s);
  if (rc != NRT_OK) return rc;
  if (!skip_shadow_pass) {
    rc = launch_traverse_path_shadow(a, q, ctr + 1, (size_t)n_rays, d_accum_rgb, opt, trav_flags, s);
    if (rc != NRT_OK) return rc;
  }
  unsigned long long counts[2] = {0, 0};
  return finish_bounce(ctr, counts, n_continue, n_shadow, s);
}
