// Device-resident wavefront pass "primary + 1-bounce AO" (the headline metric of BASELINE.json).
//
// The reference has no AO example; the pass is composed from pieces of its path tracer
// (examples/path_tracer/main.cc):
//   camera ray        main.cc:809-817, 839-849   (jittered pinhole; counter-based hash instead of rand())
//   hit point         main.cc:860                (P = org + dir * t)
//   geometric normal  main.cc:306-312 (calcNormal), flipped towards the viewer main.cc:878-881
//   cosine direction  main.cc:216-250 (orthonormal basis + directionCosTheta)
//   occlusion query   main.cc:675-701 (CheckForOccluder: a CLOSEST-hit Traverse with max_t = radius;
//                     nanort has no any-hit, so AO rays do the same full closest-hit work here)
// Rays live in SoA queues (two float4 per ray); hits are nanort's 16-byte records.
#include <algorithm>
#include <mutex>
#include <string>

#include "common.cuh"
#include "wavefront.cuh"
#include "pass_host.cuh"

namespace nrt {

namespace {

__global__ void __launch_bounds__(256)
    gen_primary_kernel(nrt_ao_params p, unsigned long long slot0, uint32_t count, Wave w,
                       unsigned long long *counters /* [1] valid primaries of this wave */) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false;
  if (i < count) {
    uint32_t pix, smp;
    if (!slot_to_pixel(p, slot0 + i, pix, smp)) {
      w.pix[i] = 0xFFFFFFFFu;
      w.org_tmin[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      w.dir_tmax[i] = make_float4(0.f, 0.f, -1.f, -1.f);  // max_t < min_t: retires at the root
    } else {
      valid = true;
      smp += p.sample0;
      float dx, dy, dz;
      camera_ray(p.cam, p.width, p.height, p.seed, pix, smp, dx, dy, dz);
      w.pix[i] = pix;
      w.org_tmin[i] = make_float4(p.cam[0], p.cam[1], p.cam[2], p.ray_min_t);
      w.dir_tmax[i] = make_float4(dx, dy, dz, p.ray_max_t);
    }
  }
  const unsigned m = __ballot_sync(0xFFFFFFFFu, valid);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(counters + 1, (unsigned long long)__popc(m));
}

// Stand-alone AO stage (used when the queues are exported, and as the A/B partner of the fused epilogue):
// one AO ray per primary hit, compacted with one atomic per warp; primary misses count as unoccluded.
__global__ void __launch_bounds__(256)
    gen_ao_kernel(nrt_ao_params p, unsigned long long slot0, uint32_t count, Wave w,
                  const float4 *__restrict__ face_n, float *__restrict__ accum,
                  unsigned long long *counters /* [0] ao rays of this wave */) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  bool make = false;
  float4 o4 = make_float4(0, 0, 0, 0), d4 = make_float4(0, 0, 0, 0);
  uint32_t pix = 0xFFFFFFFFu;
  if (i < count) {
    pix = w.pix[i];
    if (pix != 0xFFFFFFFFu) {
      const Hit16 h = w.hits[i];
      if (h.prim_id == 0xFFFFFFFFu) {
        atomicAdd(accum + pix, 1.0f);
      } else {
        make_ao_ray(p, pix, slot_sample(p, slot0 + i), w.org_tmin[i], w.dir_tmax[i], h.t, h.prim_id, face_n, o4, d4);
        make = true;
      }
    }
  }
  const unsigned m = __ballot_sync(0xFFFFFFFFu, make);
  if (m == 0u) return;
  unsigned long long base = 0;
  if (lane == 0) base = atomicAdd(counters + 0, (unsigned long long)__popc(m));
  base = __shfl_sync(0xFFFFFFFFu, base, 0);
  if (make) {
    const unsigned long long j = base + __popc(m & ((1u << lane) - 1u));
    w.ao_org_tmin[j] = o4;
    w.ao_dir_tmax[j] = d4;
    w.ao_pix[j] = pix;
  }
}

// Accel::d_face_n: the unit normal make_ao_ray() reads, once per primitive instead of once per primary hit
__global__ void __launch_bounds__(256)
    face_normals_kernel(const float *__restrict__ verts, const uint32_t *__restrict__ faces, uint32_t n,
                        float4 *__restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float nx, ny, nz, a2;
  geometric_normal(verts, faces, i, nx, ny, nz, a2);
  out[i] = make_float4(nx, ny, nz, 0.0f);
}

__global__ void __launch_bounds__(256)
    accumulate_ao_kernel(Wave w, const unsigned long long *__restrict__ counters, float *__restrict__ accum,
                         unsigned long long *totals /* [0] ao rays, [1] ao hits, [2] primaries */) {
  const unsigned long long n = counters[0];
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  bool occluded = false;
  if (i < n) {
    occluded = w.ao_hits[i].prim_id != 0xFFFFFFFFu;
    if (!occluded) atomicAdd(accum + w.ao_pix[i], 1.0f);
  }
  const unsigned m = __ballot_sync(0xFFFFFFFFu, occluded);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(totals + 1, (unsigned long long)__popc(m));
  if (i == 0) {
    atomicAdd(totals + 0, n);
    atomicAdd(totals + 2, counters[1]);
  }
}

__global__ void fold_wave_counters_kernel(const unsigned long long *counters, unsigned long long *totals) {
  totals[0] += counters[0];
  totals[2] += counters[1];
}

// AoS copy of a SoA queue as 36-byte nanort::Ray records (workload export for the host-buffer arms)
__global__ void __launch_bounds__(256)
    soa_to_aos_kernel(const float4 *__restrict__ org_tmin, const float4 *__restrict__ dir_tmax,
                      const unsigned long long *n_ptr, unsigned long long n, Ray36 *__restrict__ out, uint32_t type) {
  if (n_ptr) n = *n_ptr;
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 o = org_tmin[i], d = dir_tmax[i];
  Ray36 r;
  r.org[0] = o.x;
  r.org[1] = o.y;
  r.org[2] = o.z;
  r.dir[0] = d.x;
  r.dir[1] = d.y;
  r.dir[2] = d.z;
  r.min_t = o.w;
  r.max_t = d.w;
  r.type = type;
  out[i] = r;
}

}  // namespace

// launch_traverse_soa needs the ray count on the host; AO counts are produced on the device, so the
// AO traversal is launched over the wave capacity with a device-side count (see traverse.cu).
int launch_traverse_soa_devcount(const Accel *a, const float4 *d_org_tmin, const float4 *d_dir_tmax,
                                 const unsigned long long *d_count, size_t capacity, Hit16 *d_hits,
                                 const TraceOptions16 &opt, uint32_t flags, cudaStream_t s);
int launch_traverse_camera_fused(Accel *a, const Wave &w, const nrt_ao_params &p, unsigned long long slot0, size_t count,
                                 const float4 *d_face_n, float *d_accum, unsigned long long *d_wave_counters,
                                 const TraceOptions16 &opt, uint32_t flags, cudaStream_t s);
int launch_traverse_ao_fused(const Accel *a, const Wave &w, const unsigned long long *d_count, size_t capacity,
                             float *d_accum, unsigned long long *d_totals, const TraceOptions16 &opt, uint32_t flags,
                             cudaStream_t s);

}  // namespace nrt

using namespace nrt;

// number of slots in [s0, s0 + count) that map to pixels inside the image (whole tiles per wave)
static unsigned long long valid_slots(const nrt_ao_params &p, unsigned long long s0, uint32_t count) {
  const unsigned long long per_tile = (unsigned long long)p.tile_w * p.tile_h * p.spp;
  const uint32_t tiles_x = (p.width + p.tile_w - 1) / p.tile_w;
  unsigned long long total = 0;
  for (unsigned long long k = s0 / per_tile; k < (s0 + count) / per_tile; k++) {
    const unsigned long long tile = k * p.n_shards + p.shard;
    const uint32_t tx = (uint32_t)(tile % tiles_x), ty = (uint32_t)(tile / tiles_x);
    const uint32_t x0 = tx * p.tile_w, y0 = ty * p.tile_h;
    if (x0 >= p.width || y0 >= p.height) continue;
    const uint32_t wv = p.width - x0 < p.tile_w ? p.width - x0 : p.tile_w;
    const uint32_t hv = p.height - y0 < p.tile_h ? p.height - y0 : p.tile_h;
    total += (unsigned long long)wv * hv * p.spp;
  }
  return total;
}

// dump_primary / dump_ao (optional, device): AoS copies of the two ray queues, primary rays at their slot
// index, AO rays appended in queue order; *n_ao_out receives the AO count (forces a sync per wave).
static int run_ao_pass(const nrt_accel *h, const nrt_ao_params *pp, float *d_accum, nrt_ao_result *res, void *stream,
                       Ray36 *dump_primary, Ray36 *dump_ao, uint64_t *n_ao_out) {
  if (!h || !pp || !d_accum) {
    set_error("nrt_render_ao_device: NULL argument");
    return NRT_ERR_INVALID;
  }
  Accel *a = const_cast<Accel *>(reinterpret_cast<const Accel *>(h));
  nrt_ao_params p = *pp;
  if (p.width == 0 || p.height == 0 || p.spp == 0 || p.n_shards == 0 || p.shard >= p.n_shards || p.tile_w == 0 ||
      p.tile_h == 0 || (p.tile_w % 8) != 0 || (p.tile_h % 4) != 0) {
    set_error("nrt_render_ao_device: bad parameters (tiles must be multiples of 8x4 pixels)");
    return NRT_ERR_INVALID;
  }
  // before anything is derived or launched: the face normals and the camera-relative copies are built from the
  // triangle layout, which sphere / box accels (and the top level of a scene) do not have
  if (!a->d_pair || !a->d_tris_cm || !a->d_faces) {
    set_error("nrt_render_ao_device: the AO pass needs a triangle accel");
    return NRT_ERR_INVALID;
  }
  NRT_DEVICE(a->device);
  // d_wave and d_counters[2..6] are per-accel scratch: passes on ONE accel run one after the other on the device
  // (passes on different accels, e.g. one per GPU, run concurrently).  host_mu orders the enqueueing; pass_done makes
  // this pass wait for the previous AO or path pass on this accel, which may still run on another stream, so that
  // nothing it reads (the wave scratch, the counters, the camera-relative copies) is rewritten before it has finished
  std::lock_guard<std::mutex> lock(a->host_mu);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (const int rc = wait_previous_pass(a, s)) return rc;
  const RecordOnExit pass_done{a->pass_done, s};
  if (const int rc = ensure_face_normals(a, s)) return rc;
  const ShardSlots sh = shard_slots(p.width, p.height, p.tile_w, p.tile_h, p.spp, p.shard, p.n_shards);
  const unsigned long long total_slots = sh.total;
  // wave capacity: whole tiles, at most 16 Mi camera rays; the compacted AO queue of such a wave (~9 M rays x
  // 36 B = 330 MB) is written by the primary launch and read back by the AO launch -- 6.6 x the 50 MB L2
  const unsigned long long cap = sh.wave(16ull << 20);
  Wave w;
  if (const int rc = carve_pass_scratch(a, [&](Carver &c) {
        w.org_tmin = c.take<float4>(cap);
        w.dir_tmax = c.take<float4>(cap);
        w.ao_org_tmin = c.take<float4>(cap);
        w.ao_dir_tmax = c.take<float4>(cap);
        w.hits = c.take<Hit16>(cap);
        w.ao_hits = c.take<Hit16>(cap);
        w.pix = c.take<uint32_t>(cap);
        w.ao_pix = c.take<uint32_t>(cap);
      }))
    return rc;
  unsigned long long *wave_ctr = pass_counters(a, kWaveCounters);  // [2],[3]
  unsigned long long *totals = pass_counters(a, kPassTotals);      // [4..6]
  NRT_CUDA(cudaMemsetAsync(totals, 0, 3 * sizeof(unsigned long long), s));

  TraceOptions16 opt = default_trace_options();
  PassClock clock(res != nullptr);
  if (const int rc = clock.start(s)) return rc;
  uint32_t launches = 0, trav_launches = 0;
  unsigned long long dumped_ao = 0, valid_primaries_host = 0;
  const bool fused = !dump_primary && !dump_ao && !(p.flags & NRT_AO_UNFUSED);
  if (!fused && (p.flags & NRT_AO_PACKED_TILES)) {
    set_error("nrt_render_ao_device: NRT_AO_PACKED_TILES needs the fused pass");
    return NRT_ERR_INVALID;
  }
  const uint32_t trav_flags = p.flags & 0xFFFFu;
  int rc = NRT_OK;
  for (unsigned long long s0 = 0; s0 < total_slots && rc == NRT_OK; s0 += cap) {
    const uint32_t count = (uint32_t)std::min<unsigned long long>(cap, total_slots - s0);
    const uint32_t grid = (count + 255) / 256;
    if (cudaMemsetAsync(wave_ctr, 0, 2 * sizeof(unsigned long long), s) != cudaSuccess) {
      rc = NRT_ERR_CUDA;
      break;
    }
    if (!fused) {
      gen_primary_kernel<<<grid, 256, 0, s>>>(p, s0, count, w, wave_ctr);
      launches++;
    }
    // a traversal launch between the clock's marks, tag 0 for camera rays and 1 for AO rays
    const auto timed = [&](int tag, auto &&launch) -> int {
      if (const int rc = clock.begin(s)) return rc;
      if (const int rc = launch()) return rc;
      return clock.end(s, tag);
    };
    if (fused) {
      // two traversal launches per wave and nothing else: camera rays are generated at ray fetch, the retire
      // steps spawn the AO rays and accumulate visibility
      if ((rc = timed(0, [&] {
             return launch_traverse_camera_fused(a, w, p, s0, count, a->d_face_n, d_accum, wave_ctr, opt, trav_flags, s);
           })))
        break;
      if ((rc = timed(1, [&] {
             return launch_traverse_ao_fused(a, w, wave_ctr, count, d_accum, totals, opt, trav_flags, s);
           })))
        break;
      fold_wave_counters_kernel<<<1, 1, 0, s>>>(wave_ctr, totals);
      launches += 3;
      trav_launches += 2;
      valid_primaries_host += valid_slots(p, s0, count);
    } else {
      if (dump_primary) {
        soa_to_aos_kernel<<<grid, 256, 0, s>>>(w.org_tmin, w.dir_tmax, nullptr, count, dump_primary + s0, 1u);
        launches++;
      }
      if ((rc = timed(0, [&] { return launch_traverse_soa(a, w.org_tmin, w.dir_tmax, count, w.hits, opt, trav_flags, s); })))
        break;
      launches++;
      trav_launches++;
      gen_ao_kernel<<<grid, 256, 0, s>>>(p, s0, count, w, a->d_face_n, d_accum, wave_ctr);
      launches++;
      if (dump_ao) {
        unsigned long long n_wave = 0;
        soa_to_aos_kernel<<<grid, 256, 0, s>>>(w.ao_org_tmin, w.ao_dir_tmax, wave_ctr, 0, dump_ao + dumped_ao, 2u);
        launches++;
        cudaMemcpyAsync(&n_wave, wave_ctr, sizeof(n_wave), cudaMemcpyDeviceToHost, s);
        cudaStreamSynchronize(s);
        dumped_ao += n_wave;
      }
      if ((rc = timed(1, [&] {
             return launch_traverse_soa_devcount(a, w.ao_org_tmin, w.ao_dir_tmax, wave_ctr, count, w.ao_hits, opt,
                                                 trav_flags, s);
           })))
        break;
      launches++;
      trav_launches++;
      accumulate_ao_kernel<<<grid, 256, 0, s>>>(w, wave_ctr, d_accum, totals);
      launches++;
    }
    if (cudaGetLastError() != cudaSuccess) rc = NRT_ERR_CUDA;
  }
  if (rc != NRT_OK && cudaGetLastError() != cudaSuccess && std::string(nrt_last_error()).empty())
    set_error("nrt_render_ao_device: CUDA launch failure");
  if (n_ao_out) *n_ao_out = dumped_ao;
  if (rc == NRT_OK && res) {
    unsigned long long ht[3] = {0, 0, 0};
    if ((rc = clock.stop(s))) return rc;
    cudaError_t e = cudaMemcpyAsync(ht, totals, sizeof(ht), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return cuda_fail(e, "nrt_render_ao_device read-back", __FILE__, __LINE__);
    float total = 0.0f, span[2];
    if ((rc = clock.read(&total, span))) return rc;
    res->ao_rays = ht[0];
    res->ao_hits = ht[1];
    res->primary_rays = ht[2] + valid_primaries_host;
    res->traverse_ms = span[0] + span[1];
    res->primary_traverse_ms = span[0];
    res->ao_traverse_ms = span[1];
    res->total_ms = total;
    res->launches = launches;
    res->traverse_launches = trav_launches;
  }
  return rc;
}

namespace nrt {
int ensure_face_normals(Accel *a, cudaStream_t s) {
  if (a->d_face_n) return NRT_OK;
  NRT_CUDA(cudaMalloc(&a->d_face_n, sizeof(float4) * (size_t)a->n_prims));
  face_normals_kernel<<<(a->n_prims + 255) / 256, 256, 0, s>>>(a->d_verts, a->d_faces, a->n_prims, a->d_face_n);
  NRT_CUDA(cudaGetLastError());
  return NRT_OK;
}

int run_ao_pass_internal(const nrt_accel *h, const nrt_ao_params *pp, float *d_accum, nrt_ao_result *res, void *stream) {
  return run_ao_pass(h, pp, d_accum, res, stream, nullptr, nullptr, nullptr);
}
}  // namespace nrt

extern "C" int nrt_render_ao_device(const nrt_accel *h, const nrt_ao_params *pp, float *d_accum, nrt_ao_result *res,
                                    void *stream) {
  return run_ao_pass(h, pp, d_accum, res, stream, nullptr, nullptr, nullptr);
}

extern "C" int nrt_ao_workload_device(const nrt_accel *h, const nrt_ao_params *pp, float *d_accum,
                                      void *d_primary_rays_36B, void *d_ao_rays_36B, uint64_t *n_primary,
                                      uint64_t *n_ao, void *stream) {
  if (!d_primary_rays_36B || !d_ao_rays_36B) {
    set_error("nrt_ao_workload_device: NULL ray buffer");
    return NRT_ERR_INVALID;
  }
  nrt_ao_result res;
  int rc = run_ao_pass(h, pp, d_accum, &res, stream, static_cast<Ray36 *>(d_primary_rays_36B),
                       static_cast<Ray36 *>(d_ao_rays_36B), n_ao);
  if (rc == NRT_OK && n_primary) *n_primary = res.primary_rays;
  return rc;
}
