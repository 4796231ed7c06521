// Host-side plumbing shared by the wavefront passes (render.cu, path.cu, bake.cu, lightmap.cu, bdpt.cu, scene.cu,
// scene_bake.cu), as host_slots.cuh is for calls: scratch layouts, pass timers, a call's own device memory, the path
// queues, the shard and wave arithmetic and the parameter rules the flat and scene forms share.  Host code only.
#pragma once
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/nanort_b200_lightmap.h"
#include "common.cuh"
#include "wavefront.cuh"

namespace nrt {

// A bump pointer over one block of scratch; every buffer starts on a 256-byte boundary.  Without a base it only
// measures: a pass writes its layout once, as one function of a Carver, and runs it first to size the block, then
// over the block to hand out the buffers.
class Carver {
 public:
  Carver() = default;
  explicit Carver(void *base) : base_(static_cast<char *>(base)) {}
  template <class T>
  T *take(size_t n) {
    const size_t at = used_;
    used_ += (n * sizeof(T) + 255) & ~(size_t)255;
    return base_ ? reinterpret_cast<T *>(base_ + at) : nullptr;
  }
  size_t size() const { return used_; }

 private:
  char *base_ = nullptr;
  size_t used_ = 0;
};

// Sizes the accel's pass scratch (Accel::d_wave) for `layout` and carves it (call under the pass ordering)
template <class Layout>
int carve_pass_scratch(Accel *a, Layout &&layout) {
  Carver measure;
  layout(measure);
  if (const int rc = grow_wave(a, measure.size())) return rc;
  Carver c(a->d_wave);
  layout(c);
  return NRT_OK;
}

// The device memory of one call that owns its scratch (the scene passes and bakes): alloc() is one cudaMalloc holding
// a layout.  The scene calls return only after their work has finished: on success a call returns drain(), which
// reports a failed wait; on every exit, the error paths included, the destructor waits for the call's stream again
// before it frees the memory.
class CallMemory {
 public:
  explicit CallMemory(cudaStream_t s) : s_(s) {}
  CallMemory(const CallMemory &) = delete;
  CallMemory &operator=(const CallMemory &) = delete;
  ~CallMemory() {
    cudaStreamSynchronize(s_);
    for (void *p : blocks_) cudaFree(p);
  }
  int drain() {
    NRT_CUDA(cudaStreamSynchronize(s_));
    return NRT_OK;
  }
  template <class Layout>
  int alloc(Layout &&layout) {
    Carver measure;
    layout(measure);
    void *d = nullptr;
    NRT_CUDA(cudaMalloc(&d, measure.size() ? measure.size() : 1));
    blocks_.push_back(d);
    Carver c(d);
    layout(c);
    return NRT_OK;
  }

 private:
  cudaStream_t s_;
  std::vector<void *> blocks_;
};

// CUDA events of one pass: the whole pass (start .. stop) and the traversal launches in it (begin .. end), summed
// under two tags so that the AO pass reports its primary and AO launches apart.  Off -- the caller asked for no
// result -- it creates and records no event.  It destroys its events on every exit.
class PassClock {
 public:
  explicit PassClock(bool on) : on_(on) {}
  PassClock(const PassClock &) = delete;
  PassClock &operator=(const PassClock &) = delete;
  ~PassClock() {
    for (cudaEvent_t e : ev_)
      if (e) cudaEventDestroy(e);
  }
  int start(cudaStream_t s) { return mark(s); }
  int begin(cudaStream_t s) { return mark(s); }
  int end(cudaStream_t s, int tag = 0) {
    if (on_) tags_.push_back(tag);
    return mark(s);
  }
  int stop(cudaStream_t s) { return mark(s); }
  // once the stream has passed stop(): the pass's time and the summed spans of each tag, in milliseconds (all zero
  // when the clock is off or has not started)
  int read(float *total_ms, float span_ms[2]) const {
    *total_ms = span_ms[0] = span_ms[1] = 0.0f;
    if (ev_.empty()) return NRT_OK;
    for (size_t k = 0; k < tags_.size(); k++) {
      float m = 0.0f;
      NRT_CUDA(cudaEventElapsedTime(&m, ev_[1 + 2 * k], ev_[2 + 2 * k]));
      span_ms[tags_[k]] += m;
    }
    NRT_CUDA(cudaEventElapsedTime(total_ms, ev_.front(), ev_.back()));
    return NRT_OK;
  }

 private:
  int mark(cudaStream_t s) {
    if (!on_) return NRT_OK;
    ev_.push_back(nullptr);
    NRT_CUDA(cudaEventCreate(&ev_.back()));
    NRT_CUDA(cudaEventRecord(ev_.back(), s));
    return NRT_OK;
  }
  bool on_;
  std::vector<cudaEvent_t> ev_;  // start, begin / end pairs, stop
  std::vector<int> tags_;        // per begin / end pair
};

// bake.cu: the scratch of the bakes' covered-texel compaction of n records
struct Compaction {
  uint32_t *offs, *list, *scratch;
};
Compaction carve_compaction(Carver &c, uint32_t n);

// The path queues of `cap` paths: the two radiance queues, the shadow queue and the throughputs
inline PathQueues carve_path_queues(Carver &c, size_t cap) {
  PathQueues q;
  for (int k = 0; k < 2; k++) {
    q.org_tmin[k] = c.take<float4>(cap);
    q.dir_tmax[k] = c.take<float4>(cap);
  }
  q.sh_org_tmin = c.take<float4>(cap);
  q.sh_dir_tmax = c.take<float4>(cap);
  q.sh_contrib_pix = c.take<float4>(cap);
  q.weight = c.take<float4>(cap);
  for (int k = 0; k < 2; k++) q.path_id[k] = c.take<uint32_t>(cap);
  return q;
}

// The queues of a one-bounce entry on the caller's buffers: queue 0 is read, queue 1 and the shadow queue written
inline PathQueues caller_path_queues(const void *org_tmin, const void *dir_tmax, const uint32_t *path_id, void *weight,
                                     void *out_org_tmin, void *out_dir_tmax, uint32_t *out_path_id, void *sh_org_tmin,
                                     void *sh_dir_tmax, void *sh_contrib_pix) {
  PathQueues q;
  q.org_tmin[0] = static_cast<float4 *>(const_cast<void *>(org_tmin));
  q.dir_tmax[0] = static_cast<float4 *>(const_cast<void *>(dir_tmax));
  q.path_id[0] = const_cast<uint32_t *>(path_id);
  q.org_tmin[1] = static_cast<float4 *>(out_org_tmin);
  q.dir_tmax[1] = static_cast<float4 *>(out_dir_tmax);
  q.path_id[1] = out_path_id;
  q.sh_org_tmin = static_cast<float4 *>(sh_org_tmin);
  q.sh_dir_tmax = static_cast<float4 *>(sh_dir_tmax);
  q.sh_contrib_pix = static_cast<float4 *>(sh_contrib_pix);
  q.weight = static_cast<float4 *>(weight);
  return q;
}

// The end of the one-bounce entries: waits for the stream, then reports the bounce's continuation and shadow rays.
// The flat entries read them from their device counters [0] and [1]; the scene entries hold them already (d_ctr NULL).
inline int finish_bounce(const unsigned long long *d_ctr, unsigned long long counts[2], uint64_t *n_continue,
                         uint64_t *n_shadow, cudaStream_t s) {
  if (d_ctr) NRT_CUDA(cudaMemcpyAsync(counts, d_ctr, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  NRT_CUDA(cudaStreamSynchronize(s));
  if (n_continue) *n_continue = counts[0];
  if (n_shadow) *n_shadow = counts[1];
  return NRT_OK;
}

// This shard's ray slots: the image's tiles (edge tiles partial: their slots outside the image map to no pixel) dealt
// round-robin over n_shards, tile_w x tile_h x spp slots each
struct ShardSlots {
  unsigned long long tiles, per_tile, total;
  // the slots of a wave: whole tiles, at most `budget` slots but at least one tile, and at most `total`
  unsigned long long wave(unsigned long long budget) const {
    const unsigned long long tiles_per_wave = budget / per_tile;
    return std::min(total, (tiles_per_wave ? tiles_per_wave : 1ull) * per_tile);
  }
};
// (the callers have checked that the tile sizes and n_shards are positive and shard < n_shards)
inline ShardSlots shard_slots(uint32_t width, uint32_t height, uint32_t tile_w, uint32_t tile_h, uint32_t spp,
                              uint32_t shard, uint32_t n_shards) {
  const unsigned long long tiles_x = (width + (unsigned long long)tile_w - 1) / tile_w;
  const unsigned long long tiles_y = (height + (unsigned long long)tile_h - 1) / tile_h;
  const unsigned long long n_tiles = tiles_x * tiles_y;
  ShardSlots r;
  r.tiles = n_tiles > shard ? (n_tiles - shard + n_shards - 1) / n_shards : 0;
  r.per_tile = (unsigned long long)tile_w * tile_h * spp;
  r.total = r.tiles * r.per_tile;
  return r;
}

// sets the error "who: why" and returns NRT_ERR_INVALID
inline int refuse(const char *who, const std::string &why) {
  set_error(std::string(who) + ": " + why);
  return NRT_ERR_INVALID;
}

// The rules of nrt_path_params that every path pass keeps (flat, scene, one-bounce): image, samples, tiles of 8 x 4
// pixels, bounces, materials and emissive faces
inline int check_path_params(const nrt_path_params &p, const char *who) {
  if (p.width == 0 || p.height == 0 || p.spp == 0 || p.n_shards == 0 || p.shard >= p.n_shards || p.tile_w == 0 ||
      p.tile_h == 0 || (p.tile_w % 8) != 0 || (p.tile_h % 4) != 0 || p.max_bounces == 0 || p.n_materials == 0 ||
      !p.d_materials || (p.n_emissive > 0 && !p.d_emissive_faces))
    return refuse(who, "bad parameters");
  return NRT_OK;
}

// The numeric rules of the AO bakes (flat and scene)
inline int check_bake_params(const nrt_bake_params &p, const char *who) {
  const uint64_t n = (uint64_t)p.width * p.height;
  if (n == 0 || n > kMaxTexels || p.spp == 0)
    return refuse(who, "width * height must lie in [1, 2^31] and spp must be positive");
  return NRT_OK;
}

// The numeric rules of the lightmap bakes (flat and scene)
inline int check_lightmap_params(const nrt_lightmap_params &p, const char *who) {
  const uint64_t n = (uint64_t)p.width * p.height;
  if (n == 0 || n > kMaxTexels || p.spp == 0 || p.max_bounces == 0 || p.n_materials == 0 || !p.d_materials ||
      (p.n_emissive > 0 && !p.d_emissive_faces))
    return refuse(who, "width * height must lie in [1, 2^31], spp, max_bounces and n_materials must be positive, and "
                       "the materials and emissive faces given");
  return NRT_OK;
}

}  // namespace nrt
