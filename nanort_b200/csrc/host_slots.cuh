// Host-side call plumbing shared by the float accel (Accel), the double accel (AccelF64) and the two-level scene
// (Scene): the ring of per-launch scratch slots, the zero-copy pool of small calls, the chunked staging pipeline of the
// host-pointer entries and the lazy host mirror of a tree.  Included by common.cuh after the error helpers.
//
// Each type owns its CUDA resources and frees them in its destructor; the owners delete their objects inside a
// DeviceGuard of their device, so the destructors run on the right one.  Lock order: a StagingPipeline, Accel::host_mu
// or AccelF64::mu may be held while a LaunchRing is run; nothing is taken while a ring's own mutex is held.
#pragma once
#include <string.h>

#include <algorithm>
#include <condition_variable>
#include <mutex>
#include <vector>

namespace nrt {

// N slots of per-launch scratch (a ray cursor, ...) handed out round-robin.  A slot's event is recorded after the last
// launch that used it, and the next launch on the slot makes its stream wait for it: any number of launches in flight
// on any streams never share a slot's scratch.
template <uint32_t N>
class LaunchRing {
 public:
  LaunchRing() = default;
  LaunchRing(const LaunchRing &) = delete;
  LaunchRing &operator=(const LaunchRing &) = delete;
  ~LaunchRing() {
    for (cudaEvent_t e : done_)
      if (e) cudaEventDestroy(e);
  }

  // Takes the next slot k, makes `s` wait for its previous launch, calls enqueue(k) -> NRT_OK or an error code, and
  // records the slot's event on `s` if enqueue succeeded.  All of it happens under one lock, so it is in the same order
  // on the host and on the device.
  template <class Enqueue>
  int run(cudaStream_t s, Enqueue enqueue) {
    std::lock_guard<std::mutex> lock(mu_);
    const uint32_t k = next_++ % N;
    if (!done_[k]) NRT_CUDA(cudaEventCreateWithFlags(&done_[k], cudaEventDisableTiming));
    NRT_CUDA(cudaStreamWaitEvent(s, done_[k], 0));
    const int rc = enqueue(k);
    if (rc != NRT_OK) return rc;
    NRT_CUDA(cudaEventRecord(done_[k], s));
    return NRT_OK;
  }

  // Waits on the host until the last launch on slot k has finished (before its scratch is reallocated).  Only from
  // inside enqueue(k).
  int wait_host(uint32_t k) {
    NRT_CUDA(cudaEventSynchronize(done_[k]));
    return NRT_OK;
  }

 private:
  std::mutex mu_;
  uint32_t next_ = 0;
  cudaEvent_t done_[N] = {};
};

// Calls of at most kMaxRays rays (the facade's one-ray Traverse, small packets from worker threads) go through N slots,
// each a pinned, mapped host buffer the kernel reads the rays from and writes the records to directly (zero copy) and a
// non-blocking stream of its own: no staging copies, one synchronisation, and calls from different host threads run
// side by side.  Slot layout: rays (kMaxRays x RayBytes) | records (kMaxRays x RecBytes) | flags (kMaxRays x 1 B).
template <int N, size_t RayBytes, size_t RecBytes>
class SmallCallPool {
 public:
  static constexpr size_t kMaxRays = 64;

  SmallCallPool() = default;
  SmallCallPool(const SmallCallPool &) = delete;
  SmallCallPool &operator=(const SmallCallPool &) = delete;
  ~SmallCallPool() {
    for (Slot &sl : slots_) {
      if (sl.h) cudaFreeHost(sl.h);
      if (sl.s) cudaStreamDestroy(sl.s);
    }
  }

  // One whole call of n <= kMaxRays rays of ray_bytes (<= RayBytes) each: waits for a free slot i, copies the rays in,
  // calls launch(i, h_rays, h_recs, h_mask or nullptr, stream) -> NRT_OK or an error code, synchronises the slot's
  // stream (after a failed launch too: nothing of the call may be left in flight) and copies the records out.
  template <class Launch>
  int run(const void *rays, size_t n, size_t ray_bytes, void *recs, uint8_t *mask, Launch launch) {
    const size_t off_recs = kMaxRays * RayBytes, off_mask = off_recs + kMaxRays * RecBytes;
    int idx = -1;
    {
      std::unique_lock<std::mutex> lk(mu_);
      for (;;) {
        for (int i = 0; i < N && idx < 0; i++)
          if (!slots_[i].busy) idx = i;
        if (idx >= 0) break;
        cv_.wait(lk);
      }
      slots_[idx].busy = true;
    }
    Slot &sl = slots_[idx];
    int rc = NRT_OK;
    cudaError_t e = cudaSuccess;
    if (!sl.h) e = cudaHostAlloc(&sl.h, off_mask + kMaxRays, cudaHostAllocPortable | cudaHostAllocMapped);
    if (e == cudaSuccess && !sl.s) e = cudaStreamCreateWithFlags(&sl.s, cudaStreamNonBlocking);
    if (e == cudaSuccess) {
      char *hb = static_cast<char *>(sl.h);
      memcpy(hb, rays, n * ray_bytes);
      rc = launch(idx, static_cast<void *>(hb), static_cast<void *>(hb + off_recs),
                  mask ? reinterpret_cast<uint8_t *>(hb + off_mask) : nullptr, sl.s);
      e = cudaStreamSynchronize(sl.s);
      if (rc == NRT_OK && e == cudaSuccess) {
        memcpy(recs, hb + off_recs, n * RecBytes);
        if (mask) memcpy(mask, hb + off_mask, n);
      }
    }
    {
      std::lock_guard<std::mutex> lk(mu_);
      sl.busy = false;
    }
    cv_.notify_one();
    if (rc != NRT_OK) return rc;
    NRT_CUDA(e);
    return NRT_OK;
  }

 private:
  struct Slot {
    void *h = nullptr;
    cudaStream_t s = nullptr;
    bool busy = false;
  };
  Slot slots_[N];
  std::mutex mu_;
  std::condition_variable cv_;
};

// The host-pointer batch call: chunks of rays flow H2D -> launch -> D2H through three stream slots, so that the copy
// engines (both directions) and the SMs overlap.  Calls are serialised per pipeline: its slots are shared.
class StagingPipeline {
 public:
  static constexpr size_t kChunkRays = (size_t)1 << 20;

  StagingPipeline() = default;
  StagingPipeline(const StagingPipeline &) = delete;
  StagingPipeline &operator=(const StagingPipeline &) = delete;
  ~StagingPipeline() {
    for (int i = 0; i < 3; i++) {
      cudaFree(d_rays_[i]);
      cudaFree(d_recs_[i]);
      cudaFree(d_mask_[i]);
      if (streams_[i]) cudaStreamDestroy(streams_[i]);
    }
  }

  // creates the three (non-blocking) streams unless they exist
  int create_streams() {
    for (cudaStream_t &s : streams_)
      if (!s) NRT_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    return NRT_OK;
  }
  cudaStream_t stream(int i) const { return streams_[i]; }

  // n rays of ray_bytes each from `rays` to n records of rec_bytes each in `recs` (and n flags in `mask` unless it is
  // nullptr): launch(d_rays, m, d_recs, d_mask or nullptr, stream) -> NRT_OK or an error code, once per chunk of at
  // most kChunkRays rays.  Success or not, nothing is still writing into the caller's buffers when this returns.
  template <class Launch>
  int run(const void *rays, size_t n, size_t ray_bytes, void *recs, size_t rec_bytes, uint8_t *mask, Launch launch) {
    std::lock_guard<std::mutex> lock(mu_);
    const size_t chunk = std::min(n, kChunkRays);
    int rc = create_streams();
    if (rc == NRT_OK) rc = reserve(chunk * ray_bytes, chunk * rec_bytes, chunk);
    if (rc != NRT_OK) return rc;
    const char *src = static_cast<const char *>(rays);
    char *dst = static_cast<char *>(recs);
    cudaError_t e = cudaSuccess;
    int slot = 0;
    for (size_t done = 0; done < n; done += chunk) {
      const size_t m = std::min(chunk, n - done);
      cudaStream_t s = streams_[slot];
      // the slot's previous chunk (3 iterations ago) must have drained before its buffers are reused
      e = cudaStreamSynchronize(s);
      if (e == cudaSuccess) e = cudaMemcpyAsync(d_rays_[slot], src + done * ray_bytes, m * ray_bytes, cudaMemcpyHostToDevice, s);
      if (e != cudaSuccess) break;
      rc = launch(static_cast<const void *>(d_rays_[slot]), m, d_recs_[slot], mask ? d_mask_[slot] : nullptr, s);
      if (rc != NRT_OK) break;
      e = cudaMemcpyAsync(dst + done * rec_bytes, d_recs_[slot], m * rec_bytes, cudaMemcpyDeviceToHost, s);
      if (e == cudaSuccess && mask) e = cudaMemcpyAsync(mask + done, d_mask_[slot], m, cudaMemcpyDeviceToHost, s);
      if (e != cudaSuccess) break;
      slot = (slot + 1) % 3;
    }
    for (cudaStream_t s : streams_) {
      const cudaError_t es = cudaStreamSynchronize(s);
      if (e == cudaSuccess) e = es;
    }
    if (rc != NRT_OK) return rc;
    NRT_CUDA(e);
    return NRT_OK;
  }

 private:
  // every slot's buffers hold at least these many bytes; they grow and never shrink
  int reserve(size_t ray_need, size_t rec_need, size_t mask_need) {
    if (ray_cap_ >= ray_need && rec_cap_ >= rec_need && mask_cap_ >= mask_need) return NRT_OK;
    ray_need = std::max(ray_need, ray_cap_);
    rec_need = std::max(rec_need, rec_cap_);
    mask_need = std::max(mask_need, mask_cap_);
    for (int i = 0; i < 3; i++) {
      cudaFree(d_rays_[i]);
      cudaFree(d_recs_[i]);
      cudaFree(d_mask_[i]);
      d_rays_[i] = d_recs_[i] = nullptr;
      d_mask_[i] = nullptr;
    }
    ray_cap_ = rec_cap_ = mask_cap_ = 0;
    for (int i = 0; i < 3; i++) {
      NRT_CUDA(cudaMalloc(&d_rays_[i], ray_need));
      NRT_CUDA(cudaMalloc(&d_recs_[i], rec_need));
      NRT_CUDA(cudaMalloc(&d_mask_[i], mask_need));
    }
    ray_cap_ = ray_need, rec_cap_ = rec_need, mask_cap_ = mask_need;
    return NRT_OK;
  }

  std::mutex mu_;
  cudaStream_t streams_[3] = {nullptr, nullptr, nullptr};
  void *d_rays_[3] = {nullptr, nullptr, nullptr};
  void *d_recs_[3] = {nullptr, nullptr, nullptr};
  uint8_t *d_mask_[3] = {nullptr, nullptr, nullptr};
  size_t ray_cap_ = 0, rec_cap_ = 0, mask_cap_ = 0;
};

// Lazy host copy of a tree's nodes and indices_ (GetNodes / GetIndices / Dump), filled on first use or assigned from
// the host arrays an accel was adopted from.
template <class NodeT>
class HostMirror {
 public:
  int get(int device, const NodeT *d_nodes, size_t n_nodes, const uint32_t *d_indices, size_t n_indices,
          const void **nodes_out, size_t *n_nodes_out, const uint32_t **indices_out, size_t *n_indices_out) {
    std::lock_guard<std::mutex> lock(mu_);
    if (!valid_) {
      NRT_DEVICE(device);
      nodes_.resize(n_nodes);
      indices_.resize(n_indices);
      NRT_CUDA(cudaMemcpy(nodes_.data(), d_nodes, sizeof(NodeT) * n_nodes, cudaMemcpyDeviceToHost));
      NRT_CUDA(cudaMemcpy(indices_.data(), d_indices, sizeof(uint32_t) * n_indices, cudaMemcpyDeviceToHost));
      valid_ = true;
    }
    if (nodes_out) *nodes_out = nodes_.data();
    if (n_nodes_out) *n_nodes_out = nodes_.size();
    if (indices_out) *indices_out = indices_.data();
    if (n_indices_out) *n_indices_out = indices_.size();
    return NRT_OK;
  }
  void assign(const NodeT *nodes, size_t n_nodes, const uint32_t *indices, size_t n_indices) {
    std::lock_guard<std::mutex> lock(mu_);
    nodes_.assign(nodes, nodes + n_nodes);
    indices_.assign(indices, indices + n_indices);
    valid_ = true;
  }
  void invalidate() {
    std::lock_guard<std::mutex> lock(mu_);
    valid_ = false;
  }

 private:
  std::mutex mu_;
  bool valid_ = false;
  std::vector<NodeT> nodes_;
  std::vector<uint32_t> indices_;
};

}  // namespace nrt
