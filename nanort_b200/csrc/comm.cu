// Multi-GPU entry points of the C-ABI (include/nanort_b200.h, "multi-GPU"): one process (or thread) per GPU, rays
// sharded by image tile, BVH replicated, ONE collective per frame -- the framebuffer all-gather over NVLink
// (SURVEY.md section 8e).  There is no exchange during traversal, so the collective is NCCL's ncclAllGather on the
// pass's own stream, in place: every rank's accumulate epilogue writes its tiles straight into its slot of the
// gather buffer (tile-major, NRT_AO_PACKED_TILES), the all-gather fills the other slots, and one small kernel of this
// library unpacks tile-major -> the caller's row-major frame.
//
// NCCL is bound at run time (dlopen of libnccl.so.2, preferring a copy the process already loaded, e.g. torch's):
// single-GPU users of libnanort_b200.so need no NCCL at all.
#include <dlfcn.h>
#include <nccl.h>

#include <mutex>
#include <new>
#include <string>

#include "common.cuh"

namespace nrt {

int run_ao_pass_internal(const nrt_accel *h, const nrt_ao_params *pp, float *d_accum, nrt_ao_result *res, void *stream);

namespace {

struct NcclApi {
  void *lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int *) = nullptr;
  std::string error;
};

NcclApi &nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char *n : names) {  // a copy that is already mapped (torch's) first: two NCCLs in one process is asking for trouble
      api.lib = dlopen(n, RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
      if (api.lib) break;
    }
    for (const char *n : names) {
      if (api.lib) break;
      api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    }
    if (!api.lib) {
      api.error = std::string("NCCL not found (dlopen libnccl.so.2): ") + dlerror();
      return;
    }
#define NRT_NCCL_SYM(field, name)                                              \
  api.field = reinterpret_cast<decltype(api.field)>(dlsym(api.lib, name));     \
  if (!api.field && api.error.empty()) api.error = std::string("NCCL symbol missing: ") + name;
    NRT_NCCL_SYM(GetUniqueId, "ncclGetUniqueId")
    NRT_NCCL_SYM(CommInitRank, "ncclCommInitRank")
    NRT_NCCL_SYM(CommDestroy, "ncclCommDestroy")
    NRT_NCCL_SYM(AllGather, "ncclAllGather")
    NRT_NCCL_SYM(GetErrorString, "ncclGetErrorString")
    NRT_NCCL_SYM(GetVersion, "ncclGetVersion")
#undef NRT_NCCL_SYM
  });
  return api;
}

int nccl_fail(ncclResult_t r, const char *what) {
  NcclApi &api = nccl();
  set_error(std::string("NCCL error in ") + what + ": " + (api.GetErrorString ? api.GetErrorString(r) : "?"));
  return NRT_ERR_CUDA;
}

struct Comm {
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1, device = 0;
  float *d_gather = nullptr;  // world x slot_floats, tile-major; slot `rank` is this rank's accumulation target
  size_t gather_floats = 0;
  // recorded after the last kernel of every sharded pass that reads d_gather; the next pass on this communicator
  // waits on it (any stream) before it zeroes its slot.  d_gather, gather_floats and the event are guarded by mu.
  cudaEvent_t gather_done = nullptr;
  std::mutex mu;
};

// tile-major gather buffer -> row-major frame.  Tile t of the image belongs to rank t % world and is that rank's
// (t / world)-th tile (wavefront.cuh:slot_to_pixel), tile_w x tile_h floats each.
__global__ void __launch_bounds__(256)
    unpack_tiles_kernel(const float *__restrict__ gathered, float *__restrict__ frame, uint32_t width, uint32_t height,
                        uint32_t tile_w, uint32_t tile_h, uint32_t world, size_t slot_floats) {
  const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t y = blockIdx.y;
  if (x >= width || y >= height) return;
  const uint32_t tiles_x = (width + tile_w - 1) / tile_w;
  const uint32_t tx = x / tile_w, ty = y / tile_h;
  const uint32_t tile = ty * tiles_x + tx;
  const uint32_t r = tile % world, k = tile / world;
  const size_t src = (size_t)r * slot_floats + (size_t)k * tile_w * tile_h + (size_t)(y - ty * tile_h) * tile_w + (x - tx * tile_w);
  frame[(size_t)y * width + x] = gathered[src];
}

}  // namespace
}  // namespace nrt

using namespace nrt;

extern "C" {

int nrt_comm_unique_id(void *id_128B) {
  if (!id_128B) {
    set_error("nrt_comm_unique_id: NULL argument");
    return NRT_ERR_INVALID;
  }
  NcclApi &api = nccl();
  if (!api.error.empty()) {
    set_error(api.error);
    return NRT_ERR_CUDA;
  }
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclUniqueId id;
  ncclResult_t r = api.GetUniqueId(&id);
  if (r != ncclSuccess) return nccl_fail(r, "ncclGetUniqueId");
  memcpy(id_128B, &id, sizeof(id));
  return NRT_OK;
}

int nrt_comm_init(const void *id_128B, int rank, int world, nrt_comm **out) {
  if (!id_128B || !out || world < 1 || rank < 0 || rank >= world) {
    set_error("nrt_comm_init: bad arguments");
    return NRT_ERR_INVALID;
  }
  *out = nullptr;
  NcclApi &api = nccl();
  if (!api.error.empty()) {
    set_error(api.error);
    return NRT_ERR_CUDA;
  }
  int device = 0;
  DeviceGuard dg_caller;  // ncclCommInitRank binds the communicator to the current device = the calling thread's nrt_set_device
  int rc = select_device(&device);
  if (rc != NRT_OK) return rc;
  Comm *c = new (std::nothrow) Comm();
  if (!c) return NRT_ERR_NOMEM;
  c->rank = rank;
  c->world = world;
  c->device = device;
  ncclUniqueId id;
  memcpy(&id, id_128B, sizeof(id));
  ncclResult_t r = api.CommInitRank(&c->comm, world, id, rank);
  if (r != ncclSuccess) {
    delete c;
    return nccl_fail(r, "ncclCommInitRank");
  }
  *out = reinterpret_cast<nrt_comm *>(c);
  return NRT_OK;
}

void nrt_comm_free(nrt_comm *h) {
  Comm *c = reinterpret_cast<Comm *>(h);
  if (!c) return;
  DeviceGuard dg(c->device);
  cudaDeviceSynchronize();
  if (c->comm && nccl().CommDestroy) nccl().CommDestroy(c->comm);
  cudaFree(c->d_gather);
  if (c->gather_done) cudaEventDestroy(c->gather_done);
  delete c;
}

int nrt_comm_rank(const nrt_comm *h, int *rank, int *world) {
  const Comm *c = reinterpret_cast<const Comm *>(h);
  if (!c) {
    set_error("nrt_comm_rank: NULL communicator");
    return NRT_ERR_INVALID;
  }
  if (rank) *rank = c->rank;
  if (world) *world = c->world;
  return NRT_OK;
}

int nrt_render_ao_sharded(const nrt_accel *accel, nrt_comm *h, const nrt_ao_params *pp, float *d_frame_full,
                          nrt_ao_result *res, void *stream) {
  Comm *c = reinterpret_cast<Comm *>(h);
  if (!accel || !c || !pp || !d_frame_full) {
    set_error("nrt_render_ao_sharded: NULL argument");
    return NRT_ERR_INVALID;
  }
  const Accel *a = reinterpret_cast<const Accel *>(accel);
  if (a->device != c->device) {
    set_error("nrt_render_ao_sharded: accel and communicator live on different devices");
    return NRT_ERR_INVALID;
  }
  nrt_ao_params p = *pp;
  if (p.width == 0 || p.height == 0 || p.tile_w == 0 || p.tile_h == 0) {
    set_error("nrt_render_ao_sharded: bad parameters");
    return NRT_ERR_INVALID;
  }
  p.shard = (uint32_t)c->rank;  // the communicator decides the sharding: tile t -> rank t % world
  p.n_shards = (uint32_t)c->world;
  p.flags = (p.flags & ~NRT_AO_UNFUSED) | NRT_AO_PACKED_TILES;
  NRT_DEVICE(c->device);
  // c->mu orders the enqueueing; gather_done makes this pass wait on the device for the previous pass on this
  // communicator, which may still accumulate into or unpack d_gather on another stream
  std::lock_guard<std::mutex> lock(c->mu);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!c->gather_done) NRT_CUDA(cudaEventCreateWithFlags(&c->gather_done, cudaEventDisableTiming));
  const uint32_t tiles_x = (p.width + p.tile_w - 1) / p.tile_w, tiles_y = (p.height + p.tile_h - 1) / p.tile_h;
  const size_t n_tiles = (size_t)tiles_x * tiles_y;
  const size_t slot_floats = ((n_tiles + c->world - 1) / c->world) * (size_t)p.tile_w * p.tile_h;  // equal for all ranks
  if (c->gather_floats < slot_floats * c->world) {
    NRT_CUDA(cudaEventSynchronize(c->gather_done));
    cudaFree(c->d_gather);
    c->d_gather = nullptr;
    c->gather_floats = 0;
    NRT_CUDA(cudaMalloc(&c->d_gather, sizeof(float) * slot_floats * c->world));
    c->gather_floats = slot_floats * c->world;
  }
  float *mine = c->d_gather + (size_t)c->rank * slot_floats;
  NRT_CUDA(cudaStreamWaitEvent(s, c->gather_done, 0));
  const RecordOnExit gather_done{c->gather_done, s};
  NRT_CUDA(cudaMemsetAsync(mine, 0, sizeof(float) * slot_floats, s));
  int rc = run_ao_pass_internal(accel, &p, mine, res, stream);
  if (rc != NRT_OK) return rc;
  if (c->world > 1) {  // in place: sendbuff == recvbuff + rank * count
    ncclResult_t r = nccl().AllGather(mine, c->d_gather, slot_floats, ncclFloat, c->comm, s);
    if (r != ncclSuccess) return nccl_fail(r, "ncclAllGather");
  }
  dim3 grid((p.width + 255) / 256, p.height);
  unpack_tiles_kernel<<<grid, 256, 0, s>>>(c->d_gather, d_frame_full, p.width, p.height, p.tile_w, p.tile_h,
                                           (uint32_t)c->world, slot_floats);
  NRT_CUDA(cudaGetLastError());
  if (res) res->launches += 1 + (c->world > 1 ? 1 : 0);
  return NRT_OK;
}

}  // extern "C"
