// Wavefront pieces shared by render.cu (stand-alone stage kernels) and traverse.cu (the same stages fused
// into the traversal kernel's retire step): ray queues, counter-based RNG, slot -> pixel mapping, AO ray
// construction.  Reference pieces restated here (file:line in the reference's examples/path_tracer):
//   hit point main.cc:860, geometric normal main.cc:306-312 flipped to the viewer main.cc:878-881,
//   orthonormal basis + cosine direction main.cc:216-250, occlusion query main.cc:675-701.
#pragma once
#include "../../include/nanort_b200_bdpt.h"
#include "common.cuh"

namespace nrt {

struct Wave {
  float4 *org_tmin;  // primary queue (SoA): org.xyz, min_t
  float4 *dir_tmax;  //                      dir.xyz, max_t
  Hit16 *hits;
  uint32_t *pix;        // pixel of a primary slot (0xFFFFFFFF = slot outside the image)
  float4 *ao_org_tmin;  // compacted AO queue
  float4 *ao_dir_tmax;
  uint32_t *ao_pix;
  Hit16 *ao_hits;
};

__device__ __forceinline__ uint32_t hash_u32(uint32_t x) {  // lowbias32, same as scenes.py:hash_u32
  x ^= x >> 16;
  x *= 0x7FEB352Du;
  x ^= x >> 15;
  x *= 0x846CA68Bu;
  x ^= x >> 16;
  return x;
}

// scenes.py:rand_ps
__device__ __forceinline__ float rand_ps(uint32_t pix, uint32_t smp, uint32_t dim, uint32_t seed) {
  uint32_t h = hash_u32(pix + seed * 0x9E3779B1u);
  h = hash_u32(h + smp * 0x85EBCA77u + dim * 0xC2B2AE3Du);
  return (float)(h >> 8) * (1.0f / 16777216.0f);
}

// The part of nrt_ao_params / nrt_path_params that maps ray slots to pixels.
struct TileMap {
  uint32_t width, height, spp, sample0, tile_w, tile_h, shard, n_shards;
  uint32_t packed;  // accumulate into a tile-major buffer of this shard's tiles (NRT_AO_PACKED_TILES) instead of the image
};
__host__ __device__ __forceinline__ TileMap tile_map(const nrt_ao_params &p) {
  return TileMap{p.width, p.height, p.spp, p.sample0, p.tile_w, p.tile_h, p.shard, p.n_shards,
                 (p.flags & NRT_AO_PACKED_TILES) ? 1u : 0u};
}
__host__ __device__ __forceinline__ TileMap tile_map(const nrt_path_params &p) {
  return TileMap{p.width, p.height, p.spp, p.sample0, p.tile_w, p.tile_h, p.shard, p.n_shards, 0u};
}

// Division of a 32-bit value by a run-time constant without a divide (Granlund-Montgomery round-up method, exact for
// every uint32 x): the slot -> pixel mapping of a camera ray needs four of them, and an integer division costs more
// instructions than the slab test of a node pair.
struct FastDiv {
  uint32_t d, mul, shift;  // shift == 0xFFFFFFFF: d is 1
  __host__ __device__ FastDiv() : d(1), mul(0), shift(0xFFFFFFFFu) {}
  __host__ explicit FastDiv(uint32_t dd) : d(dd ? dd : 1), mul(0), shift(0xFFFFFFFFu) {
    if (d > 1) {
      uint32_t l = 0;
      while ((1ull << l) < d) l++;  // ceil(log2 d) >= 1
      mul = (uint32_t)(((1ull << 32) * ((1ull << l) - d)) / d + 1ull);
      shift = l - 1;
    }
  }
  __device__ __forceinline__ uint32_t div(uint32_t x) const {
    if (shift == 0xFFFFFFFFu) return x;
    const uint32_t t = __umulhi(mul, x);
    return (t + ((x - t) >> 1)) >> shift;
  }
  __device__ __forceinline__ void divmod(uint32_t x, uint32_t &q, uint32_t &r) const {
    q = div(x);
    r = x - q * d;
  }
};

// Slot -> (pixel, sample).  Slots enumerate this shard's tiles; inside a tile the order is sample-major over
// 8x4 pixel blocks, so the 32 lanes of a warp start as one coherent 8x4 packet.
// `acc` = where the pixel's samples are accumulated: the pixel itself, or -- tile-major packing for the multi-GPU
// gather (comm.cu) -- k * tile_pixels + row-major offset inside the tile.
__device__ __forceinline__ bool slot_to_pixel(const TileMap &p, unsigned long long slot, uint32_t &pix,
                                              uint32_t &smp, uint32_t &acc) {
  const uint32_t tile_pix = p.tile_w * p.tile_h;
  const unsigned long long per_tile = (unsigned long long)tile_pix * p.spp;
  const uint32_t k = (uint32_t)(slot / per_tile);  // k-th tile of this shard
  const uint32_t rem = (uint32_t)(slot % per_tile);
  smp = rem / tile_pix;
  const uint32_t q = rem % tile_pix;
  const uint32_t bw = p.tile_w / 8;  // 8x4 blocks per tile row
  const uint32_t blk = q / 32, in = q % 32;
  const uint32_t bx = blk % bw, by = blk / bw;
  const uint32_t lx = bx * 8 + (in & 7), ly = by * 4 + (in >> 3);
  const uint32_t tiles_x = (p.width + p.tile_w - 1) / p.tile_w;
  const uint32_t tile = k * p.n_shards + p.shard;
  const uint32_t tx = tile % tiles_x, ty = tile / tiles_x;
  const uint32_t x = tx * p.tile_w + lx, y = ty * p.tile_h + ly;
  if (x >= p.width || y >= p.height) return false;
  pix = y * p.width + x;
  acc = p.packed ? k * tile_pix + ly * p.tile_w + lx : pix;
  return true;
}

__device__ __forceinline__ bool slot_to_pixel(const TileMap &p, unsigned long long slot, uint32_t &pix,
                                              uint32_t &smp) {
  uint32_t acc;
  return slot_to_pixel(p, slot, pix, smp, acc);
}

__device__ __forceinline__ bool slot_to_pixel(const nrt_ao_params &p, unsigned long long slot, uint32_t &pix,
                                              uint32_t &smp) {
  return slot_to_pixel(tile_map(p), slot, pix, smp);
}

__device__ __forceinline__ uint32_t slot_sample(const nrt_ao_params &p, unsigned long long slot) {
  const uint32_t tile_pix = p.tile_w * p.tile_h;
  return p.sample0 + (uint32_t)((slot % ((unsigned long long)tile_pix * p.spp)) / tile_pix);
}

// Jittered pinhole camera ray of (pixel, sample) -- examples/path_tracer/main.cc:809-817.  One definition for the
// stand-alone generator kernel, the in-kernel generator (CameraRays) and the AO epilogue, so that all of them
// produce bit-identical rays.
__device__ __forceinline__ void camera_ray(const float *cam, uint32_t width, uint32_t height, uint32_t seed,
                                           uint32_t pix, uint32_t smp, float &dx, float &dy, float &dz) {
  const float jx = rand_ps(pix, smp, 0, seed), jy = rand_ps(pix, smp, 1, seed);
  const float px = (float)(pix % width), py = (float)(pix / width);
  const float sx = (px + jx) / (float)width - 0.5f;
  const float sy = 0.5f - (py + jy) / (float)height;
  dx = cam[3] * sx + cam[6] * sy + cam[9];
  dy = cam[4] * sx + cam[7] * sy + cam[10];
  dz = cam[5] * sx + cam[8] * sy + cam[11];
  const float inv = 1.0f / sqrtf(dx * dx + dy * dy + dz * dz);
  dx *= inv;
  dy *= inv;
  dz *= inv;
}

// Ray "loader" that generates the camera ray of slot (slot0 + i) instead of reading a queue: the primary
// traversal then needs no generator kernel and no primary ray queue at all.  The mapping is slot_to_pixel() with its
// divisions replaced by multiplications (slot0 is a multiple of the per-tile slot count: waves are whole tiles), and
// what the retire step needs again -- direction, pixel, sample, accumulation index -- travels as the ray's payload
// (6 words the kernel parks in thread-local memory) instead of being recomputed.
// SHARED_ORIGIN: the loader's kSharedOrigin, which every ray loader has -- true: all rays start at p.cam[0..2] and the
// launch passes the nodes and triangles relative to that origin (Accel::d_pair_rel / d_tris_rel), so the traversal
// kernel does not subtract it again (traverse3.cuh, from_origin).
template <bool SHARED_ORIGIN>
struct CameraRaysT {
  static constexpr int kPayloadWords = 6;
  static constexpr bool kSharedOrigin = SHARED_ORIGIN;
  nrt_ao_params p;
  uint32_t k0;  // slot0 / per_tile: ordinal (within the shard) of the wave's first tile
  FastDiv per_tile, tile_pix, bw, tiles_x;
  uint32_t packed;
  __host__ CameraRaysT(const nrt_ao_params &pp, unsigned long long slot0) : p(pp) {
    const uint32_t tp = pp.tile_w * pp.tile_h;
    per_tile = FastDiv(tp * pp.spp);
    tile_pix = FastDiv(tp);
    bw = FastDiv(pp.tile_w / 8);
    tiles_x = FastDiv((pp.width + pp.tile_w - 1) / pp.tile_w);
    k0 = (uint32_t)(slot0 / ((unsigned long long)tp * pp.spp));
    packed = (pp.flags & NRT_AO_PACKED_TILES) ? 1u : 0u;
  }
  __device__ __forceinline__ void load(size_t i, float &ox, float &oy, float &oz, float &dx, float &dy, float &dz,
                                       float &tmin, float &tmax, uint32_t *payload) const {
    uint32_t k, rem, smp, q, blk, bx, by, ty, tx;
    per_tile.divmod((uint32_t)i, k, rem);
    k += k0;
    tile_pix.divmod(rem, smp, q);
    blk = q >> 5;
    const uint32_t in = q & 31u;
    bw.divmod(blk, by, bx);
    const uint32_t lx = bx * 8 + (in & 7), ly = by * 4 + (in >> 3);
    tiles_x.divmod(k * p.n_shards + p.shard, ty, tx);
    const uint32_t x = tx * p.tile_w + lx, y = ty * p.tile_h + ly;
    ox = p.cam[0];
    oy = p.cam[1];
    oz = p.cam[2];
    if (x < p.width && y < p.height) {
      const uint32_t pix = y * p.width + x;
      smp += p.sample0;
      // camera_ray() with the pixel coordinates at hand (same arithmetic, same rays bit for bit)
      const float jx = rand_ps(pix, smp, 0, p.seed), jy = rand_ps(pix, smp, 1, p.seed);
      const float sx = ((float)x + jx) / (float)p.width - 0.5f;
      const float sy = 0.5f - ((float)y + jy) / (float)p.height;
      dx = p.cam[3] * sx + p.cam[6] * sy + p.cam[9];
      dy = p.cam[4] * sx + p.cam[7] * sy + p.cam[10];
      dz = p.cam[5] * sx + p.cam[8] * sy + p.cam[11];
      const float inv = 1.0f / sqrtf(dx * dx + dy * dy + dz * dz);
      dx *= inv;
      dy *= inv;
      dz *= inv;
      tmin = p.ray_min_t;
      tmax = p.ray_max_t;
      payload[0] = __float_as_uint(dx);
      payload[1] = __float_as_uint(dy);
      payload[2] = __float_as_uint(dz);
      payload[3] = pix;
      payload[4] = smp;
      payload[5] = packed ? k * tile_pix.d + ly * p.tile_w + lx : pix;
    } else {  // slot outside the image: retires at the root as a miss
      dx = 0.0f;
      dy = 0.0f;
      dz = -1.0f;
      tmin = 0.0f;
      tmax = -1.0f;
      payload[3] = 0xFFFFFFFFu;
    }
  }
};
typedef CameraRaysT<true> CameraRays;      // over the camera-relative copies
typedef CameraRaysT<false> CameraRaysAbs;  // over the accel's own arrays

// Work units of the packet walk (traverse_packet_kernel): one 8x4 block of one tile at K consecutive samples.  Unit u
// of a wave is tile u / per_tile, sample group j and block blk (u % per_tile = j * blocks + blk), and its ray (r, lane)
// is slot  tile * tile_slots + (K * j + r) * tile_pix + blk * 32 + lane  of CameraRaysT's order.  A sample K * j + r
// past spp is no ray (spp not a multiple of K).
template <int K>
struct CameraUnits {
  FastDiv per_tile, blocks;  // units per tile (ceil(spp / K) sample groups of every block), 8x4 blocks per tile
  uint32_t tile_pix, tile_slots, spp;
  __host__ explicit CameraUnits(const nrt_ao_params &p) {
    tile_pix = p.tile_w * p.tile_h;
    tile_slots = tile_pix * p.spp;
    spp = p.spp;
    blocks = FastDiv(tile_pix / 32);
    per_tile = FastDiv((p.spp + K - 1) / K * (tile_pix / 32));
  }
  // units of a wave of n_slots slots (whole tiles)
  __host__ size_t count(size_t n_slots) const { return (n_slots + tile_slots - 1) / tile_slots * per_tile.d; }
  __device__ __forceinline__ bool slot(uint32_t unit, int r, uint32_t lane, uint32_t &s) const {
    uint32_t k, rem, j, blk;
    per_tile.divmod(unit, k, rem);
    blocks.divmod(rem, j, blk);
    const uint32_t smp = (uint32_t)K * j + (uint32_t)r;
    s = k * tile_slots + smp * tile_pix + blk * 32u + lane;
    return smp < spp;
  }
};

// Unit normalize(cross(v1 - v0, v2 - v0)) of a triangle (zero for a degenerate one) and twice its area.
__device__ __forceinline__ void geometric_normal(const float *__restrict__ verts, const uint32_t *__restrict__ faces,
                                                 uint32_t prim, float &nx, float &ny, float &nz, float &area2) {
  const uint32_t f0 = faces[3 * (size_t)prim], f1 = faces[3 * (size_t)prim + 1], f2 = faces[3 * (size_t)prim + 2];
  const float *p0 = verts + 3 * (size_t)f0, *p1 = verts + 3 * (size_t)f1, *p2 = verts + 3 * (size_t)f2;
  const float e1x = p1[0] - p0[0], e1y = p1[1] - p0[1], e1z = p1[2] - p0[2];
  const float e2x = p2[0] - p0[0], e2y = p2[1] - p0[1], e2z = p2[2] - p0[2];
  nx = e1y * e2z - e1z * e2y;
  ny = e1z * e2x - e1x * e2z;
  nz = e1x * e2y - e1y * e2x;
  area2 = sqrtf(nx * nx + ny * ny + nz * nz);
  const float il = area2 > 0.0f ? 1.0f / area2 : 0.0f;
  nx *= il;
  ny *= il;
  nz *= il;
}

// Unit cosine-distributed AO direction about the unit normal n for (pixel or texel, sample): branch-free orthonormal
// basis around n, then the cosine direction from the random dimensions 2 and 3, normalised (main.cc:216-250).  The AO
// spawn and the texel bake both take it.
__device__ __forceinline__ void ao_direction(float nx, float ny, float nz, uint32_t pix, uint32_t smp, uint32_t seed,
                                             float &ox, float &oy, float &oz) {
  const float sg = nz >= 0.0f ? 1.0f : -1.0f;
  const float a = -1.0f / (sg + nz), b = nx * ny * a;
  const float t1x = 1.0f + sg * nx * nx * a, t1y = sg * b, t1z = -sg * nx;
  const float t2x = b, t2y = sg + ny * ny * a, t2z = -ny;
  const float u1 = rand_ps(pix, smp, 2, seed), u2 = rand_ps(pix, smp, 3, seed);
  const float r = sqrtf(u1), ph = 6.28318530718f * u2;
  float sn, cs;
  sincosf(ph, &sn, &cs);
  const float lx = r * cs, ly = r * sn, lz = sqrtf(fmaxf(0.0f, 1.0f - u1));
  const float wx = t1x * lx + t2x * ly + nx * lz, wy = t1y * lx + t2y * ly + ny * lz, wz = t1z * lx + t2z * ly + nz * lz;
  const float il = 1.0f / sqrtf(wx * wx + wy * wy + wz * wz);
  ox = wx * il;
  oy = wy * il;
  oz = wz * il;
}

// One cosine-hemisphere AO ray from a primary hit.  normals[prim]: geometric_normal() of the primitive, computed once
// per accel (Accel::d_face_n), so that the spawn needs one 128-bit load instead of two dependent rounds of gathers.
__device__ __forceinline__ void make_ao_ray(const nrt_ao_params &p, uint32_t pix, uint32_t smp, float4 o, float4 d,
                                            float t, uint32_t prim, const float4 *__restrict__ normals, float4 &o4,
                                            float4 &d4) {
  const float Px = o.x + d.x * t, Py = o.y + d.y * t, Pz = o.z + d.z * t;
  const float4 n = __ldg(normals + prim);
  float nx = n.x, ny = n.y, nz = n.z;
  if (nx * d.x + ny * d.y + nz * d.z > 0.0f) {
    nx = -nx;
    ny = -ny;
    nz = -nz;
  }
  float wx, wy, wz;
  ao_direction(nx, ny, nz, pix, smp, p.seed, wx, wy, wz);
  o4 = make_float4(Px, Py, Pz, p.ao_min_t);
  d4 = make_float4(wx, wy, wz, p.ao_max_t);
}

// ---- retire-step functors of traverse_fast3_kernel.  Called by ALL 32 lanes of a warp (`retiring` says
// whether this lane's ray just finished), so they may use full-mask warp votes.
struct StoreHitsEpilogue {
  static constexpr bool kAnyHit = false;  // true: the kernel retires a ray at its first hit inside [min_t, max_t)
  Hit16 *hits;
  uint8_t *mask;
  __device__ __forceinline__ void operator()(bool retiring, size_t ray_idx, float t, float u, float v, uint32_t prim,
                                             float max_t, const uint32_t *) const {
    if (retiring && hits) {
      const bool hit = t < max_t;  // a hit exactly at max_t is a miss (nanort.h:2552)
      float4 r = hit ? make_float4(u, v, t, __uint_as_float(prim)) : make_float4(0.0f, 0.0f, max_t, __uint_as_float(0xFFFFFFFFu));
      __stcs(reinterpret_cast<float4 *>(hits) + ray_idx, r);  // written once, never re-read by this kernel
      if (mask) mask[ray_idx] = hit ? 1 : 0;
    }
  }
};

// camera rays generated in the kernel (CameraRays): a hit spawns its AO ray straight into the compacted AO queue, a
// miss adds 1 to its pixel.  Pixel and ray come back from the payload the ray loader parked.
struct PrimaryToAoEpilogue {
  static constexpr bool kAnyHit = false;
  nrt_ao_params p;
  Wave w;
  const float4 *normals;
  float *accum;
  unsigned long long *counters;  // [0] AO rays of this wave
  __device__ __forceinline__ void operator()(bool retiring, size_t ray_idx, float t, float u, float v, uint32_t prim,
                                             float max_t, const uint32_t *payload) const {
    (void)u;
    (void)v;
    bool make = false;
    float4 o4 = make_float4(0.f, 0.f, 0.f, 0.f), d4 = o4;
    uint32_t pix = 0xFFFFFFFFu, acc = 0;
    if (retiring) {
      pix = payload[3];  // the camera ray's payload (CameraRays::load): direction, pixel, sample, accumulation index
      if (pix != 0xFFFFFFFFu) {
        const uint32_t smp = payload[4];
        acc = payload[5];
        const float4 ro = make_float4(p.cam[0], p.cam[1], p.cam[2], p.ray_min_t);
        const float4 rd = make_float4(__uint_as_float(payload[0]), __uint_as_float(payload[1]),
                                      __uint_as_float(payload[2]), p.ray_max_t);
        if (t < max_t) {
          make_ao_ray(p, pix, smp, ro, rd, t, prim, normals, o4, d4);
          make = true;
        } else {
          atomicAdd(accum + acc, 1.0f);
        }
      }
    }
    const unsigned m = __ballot_sync(0xFFFFFFFFu, make);
    if (m == 0u) return;
    const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
    unsigned long long base = 0;
    if (lane == leader) base = atomicAdd(counters, (unsigned long long)__popc(m));
    base = __shfl_sync(0xFFFFFFFFu, base, leader);
    if (make) {
      const unsigned long long j = base + __popc(m & ((1u << lane) - 1u));
      w.ao_org_tmin[j] = o4;
      w.ao_dir_tmax[j] = d4;
      w.ao_pix[j] = acc;  // the AO retire step only needs the accumulation index
    }
  }
};

// AO rays: an unoccluded ray adds 1 to its pixel; nothing else is written
struct AoAccumulateEpilogue {
  static constexpr bool kAnyHit = false;
  const uint32_t *ao_pix;
  float *accum;
  unsigned long long *totals;  // [1] occluded AO rays
  __device__ __forceinline__ void operator()(bool retiring, size_t ray_idx, float t, float u, float v, uint32_t prim,
                                             float max_t, const uint32_t *) const {
    (void)u;
    (void)v;
    (void)prim;
    const bool occluded = retiring && (t < max_t);
    if (retiring && !occluded) atomicAdd(accum + ao_pix[ray_idx], 1.0f);
    const unsigned m = __ballot_sync(0xFFFFFFFFu, occluded);
    if (m != 0u && (int)(threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(totals + 1, (unsigned long long)__popc(m));
  }
};

// ------------------------------------------------------------------ texture-space baking (bake.cu)
// texel indices are uint32, and the scan indexes its tiles in uint32
constexpr uint64_t kMaxTexels = 1ull << 31;

// Texel cast of the reference's uv_raster (examples/uv_raster/main.cc:752-770): ray i is texel (i % width, i / width),
// generated at fetch.  Payload: the texel its record goes to, after the flips (main.cc:779-782).
struct TexelRays {
  static constexpr int kPayloadWords = 1;
  static constexpr bool kSharedOrigin = false;
  FastDiv width;
  uint32_t height, flip_x, flip_y;
  float r0, r2, usize, vsize, off0, off1, fw, fh;
  __device__ __forceinline__ void load(size_t i, float &ox, float &oy, float &oz, float &dx, float &dy, float &dz,
                                       float &tmin, float &tmax, uint32_t *payload = nullptr) const {
    uint32_t y, x;
    width.divmod((uint32_t)i, y, x);
    ox = r0 + ((float)x * usize + off0) / fw;
    oy = r2 + ((float)y * vsize + off1) / fh;
    oz = 1.0f;
    dx = 0.0f;
    dy = 0.0f;
    dz = -1.0f;
    tmin = 0.0f;
    tmax = 1.0e30f;
    if (payload) payload[0] = dest(x, y);
  }
  __device__ __forceinline__ uint32_t dest(uint32_t x, uint32_t y) const {
    const uint32_t px = flip_x ? width.d - 1u - x : x, py = flip_y ? height - 1u - y : y;
    return py * width.d + px;
  }
};

// (1 - u - v) a + u b + v c of three float3 at a, b, c (uv_raster's Lerp, main.cc:58-60)
__device__ __forceinline__ void lerp3(const float *a, const float *b, const float *c, float u, float v, float &x,
                                      float &y, float &z) {
  const float w = 1.0f - u - v;
  x = w * a[0] + u * b[0] + v * c[0];
  y = w * a[1] + u * b[1] + v * c[1];
  z = w * a[2] + u * b[2] + v * c[2];
}

// What a texel keeps of its cast: the nanort hit record and, with a world mesh, the position and normal AOVs
// (main.cc:786-829; zeros on an empty texel).  Counts covered texels with one atomic per warp; called by all 32 lanes.
struct TexelStore {
  Hit16 *records;
  float *position, *normal;  // float3 per texel, or nullptr
  const float *verts;        // world mesh (packed float3) and faces, when an AOV is wanted
  const uint32_t *faces;
  const float *fv_normals;  // float[9] per face, for `normal`
  unsigned long long *covered;
  __device__ __forceinline__ void operator()(bool active, uint32_t texel, float t, float u, float v, uint32_t prim,
                                             float max_t) const {
    const bool hit = active && t < max_t;
    if (active) {
      const float4 r = hit ? make_float4(u, v, t, __uint_as_float(prim))
                           : make_float4(0.0f, 0.0f, 1.0e30f, __uint_as_float(0xFFFFFFFFu));
      reinterpret_cast<float4 *>(records)[texel] = r;
      float px = 0.0f, py = 0.0f, pz = 0.0f;
      if (position) {
        if (hit) {
          const uint32_t *f = faces + 3 * (size_t)prim;
          lerp3(verts + 3 * (size_t)f[0], verts + 3 * (size_t)f[1], verts + 3 * (size_t)f[2], u, v, px, py, pz);
        }
        position[3 * (size_t)texel + 0] = px;
        position[3 * (size_t)texel + 1] = py;
        position[3 * (size_t)texel + 2] = pz;
      }
      if (normal) {
        px = py = pz = 0.0f;
        if (hit) {
          const float *n = fv_normals + 9 * (size_t)prim;
          lerp3(n, n + 3, n + 6, u, v, px, py, pz);
        }
        normal[3 * (size_t)texel + 0] = px;
        normal[3 * (size_t)texel + 1] = py;
        normal[3 * (size_t)texel + 2] = pz;
      }
    }
    const unsigned m = __ballot_sync(0xFFFFFFFFu, hit);
    if (m != 0u && (int)(threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(covered, (unsigned long long)__popc(m));
  }
};

struct TexelStoreEpilogue {
  static constexpr bool kAnyHit = false;
  TexelStore store;
  __device__ __forceinline__ void operator()(bool retiring, size_t, float t, float u, float v, uint32_t prim,
                                             float max_t, const uint32_t *payload) const {
    store(retiring, payload[0], t, u, v, prim, max_t);
  }
};

// The surface point of a covered texel: P = the position AOV (lerp3 of the record's world triangle) and the bake's
// normal, the unit geometric normal as wound (Accel::d_face_n), flipped to the side of the interpolated face-varying
// normal when those are given.  The AO bake's rays and the lightmap's texel vertex start here.
__device__ __forceinline__ void texel_point(const float4 *__restrict__ records, const float *__restrict__ verts,
                                            const uint32_t *__restrict__ faces, const float4 *__restrict__ face_n,
                                            const float *__restrict__ fv_normals, uint32_t texel, float &ox, float &oy,
                                            float &oz, float &nx, float &ny, float &nz) {
  const float4 r = __ldg(records + texel);
  const float u = r.x, v = r.y;
  const uint32_t prim = __float_as_uint(r.w);
  const uint32_t *f = faces + 3 * (size_t)prim;
  lerp3(verts + 3 * (size_t)__ldg(f), verts + 3 * (size_t)__ldg(f + 1), verts + 3 * (size_t)__ldg(f + 2), u, v, ox, oy,
        oz);
  const float4 n = __ldg(face_n + prim);
  nx = n.x;
  ny = n.y;
  nz = n.z;
  if (fv_normals) {  // the geometric normal, on the side of the interpolated shading normal
    const float *fn = fv_normals + 9 * (size_t)prim;
    float sx, sy, sz;
    lerp3(fn, fn + 3, fn + 6, u, v, sx, sy, sz);
    if (nx * sx + ny * sy + nz * sz < 0.0f) {
      nx = -nx;
      ny = -ny;
      nz = -nz;
    }
  }
}

// AO rays of the bake: slot i of a launch is sample sample0 + i / n_cov of covered texel texels[i % n_cov], with the
// texel's record (nrt_uv_raster_device) giving the world triangle and the barycentrics.  Payload: the texel.
struct BakeAoRays {
  static constexpr int kPayloadWords = 1;
  static constexpr bool kSharedOrigin = false;
  const uint32_t *texels;  // covered texels, ascending
  const float4 *records;   // Hit16 per texel
  const float *verts;
  const uint32_t *faces;
  const float4 *face_n;      // Accel::d_face_n
  const float *fv_normals;   // float[9] per face, or nullptr
  FastDiv n_cov;
  uint32_t sample0, seed;
  float min_t, max_t;
  __device__ __forceinline__ void load(size_t i, float &ox, float &oy, float &oz, float &dx, float &dy, float &dz,
                                       float &tmin, float &tmax, uint32_t *payload) const {
    uint32_t s, k;
    n_cov.divmod((uint32_t)i, s, k);
    const uint32_t texel = __ldg(texels + k), smp = sample0 + s;
    float nx, ny, nz;
    texel_point(records, verts, faces, face_n, fv_normals, texel, ox, oy, oz, nx, ny, nz);
    ao_direction(nx, ny, nz, texel, smp, seed, dx, dy, dz);
    tmin = min_t;
    tmax = max_t;
    payload[0] = texel;
  }
};

// A bake AO ray: an unoccluded one adds 1 to its texel; occluded ones are counted (one atomic per warp)
struct BakeAccumulateEpilogue {
  static constexpr bool kAnyHit = false;
  float *accum;
  unsigned long long *occluded;
  __device__ __forceinline__ void operator()(bool retiring, size_t, float t, float, float, uint32_t, float max_t,
                                             const uint32_t *payload) const {
    const bool hit = retiring && (t < max_t);
    if (retiring && !hit) atomicAdd(accum + payload[0], 1.0f);
    const unsigned m = __ballot_sync(0xFFFFFFFFu, hit);
    if (m != 0u && (int)(threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(occluded, (unsigned long long)__popc(m));
  }
};

// ------------------------------------------------------------------ path tracing wavefront
struct PathQueues {
  // radiance queue in / out (ping-pong), SoA rays + the path (= primary slot of the wave) each ray belongs to
  float4 *org_tmin[2];
  float4 *dir_tmax[2];
  uint32_t *path_id[2];
  // shadow queue: ray + (contribution.rgb, pixel)
  float4 *sh_org_tmin;
  float4 *sh_dir_tmax;
  float4 *sh_contrib_pix;
  float4 *weight;  // per path: throughput rgb
};

// 16 floats per material, the tinyobj fields the reference reads (main.cc:884-892)
struct PathMaterial {
  float diffuse[3];
  float specular[3];
  float transmittance[3];
  float emission[3];
  float ior;
  float dissolve;
  float pad[2];
};

// Emissive faces of one triangle accel, as MeshLight lists them (main.cc:323-335): the flat pass samples them in place.
struct FlatLights {
  const float *verts;
  const uint32_t *faces;
  const uint32_t *emissive;  // face ids
  const uint32_t *mat_ids;
  const PathMaterial *mats;
  // light `k`: (sample point c0 v0 + c1 v1 + c2 v2) - P, the unit geometric normal, the area and the emission
  __device__ __forceinline__ void sample(uint32_t k, float c0, float c1, float c2, float Px, float Py, float Pz,
                                         float &lx, float &ly, float &lz, float &lnx, float &lny, float &lnz,
                                         float &area, float &ex, float &ey, float &ez) const {
    const uint32_t fid = emissive[k];
    const PathMaterial lm = mats[mat_ids ? mat_ids[fid] : 0u];
    const uint32_t f0 = faces[3 * (size_t)fid], f1 = faces[3 * (size_t)fid + 1], f2 = faces[3 * (size_t)fid + 2];
    const float *v0 = verts + 3 * (size_t)f0, *v1 = verts + 3 * (size_t)f1, *v2 = verts + 3 * (size_t)f2;
    float la2;
    geometric_normal(verts, faces, fid, lnx, lny, lnz, la2);
    area = 0.5f * la2;
    lx = c0 * v0[0] + c1 * v1[0] + c2 * v2[0] - Px;
    ly = c0 * v0[1] + c1 * v1[1] + c2 * v2[1] - Py;
    lz = c0 * v0[2] + c1 * v1[2] + c2 * v2[2] - Pz;
    ex = lm.emission[0];
    ey = lm.emission[1];
    ez = lm.emission[2];
  }
};

// Where the flat pass starts the rays it spawns at a hit: at the hit point, kept off the surface by their min_t.
struct FlatSpawn {
  __device__ __forceinline__ void continuation(const nrt_path_params &p, float Px, float Py, float Pz, float ox,
                                               float oy, float oz, float4 &co, float4 &cd) const {
    co = make_float4(Px, Py, Pz, p.ray_min_t);
    cd = make_float4(ox, oy, oz, p.ray_max_t);
  }
  __device__ __forceinline__ void shadow(const nrt_path_params &, float Px, float Py, float Pz, float lx, float ly,
                                         float lz, float dist, float, float, float, float4 &so, float4 &sd) const {
    so = make_float4(Px, Py, Pz, 0.00001f);
    sd = make_float4(lx, ly, lz, dist - 0.00001f);
  }
};

// The reference's per-hit shading block (examples/path_tracer/main.cc:876-976) for a ray (o, d) that hit at distance t:
// normal flip, material, Fresnel, lobe probabilities, lobe choice, light sample, cosine direction, emission, Russian
// roulette.  (nx, ny, nz) is originalNorm; w the path's throughput + do_emission, written back to *wslot when the path
// continues.  Lights (FlatLights, or the scene pass's world-space records) give the light sample; Spawn places the
// continuation and shadow rays.  Returns in cont / shadow whether this lane appends a continuation or a shadow ray.
// ONE_SIDED: a light sample below the (flipped) normal, dot(l, n) <= 0, contributes nothing and spawns no shadow ray,
// instead of the reference's |cos| -- the lightmap's texel vertex, a receiver that only sees its own hemisphere.
template <class Lights, class Spawn, bool ONE_SIDED = false>
__device__ __forceinline__ void path_shade_hit(const nrt_path_params &p, uint32_t bounce, uint32_t pix, uint32_t smp,
                                               float4 o, float4 d, float t, float nx, float ny, float nz,
                                               const PathMaterial *mat, const Lights &lights, const Spawn &spawn,
                                               float4 w, float4 *wslot, float *accum, bool &cont, bool &shadow,
                                               float4 &co, float4 &cd, float4 &so, float4 &sd, float4 &sc) {
  const float onx = nx, ony = ny, onz = nz;  // originalNorm
  const float ndotd = nx * d.x + ny * d.y + nz * d.z;
  if (ndotd > 0.0f) {  // flip towards the incoming ray (main.cc:878-881)
    nx = -nx;
    ny = -ny;
    nz = -nz;
  }
  const PathMaterial m = *mat;
  // ---- Fresnel and lobe probabilities (main.cc:894-929)
  const float inside = ndotd < 0.0f ? -1.0f : 1.0f;  // sign(dot(rayDir, originalNorm))
  const float n1 = inside < 0.0f ? 1.0f / m.ior : m.ior;
  const float n2 = 1.0f / n1;
  const float r0s = (n1 - n2) / (n1 + n2);
  const float r0 = r0s * r0s;
  const float hdn = 1.0f - (-(d.x * nx + d.y * ny + d.z * nz));
  const float fresnel = r0 + (1.0f - r0) * (hdn * hdn * hdn * hdn * hdn);
  const float third = 1.0f / 3.0f;
  float rhoS = (third * m.specular[0] + third * m.specular[1] + third * m.specular[2]) * fresnel;
  float rhoD = (third * m.diffuse[0] + third * m.diffuse[1] + third * m.diffuse[2]) * (1.0f - fresnel) *
               (1.0f - m.dissolve);
  float rhoR = (third * m.transmittance[0] + third * m.transmittance[1] + third * m.transmittance[2]) *
               (1.0f - fresnel) * m.dissolve;
  float rhoE = third * m.emission[0] + third * m.emission[1] + third * m.emission[2];
  const float total = rhoS + rhoD + rhoR + rhoE;
  if (total < 0.0001f) return;
  rhoS /= total;
  rhoD /= total;
  rhoR /= total;
  const uint32_t dim = 8u + 8u * bounce;
  const float pick = rand_ps(pix, smp, dim + 5, p.seed);
  const float Px = o.x + d.x * t, Py = o.y + d.y * t, Pz = o.z + d.z * t;
  float ox = 0.f, oy = 0.f, oz = 0.f;  // outDir
  bool scatter = true;
  if (pick < rhoS) {  // glossy reflection
    const float k = 2.0f * (d.x * nx + d.y * ny + d.z * nz);
    ox = d.x - k * nx;
    oy = d.y - k * ny;
    oz = d.z - k * nz;
    w.x *= m.specular[0];
    w.y *= m.specular[1];
    w.z *= m.specular[2];
    w.w = 1.0f;
  } else if (pick < rhoS + rhoD) {  // diffuse + next-event estimation
    if (p.n_emissive > 0) {  // MeshLight::sampleDirect (main.cc:337-392)
      float xi1 = rand_ps(pix, smp, dim + 0, p.seed);
      const float xi2 = rand_ps(pix, smp, dim + 1, p.seed);
      const float nf = (float)p.n_emissive;
      const uint32_t face = min((uint32_t)floorf(xi1 * nf), p.n_emissive - 1u);
      xi1 = xi1 * nf - (float)face;
      const float s1 = sqrtf(xi1), c0 = 1.0f - s1, c1 = s1 * (1.0f - xi2), c2 = s1 * xi2;
      float lx, ly, lz, lnx, lny, lnz, area, lex, ley, lez;
      lights.sample(face, c0, c1, c2, Px, Py, Pz, lx, ly, lz, lnx, lny, lnz, area, lex, ley, lez);
      const float dist = sqrtf(lx * lx + ly * ly + lz * lz);
      if (dist > 0.000001f) {
        const float id = 1.0f / dist;
        lx *= id;
        ly *= id;
        lz *= id;
        // The reference traces the shadow ray whenever the solid-angle pdf is positive -- also when the light
        // faces away (cosAtLight = 0 makes PdfAtoW infinite and the contribution exactly 0, main.cc:381-390,
        // 943-950): those Traverse calls are part of its loop, so they are part of ours.
        const float cos_l = fmaxf(-(lx * lnx + ly * lny + lz * lnz), 0.0f);
        const float pdf = (1.0f / nf) * (1.0f / area) * (dist * dist) / fabsf(cos_l);  // PdfAtoW
        const float cos_s = lx * nx + ly * ny + lz * nz;
        if (pdf > 0.0f && (!ONE_SIDED || cos_s > 0.0f)) {
          const float cos_t = fabsf(cos_s);
          const float k = (1.0f / 3.14159265358979f) * cos_l * cos_t / pdf;  // brdf * cosine EDF * cos / pdf
          spawn.shadow(p, Px, Py, Pz, lx, ly, lz, dist, lnx, lny, lnz, so, sd);
          sc = make_float4(k * m.diffuse[0] * lex * w.x, k * m.diffuse[1] * ley * w.y, k * m.diffuse[2] * lez * w.z,
                           __uint_as_float(pix));
          shadow = true;
        }
      }
    }
    // cosine-weighted direction about the flipped normal (main.cc:216-250)
    const float sg = nz >= 0.0f ? 1.0f : -1.0f;
    const float a = -1.0f / (sg + nz), b = nx * ny * a;
    const float t1x = 1.0f + sg * nx * nx * a, t1y = sg * b, t1z = -sg * nx;
    const float t2x = b, t2y = sg + ny * ny * a, t2z = -ny;
    const float u1 = rand_ps(pix, smp, dim + 2, p.seed), u2 = rand_ps(pix, smp, dim + 3, p.seed);
    const float r = sqrtf(u1);
    float sn, cs;
    sincosf(6.28318530718f * u2, &sn, &cs);
    const float hx = r * cs, hy = r * sn, hz = sqrtf(fmaxf(0.0f, 1.0f - u1));
    ox = t1x * hx + t2x * hy + nx * hz;
    oy = t1y * hx + t2y * hy + ny * hz;
    oz = t1z * hx + t2z * hy + nz * hz;
    w.x *= m.diffuse[0];
    w.y *= m.diffuse[1];
    w.z *= m.diffuse[2];
    w.w = 0.0f;
  } else if (pick < rhoD + rhoS + rhoR) {  // refraction: refract(rayDir, -inside * originalNorm, n1)
    const float rnx = -inside * onx, rny = -inside * ony, rnz = -inside * onz;
    const float ndi = rnx * d.x + rny * d.y + rnz * d.z;
    const float k = 1.0f - n1 * n1 * (1.0f - ndi * ndi);
    if (k < 0.0f) {
      ox = oy = oz = 0.0f;  // the reference continues with a zero direction (a ray that hits nothing)
    } else {
      const float c = n1 * ndi + sqrtf(k);
      ox = n1 * d.x - c * rnx;
      oy = n1 * d.y - c * rny;
      oz = n1 * d.z - c * rnz;
    }
    w.x *= m.transmittance[0];
    w.y *= m.transmittance[1];
    w.z *= m.transmittance[2];
    w.w = 1.0f;
  } else {  // emission (cosine EDF), only if the previous event did not sample the lights
    if (w.w != 0.0f) {
      const float c = fmaxf(-(onx * d.x + ony * d.y + onz * d.z), 0.0f);
      atomicAdd(accum + 3 * (size_t)pix + 0, c * m.emission[0] * w.x);
      atomicAdd(accum + 3 * (size_t)pix + 1, c * m.emission[1] * w.y);
      atomicAdd(accum + 3 * (size_t)pix + 2, c * m.emission[2] * w.z);
    }
    scatter = false;
  }
  // ---- continuation + Russian roulette of the NEXT bounce (main.cc:828-837)
  if (scatter && bounce + 1 < p.max_bounces) {
    bool alive = true;
    if (bounce + 1 > 3) {
      alive = rand_ps(pix, smp, dim + 4, p.seed) >= 0.2f;
      const float inv = 1.0f / 0.8f;
      w.x *= inv;
      w.y *= inv;
      w.z *= inv;
    }
    if (alive) {
      spawn.continuation(p, Px, Py, Pz, ox, oy, oz, co, cd);
      *wslot = w;
      cont = true;
    }
  }
}

// Appends this lane's continuation ray (to queue `out`) and shadow ray, one atomic per warp and queue.  Called by all
// 32 lanes of a warp.
__device__ __forceinline__ void path_append(const PathQueues &q, int out, unsigned long long *counters, bool cont,
                                            bool shadow, uint32_t pid, float4 co, float4 cd, float4 so, float4 sd,
                                            float4 sc) {
  const int lane = threadIdx.x & 31;
  const unsigned mc = __ballot_sync(0xFFFFFFFFu, cont), ms = __ballot_sync(0xFFFFFFFFu, shadow);
  if ((mc | ms) == 0u) return;
  unsigned long long bc = 0, bs = 0;
  if (lane == 0) {
    if (mc) bc = atomicAdd(counters + 0, (unsigned long long)__popc(mc));
    if (ms) bs = atomicAdd(counters + 1, (unsigned long long)__popc(ms));
  }
  bc = __shfl_sync(0xFFFFFFFFu, bc, 0);
  bs = __shfl_sync(0xFFFFFFFFu, bs, 0);
  const unsigned lt = (1u << lane) - 1u;
  if (cont) {
    const unsigned long long j = bc + __popc(mc & lt);
    q.org_tmin[out][j] = co;
    q.dir_tmax[out][j] = cd;
    q.path_id[out][j] = pid;
  }
  if (shadow) {
    const unsigned long long j = bs + __popc(ms & lt);
    q.sh_org_tmin[j] = so;
    q.sh_dir_tmax[j] = sd;
    q.sh_contrib_pix[j] = sc;
  }
}

// Slot maps of the radiance retire step: path id -> (pixel or texel, sample), the pair that keys rand_ps and picks the
// accumulation index.  False: the slot carries no path.
// The path pass: slot slot0 + pid of the tile map (slot_to_pixel), samples counted from p.sample0.
struct TileSlots {
  unsigned long long slot0;
  __device__ __forceinline__ bool operator()(const nrt_path_params &p, uint32_t pid, uint32_t &pix, uint32_t &smp) const {
    if (!slot_to_pixel(tile_map(p), slot0 + pid, pix, smp)) return false;
    smp += p.sample0;
    return true;
  }
};

// The lightmap bake: slot s = base + pid of a call is sample p.sample0 + s / n_cov of covered texel texels[s % n_cov].
// The 64-bit wave base enters as base / n_cov (base_sample) and base % n_cov (base_k), so that base_k + pid, below
// 2^31 + 2^23 in a wave and a 32-bit path id at base 0, takes the 32-bit FastDiv.
struct TexelSlots {
  const uint32_t *texels;  // covered texels, ascending
  FastDiv n_cov;
  uint32_t base_k, base_sample;
  __device__ __forceinline__ bool operator()(const nrt_path_params &p, uint32_t pid, uint32_t &texel,
                                             uint32_t &smp) const {
    uint32_t s, k;
    n_cov.divmod(base_k + pid, s, k);
    texel = __ldg(texels + k);
    smp = p.sample0 + base_sample + s;
    return true;
  }
};

// Radiance rays of bounce `bounce`: the retire step is the reference's per-hit shading block
// (examples/path_tracer/main.cc:856-976): normal, then path_shade_hit.
template <class Slots>
struct PathShadeEpilogueT {
  static constexpr bool kAnyHit = false;
  nrt_path_params p;
  Slots slots;
  int in;  // which radiance queue is being traversed; (in ^ 1) receives the continuation rays
  uint32_t bounce;
  PathQueues q;
  const float *verts;
  const uint32_t *faces;
  float *accum;                  // rgb
  unsigned long long *counters;  // [0] continuation rays, [1] shadow rays of this bounce
  __device__ __forceinline__ void operator()(bool retiring, size_t ray_idx, float t, float u, float v, uint32_t prim,
                                             float max_t, const uint32_t *) const {
    bool cont = false, shadow = false;
    float4 co = make_float4(0, 0, 0, 0), cd = co, so = co, sd = co, sc = co;
    uint32_t pid = 0;
    if (retiring && t < max_t) {
      pid = q.path_id[in][ray_idx];
      uint32_t pix, smp;
      if (slots(p, pid, pix, smp)) {
        const float4 o = q.org_tmin[in][ray_idx], d = q.dir_tmax[in][ray_idx];
        const float4 w = q.weight[pid];  // throughput rgb, w.w = do_emission (no light sampling at the previous event)
        const PathMaterial *mats = reinterpret_cast<const PathMaterial *>(p.d_materials);
        const uint32_t *mat_ids = reinterpret_cast<const uint32_t *>(p.d_material_ids);
        const uint32_t *emissive = reinterpret_cast<const uint32_t *>(p.d_emissive_faces);
        const float *fv_normals = reinterpret_cast<const float *>(p.d_facevarying_normals);
        // ---- normal: interpolated face-varying normals when given (main.cc:862-875), else geometric
        float nx, ny, nz, a2;
        if (fv_normals) {
          const float *n0 = fv_normals + 9 * (size_t)prim;
          const float b0 = 1.0f - u - v;
          nx = b0 * n0[0] + u * n0[3] + v * n0[6];
          ny = b0 * n0[1] + u * n0[4] + v * n0[7];
          nz = b0 * n0[2] + u * n0[5] + v * n0[8];
          const float l = sqrtf(nx * nx + ny * ny + nz * nz);
          if (fabsf(l) > 1.0e-6f) {
            const float il = 1.0f / l;
            nx *= il;
            ny *= il;
            nz *= il;
          }
        } else {
          // no normals given: the flat normal the example's loader stores for such a mesh, calcNormal's
          // cross(v2 - v0, v1 - v0) (main.cc:306-312, 566-601) -- the opposite of cross(e1, e2)
          geometric_normal(verts, faces, prim, nx, ny, nz, a2);
          nx = -nx;
          ny = -ny;
          nz = -nz;
        }
        path_shade_hit(p, bounce, pix, smp, o, d, t, nx, ny, nz, mats + (mat_ids ? mat_ids[prim] : 0u),
                       FlatLights{verts, faces, emissive, mat_ids, mats}, FlatSpawn{}, w, q.weight + pid, accum, cont,
                       shadow, co, cd, so, sd, sc);
      }
    }
    path_append(q, in ^ 1, counters, cont, shadow, pid, co, cd, so, sd, sc);
  }
};
typedef PathShadeEpilogueT<TileSlots> PathShadeEpilogue;    // the path pass (path.cu)
typedef PathShadeEpilogueT<TexelSlots> LightmapShadeEpilogue;  // the lightmap bake's bounces 1 and up (lightmap.cu)

// Bounce 0 of the lightmap bake for path `pid`: no ray is traced.  The texel's surface point (texel_point) is shaded
// by path_shade_hit as a white Lambertian seen along its normal -- a ray (P, -n) that hit at t = 0, whose lobe choice
// is then always the diffuse one with albedo (1, 1, 1): next-event estimation from random dimensions 8 and 9, a cosine
// continuation from 10 and 11 with weight 1 and do_emission 0.  ONE_SIDED: a light sample below the texel's
// hemisphere contributes nothing and spawns no shadow ray.  Returns the appends as path_shade_hit does.
__device__ __forceinline__ void lightmap_texel_vertex(const nrt_path_params &p, const TexelSlots &slots, uint32_t pid,
                                                      const float4 *records, const float *verts, const uint32_t *faces,
                                                      const float4 *face_n, float4 *wslot, float *accum, bool &cont,
                                                      bool &shadow, float4 &co, float4 &cd, float4 &so, float4 &sd,
                                                      float4 &sc) {
  uint32_t texel, smp;
  slots(p, pid, texel, smp);
  float Px, Py, Pz, nx, ny, nz;
  texel_point(records, verts, faces, face_n, reinterpret_cast<const float *>(p.d_facevarying_normals), texel, Px, Py,
              Pz, nx, ny, nz);
  PathMaterial white = {};
  white.diffuse[0] = white.diffuse[1] = white.diffuse[2] = 1.0f;
  white.ior = 1.0f;
  const PathMaterial *mats = reinterpret_cast<const PathMaterial *>(p.d_materials);
  const uint32_t *mat_ids = reinterpret_cast<const uint32_t *>(p.d_material_ids);
  const uint32_t *emissive = reinterpret_cast<const uint32_t *>(p.d_emissive_faces);
  path_shade_hit<FlatLights, FlatSpawn, true>(
      p, 0u, texel, smp, make_float4(Px, Py, Pz, p.ray_min_t), make_float4(-nx, -ny, -nz, p.ray_max_t), 0.0f, nx, ny,
      nz, &white, FlatLights{verts, faces, emissive, mat_ids, mats}, FlatSpawn{}, make_float4(1.0f, 1.0f, 1.0f, 1.0f),
      wslot, accum, cont, shadow, co, cd, so, sd, sc);
}

// Shadow rays: an unoccluded light sample adds its contribution (CheckForOccluder returned false)
struct ShadowAccumulateEpilogue {
  static constexpr bool kAnyHit = false;
  const float4 *contrib_pix;
  float *accum;
  __device__ __forceinline__ void operator()(bool retiring, size_t ray_idx, float t, float u, float v, uint32_t prim,
                                             float max_t, const uint32_t *) const {
    (void)u;
    (void)v;
    (void)prim;
    if (retiring && !(t < max_t)) {
      const float4 c = contrib_pix[ray_idx];
      const size_t pix = __float_as_uint(c.w);
      atomicAdd(accum + 3 * pix + 0, c.x);
      atomicAdd(accum + 3 * pix + 1, c.y);
      atomicAdd(accum + 3 * pix + 2, c.z);
    }
  }
};

// ------------------------------------------------------------------ bidirectional path tracing (bdpt.cu)
// The reference's examples/bidir_path_tracer/main.cc restated in float32 with its operation order (the library is
// compiled with --fmad=false).  float3 is the reference's float3: `f * v` and `v * f` both round v.x * f, `v / f`
// divides each component.
namespace bd {

constexpr float kEps = 0.001f;
constexpr float kInf = 1.0e30f;
constexpr float kPi = 3.14159274101257324f;  // 4.0f * std::atan(1.0f)
constexpr uint32_t kNone = 0xFFFFFFFFu;

__device__ __forceinline__ float3 f3(float x, float y, float z) { return make_float3(x, y, z); }
__device__ __forceinline__ float3 f3(const float *p) { return make_float3(p[0], p[1], p[2]); }
__device__ __forceinline__ float3 add(float3 a, float3 b) { return f3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float3 sub(float3 a, float3 b) { return f3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float3 mul(float3 a, float3 b) { return f3(a.x * b.x, a.y * b.y, a.z * b.z); }
__device__ __forceinline__ float3 mul(float3 v, float f) { return f3(v.x * f, v.y * f, v.z * f); }
__device__ __forceinline__ float3 div(float3 v, float f) { return f3(v.x / f, v.y / f, v.z / f); }
__device__ __forceinline__ float3 neg(float3 v) { return f3(-v.x, -v.y, -v.z); }
__device__ __forceinline__ float dot(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float3 cross(float3 a, float3 b) {
  return f3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
__device__ __forceinline__ float length(float3 v) { return sqrtf(v.x * v.x + v.y * v.y + v.z * v.z); }
// float3::normalize: the threshold test and 1.0 / len in double (main.cc:218-226)
__device__ __forceinline__ float3 normalize(float3 v) {
  const float len = length(v);
  if (fabs((double)len) > 1.0e-6) {
    const float inv = (float)(1.0 / (double)len);
    v = mul(v, inv);
  }
  return v;
}
__device__ __forceinline__ bool black(float3 v) { return v.x == 0.0f && v.y == 0.0f && v.z == 0.0f; }
__device__ __forceinline__ float fmax0(float x) { return 0.0f < x ? x : 0.0f; }  // std::max(0.0f, x)

// Random (main.cc:132-157): xorshift128 seeded by the reference's recurrence; nextReal can return 1.0f
struct Random {
  uint32_t s[4];
  __device__ __forceinline__ void seed(uint32_t x) {
#pragma unroll
    for (int i = 1; i <= 4; i++) s[i - 1] = x = 1812433253u * (x ^ (x >> 30)) + (uint32_t)i;
  }
  __device__ __forceinline__ uint32_t next() {
    const uint32_t t = s[0] ^ (s[0] << 11);
    s[0] = s[1];
    s[1] = s[2];
    s[2] = s[3];
    return s[3] = (s[3] ^ (s[3] >> 19)) ^ (t ^ (t >> 8));
  }
  __device__ __forceinline__ float real() { return (float)next() / 4294967296.0f; }  // (float)UINT_MAX
};

__device__ __forceinline__ bool is_delta(const PathMaterial *m) {  // Vertex::isDelta; no material: not delta
  if (!m) return false;
  return m->specular[0] != 0.0f || m->specular[1] != 0.0f || m->specular[2] != 0.0f ||
         m->transmittance[0] != 0.0f || m->transmittance[1] != 0.0f || m->transmittance[2] != 0.0f;
}

// The Fresnel factor and lobe probabilities shared by Vertex::f, sampleBRDF and pdfBRDF (main.cc:641-665, 782-808,
// 846-870).  Returns totalrho; the rho are normalised only when it is >= 0.0001f.
__device__ __forceinline__ float lobes(const PathMaterial &m, float3 wo, float3 on, float3 n, float &rhoS, float &rhoD,
                                       float &rhoR, float &inside, float &n1) {
  const float dd = dot(neg(wo), on);
  inside = dd < 0 ? -1.0f : 1.0f;  // sign()
  n1 = inside < 0 ? (float)(1.0 / (double)m.ior) : m.ior;
  const float n2 = (float)(1.0 / (double)n1);
  const float r0s = (n1 - n2) / (n1 + n2);
  const float r0 = r0s * r0s;  // fresnel_schlick
  const float c = 1.0f - dot(wo, n);
  const float fresnel = r0 + (1.0f - r0) * (c * c * c * c * c);
  const float3 third = f3(1.0f / 3.0f, 1.0f / 3.0f, 1.0f / 3.0f);
  rhoS = dot(third, f3(m.specular)) * fresnel;
  rhoD = (float)((double)dot(third, f3(m.diffuse)) * (1.0 - (double)fresnel) * (1.0 - (double)m.dissolve));
  rhoR = (float)((double)dot(third, f3(m.transmittance)) * (1.0 - (double)fresnel) * (double)m.dissolve);
  const float total = rhoS + rhoD + rhoR;
  if (!(total < 0.0001f)) {
    rhoS /= total;
    rhoD /= total;
    rhoR /= total;
  }
  return total;
}

// Vertex::f (main.cc:634-689) of vertex (p, on, n, wo, material m) towards position q
__device__ __forceinline__ float3 vertex_f(const nrt_bdpt_vertex &v, const PathMaterial *m, float3 q) {
  const float3 n = f3(v.norm), wo = f3(v.wo);
  const float3 wi = sub(q, f3(v.position));
  const bool refl = dot(wi, n) * dot(wo, n) > 0.0f;
  const PathMaterial mm = m ? *m : PathMaterial{};
  float rhoS, rhoD, rhoR, inside, n1;
  if (lobes(mm, wo, f3(v.original_norm), n, rhoS, rhoD, rhoR, inside, n1) < 0.0001f) return f3(0.0f, 0.0f, 0.0f);
  float3 ret = f3(0.0f, 0.0f, 0.0f);
  float weight = 0.0f;
  if (rhoS > 0.0f && refl) {
    ret = add(ret, mul(f3(0.0f, 0.0f, 0.0f), rhoS));
    weight += rhoS;
  }
  if (rhoD > 0.0f && refl) {
    ret = add(ret, div(mul(f3(mm.diffuse), rhoD), kPi));
    weight += rhoD;
  }
  if (rhoR > 0.0f && !refl) {
    ret = add(ret, mul(f3(0.0f, 0.0f, 0.0f), rhoR));
    weight += rhoR;
  }
  if (weight != 0.0f) ret = div(ret, weight);
  return ret;
}

// pdfBRDF (main.cc:839-886); no material: 0
__device__ __forceinline__ float pdf_brdf(const PathMaterial *m, float3 wi, float3 wo, float3 on, float3 n) {
  const bool refl = dot(wi, n) * dot(wo, n) > 0.0f;
  const PathMaterial mm = m ? *m : PathMaterial{};
  float rhoS, rhoD, rhoR, inside, n1;
  if (lobes(mm, wo, on, n, rhoS, rhoD, rhoR, inside, n1) < 0.0001f) return 0.0f;
  float pdf = 0.0f;
  if (rhoS > 0.0f && refl) pdf += 0.0f;
  if (rhoD > 0.0f && refl) pdf += rhoD * fabsf(dot(wi, n)) / kPi;
  if (rhoR > 0.0f && !refl) pdf += 0.0f;
  return pdf;
}

// directionCosTheta (main.cc:264-280): 2.0 * kPi * u2, sqrt(u1) and 1.0 - u1 in double; cosf / sinf as the correctly
// rounded cos / sin of the float phi
__device__ __forceinline__ float3 direction_cos_theta(float3 n, float u1, float u2, float &pdf) {
  const float phi = (float)(2.0 * (double)kPi * (double)u2);
  const float r = (float)sqrt((double)u1);
  const float x = r * (float)cos((double)phi);
  const float y = r * (float)sin((double)phi);
  const float z = sqrtf((float)(1.0 - (double)u1));
  pdf = z / kPi;
  float3 xd = fabsf(n.x) < fabsf(n.y) ? f3(1.0f, 0.0f, 0.0f) : f3(0.0f, 1.0f, 0.0f);
  const float3 yd = normalize(cross(n, xd));
  xd = cross(yd, n);
  return add(add(mul(xd, x), mul(yd, y)), mul(n, z));
}

// sampleBRDF (main.cc:776-837).  The diffuse lobe's directionCosTheta(norm, rng.nextReal(), rng.nextReal(), pdf) draws
// its arguments right to left, as GCC on x86-64 evaluates them: u2 first.
__device__ __forceinline__ float3 sample_brdf(const PathMaterial &m, float3 wo, float3 on, float3 n, Random &rng,
                                              float3 &wi, float &pdf) {
  float rhoS, rhoD, rhoR, inside, n1;
  if (lobes(m, wo, on, n, rhoS, rhoD, rhoR, inside, n1) < 0.0001f) {
    pdf = 0.0f;
    return f3(0.0f, 0.0f, 0.0f);
  }
  float3 f = f3(0.0f, 0.0f, 0.0f);
  const float rnd = rng.real();
  pdf = 0.0f;
  if (rnd < rhoS) {
    const float3 I = neg(wo);
    wi = sub(I, mul(n, 2.0f * dot(I, n)));  // reflect
    const float c = fabsf(dot(wi, n));
    if (c >= kEps) {
      pdf = rhoS;
      f = div(mul(f3(m.specular), rhoS), c);
    }
  } else if (rnd < rhoS + rhoD) {
    const float u2 = rng.real();
    const float u1 = rng.real();
    wi = direction_cos_theta(n, u1, u2, pdf);
    pdf *= rhoD;
    f = div(mul(f3(m.diffuse), rhoD), kPi);
  } else if (rnd < rhoD + rhoS + rhoR) {
    const float3 I = neg(wo), N = mul(on, -inside);  // refract(-wo, -inside * origNorm, n1)
    const float ndi = dot(N, I);
    const float k = 1.0f - n1 * n1 * (1.0f - ndi * ndi);
    wi = k < 0.0f ? f3(0.0f, 0.0f, 0.0f) : sub(mul(I, n1), mul(N, n1 * ndi + sqrtf(k)));
    const float c = fabsf(dot(wi, n));
    if (c >= kEps) {
      pdf = rhoR;
      f = div(mul(f3(m.transmittance), rhoR), c);
    }
  }
  return f;
}

// What the stage kernels and retire steps read of the mesh and its lights.
struct Scene {
  const PathMaterial *mats;
  const uint32_t *mat_ids;
  const float *fv_normals;  // float[9] per face
  const float *verts;
  const uint32_t *faces;
  const float *cdf;          // LightSampler::cdf_
  const uint32_t *light_ids; // LightSampler::ids_
  const float *total_area;   // LightSampler::totalArea_ (device scalar)
  uint32_t n_lights, n_materials;
  __device__ __forceinline__ const PathMaterial *mat(uint32_t id) const { return id == kNone ? nullptr : mats + id; }
};

// Per sample: the ray about to be traced and what raytrace keeps between bounces, and the sample's generator
struct PathState {
  float4 org_pdf;  // rayOrg, pdfFwd
  float4 dir;      // rayDir
  float4 beta;
  uint4 rng;
};

// Pass layout of a wave: vertex records of sample `slot` at verts + slot * stride
struct Subpaths {
  nrt_bdpt_vertex *eye, *light;
  uint32_t *n_eye, *n_light;
  uint32_t stride;  // max_bounces + 1
};

__device__ __forceinline__ void vstore(nrt_bdpt_vertex &d, float3 p, float3 on, float3 n, float3 beta, float3 wo,
                                       float pdf_fwd, float pdf_rev, uint32_t type, uint32_t mat, uint32_t prim) {
  nrt_bdpt_vertex v;
  v.position[0] = p.x, v.position[1] = p.y, v.position[2] = p.z;
  v.original_norm[0] = on.x, v.original_norm[1] = on.y, v.original_norm[2] = on.z;
  v.norm[0] = n.x, v.norm[1] = n.y, v.norm[2] = n.z;
  v.beta[0] = beta.x, v.beta[1] = beta.y, v.beta[2] = beta.z;
  v.wo[0] = wo.x, v.wo[1] = wo.y, v.wo[2] = wo.z;
  v.pdf_fwd = pdf_fwd;
  v.pdf_rev = pdf_rev;
  v.type = type;
  v.material = mat;
  v.prim_id = prim;
  d = v;
}

// The interpolated shading normal of a hit (main.cc:954-957): (1.0 - u - v) in double, the reference's normalize
__device__ __forceinline__ float3 hit_normal(const float *fn, float u, float v) {
  const float w = (float)(1.0 - (double)u - (double)v);
  return normalize(add(add(mul(f3(fn), w), mul(f3(fn + 3), u)), mul(f3(fn + 6), v)));
}

// Where the flat pass starts a subpath's next ray: at the vertex (min_t keeps it off the surface)
struct FlatOrigin {
  __device__ __forceinline__ float3 operator()(float3 p, float3) const { return p; }
};

// raytrace's per-hit block (main.cc:925-1011) for a ray of subpath `verts` (n vertices so far) that hit at `next`,
// with shading normal nrm, on face `prim` of material `mid`.  Appends the vertex (unless a light subpath hit a
// light), converts its pdfFwd, samples the BRDF with the sample's generator, writes prev.pdfRev and the next ray into
// st; origin(next, direction) is where that ray starts.  Returns whether the subpath traces another ray.
template <class Origin>
__device__ __forceinline__ bool subpath_vertex(const Scene &sc, bool eye, uint32_t max_bounces, PathState &st,
                                               nrt_bdpt_vertex *verts, uint32_t &n, float3 next, float3 nrm,
                                               uint32_t mid, uint32_t prim, const Origin &origin) {
  const float3 dir = f3(st.dir.x, st.dir.y, st.dir.z);
  float3 beta = f3(st.beta.x, st.beta.y, st.beta.z);
  const float3 on = nrm;
  if (dot(nrm, dir) > 0) nrm = mul(nrm, -1.0f);
  const PathMaterial m = sc.mats[mid];
  const bool light = m.emission[0] != 0.0f || m.emission[1] != 0.0f || m.emission[2] != 0.0f;  // isLight
  if (light && !eye) return false;
  if (light) beta = mul(mul(beta, f3(m.emission)), fmax0(dot(on, neg(dir))));
  const nrt_bdpt_vertex prev = verts[n - 1];
  float3 to = sub(next, f3(prev.position));
  const float dist = length(to);
  to = div(to, dist);
  const float pdf_fwd = st.org_pdf.w * (dot(to, f3(prev.norm)) / (dist * dist));
  vstore(verts[n], next, on, nrm, beta, normalize(neg(dir)), pdf_fwd, 0.0f, light ? NRT_BDPT_LIGHT : NRT_BDPT_SURFACE,
         mid, prim);
  const uint32_t b = n - 1;  // raytrace's loop counter
  n++;
  if (light) return false;
  Random rng;
  rng.s[0] = st.rng.x, rng.s[1] = st.rng.y, rng.s[2] = st.rng.z, rng.s[3] = st.rng.w;
  float3 out = f3(0.0f, 0.0f, 0.0f);
  float pdf;
  const float3 f = sample_brdf(m, neg(dir), on, nrm, rng, out, pdf);
  st.rng = make_uint4(rng.s[0], rng.s[1], rng.s[2], rng.s[3]);
  if (pdf == 0.0f) return false;
  beta = div(mul(mul(f, beta), fabsf(dot(nrm, out))), pdf);
  if (black(beta)) return false;
  const float pdf_rev = pdf_brdf(&m, out, neg(dir), on, nrm);
  const float3 o = origin(next, out);
  st.org_pdf = make_float4(o.x, o.y, o.z, pdf);
  st.dir = make_float4(out.x, out.y, out.z, 0.0f);
  st.beta = make_float4(beta.x, beta.y, beta.z, 0.0f);
  verts[n - 2].pdf_rev = pdf_rev * fabsf(dot(neg(to), nrm)) / (dist * dist);
  return b + 1 < max_bounces;
}

// subpath_vertex for a ray of the flat mesh that hit `prim` at t: P = org + t dir, the face's normals and material
__device__ __forceinline__ bool subpath_hit(const Scene &sc, bool eye, uint32_t max_bounces, PathState &st,
                                            nrt_bdpt_vertex *verts, uint32_t &n, float t, float u, float v,
                                            uint32_t prim) {
  const float3 org = f3(st.org_pdf.x, st.org_pdf.y, st.org_pdf.z), dir = f3(st.dir.x, st.dir.y, st.dir.z);
  const float3 next = add(org, mul(dir, t));
  return subpath_vertex(sc, eye, max_bounces, st, verts, n, next, hit_normal(sc.fv_normals + 9 * (size_t)prim, u, v),
                        sc.mat_ids[prim], prim, FlatOrigin{});
}

// One connection of connectPath (main.cc:1263-1283): eye vertex e - 1 and light vertex l - 1 of sample `slot`, its
// unshadowed L and its weightMIS; the retire step of its calcG ray turns L into mis * (L * G).
struct Conn {
  uint32_t slot;
  uint32_t el;  // e | l << 16
  float L[3];
  float mis;
};
static_assert(sizeof(Conn) == 24, "Conn");

// calcG's ray (main.cc:1215-1227): from the eye vertex towards the light vertex, [kEps, kInf)
__device__ __forceinline__ void conn_ray(float3 pe, float3 pl, float3 &to, float &dist) {
  to = sub(pl, pe);
  dist = length(to);
  to = div(to, dist);
}

// calcG's cosines and 1 / dist^2 (main.cc:1237-1243) of a visible connection
__device__ __forceinline__ float g_term(float3 to, float dist, float3 ne, float3 nl) {
  const float d1 = fmax0(dot(to, ne)), d2 = fmax0(dot(neg(to), nl));
  return d1 * d2 / (dist * dist);
}

// calcG's test and cosines (main.cc:1233-1243) from the closest hit at t (hit: t < max_t)
__device__ __forceinline__ float calc_g(float3 to, float dist, float3 ne, float3 nl, bool hit, float t) {
  if (!hit) return 0.0f;
  if (fabsf(dist - t) > kEps) return 0.0f;
  return g_term(to, dist, ne, nl);
}

// A traced connection: L becomes mis * (L * G) in place
__device__ __forceinline__ void conn_finish(Conn &c, float G) {
  const float mis = c.mis;
  c.L[0] = (c.L[0] * G) * mis;
  c.L[1] = (c.L[1] * G) * mis;
  c.L[2] = (c.L[2] * G) * mis;
}

// Ray loader of the connection launch: the ray is rebuilt from the record's two vertices at fetch
struct ConnRays {
  static constexpr int kPayloadWords = 0;
  static constexpr bool kSharedOrigin = false;
  const Conn *conns;
  Subpaths sp;
  __device__ __forceinline__ void load(size_t i, float &ox, float &oy, float &oz, float &dx, float &dy, float &dz,
                                       float &tmin, float &tmax, uint32_t * = nullptr) const {
    const uint32_t slot = __ldg(&conns[i].slot), el = __ldg(&conns[i].el);
    const float *pe = sp.eye[(size_t)slot * sp.stride + (el & 0xFFFFu) - 1].position;
    const float *pl = sp.light[(size_t)slot * sp.stride + (el >> 16) - 1].position;
    float3 to;
    float dist;
    conn_ray(f3(pe), f3(pl), to, dist);
    ox = pe[0];
    oy = pe[1];
    oz = pe[2];
    dx = to.x;
    dy = to.y;
    dz = to.z;
    tmin = kEps;
    tmax = kInf;
  }
};

// Connection retire step: L becomes mis * (L * G) in place
struct ConnEpilogue {
  static constexpr bool kAnyHit = false;
  Conn *conns;
  Subpaths sp;
  __device__ __forceinline__ void operator()(bool retiring, size_t ray_idx, float t, float, float, uint32_t,
                                             float max_t, const uint32_t *) const {
    if (!retiring) return;
    Conn &c = conns[ray_idx];
    const uint32_t slot = c.slot, el = c.el;
    const nrt_bdpt_vertex &ev = sp.eye[(size_t)slot * sp.stride + (el & 0xFFFFu) - 1];
    const nrt_bdpt_vertex &lv = sp.light[(size_t)slot * sp.stride + (el >> 16) - 1];
    float3 to;
    float dist;
    conn_ray(f3(ev.position), f3(lv.position), to, dist);
    conn_finish(c, calc_g(to, dist, f3(ev.norm), f3(lv.norm), t < max_t, t));
  }
};

// Ray loader of a subpath bounce: the queued sample's next ray
struct BounceRays {
  static constexpr int kPayloadWords = 0;
  static constexpr bool kSharedOrigin = false;
  const uint32_t *queue;
  const PathState *st;
  __device__ __forceinline__ void load(size_t i, float &ox, float &oy, float &oz, float &dx, float &dy, float &dz,
                                       float &tmin, float &tmax, uint32_t * = nullptr) const {
    const uint32_t slot = __ldg(queue + i);
    const float4 o = __ldg(&st[slot].org_pdf), d = __ldg(&st[slot].dir);
    ox = o.x;
    oy = o.y;
    oz = o.z;
    dx = d.x;
    dy = d.y;
    dz = d.z;
    tmin = kEps;
    tmax = kInf;
  }
};

// Appends `slot` to a queue, one atomic per warp; called by all 32 lanes
__device__ __forceinline__ void queue_append(uint32_t *queue, unsigned long long *count, bool put, uint32_t slot) {
  const unsigned m = __ballot_sync(0xFFFFFFFFu, put);
  if (m == 0u) return;
  const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
  unsigned long long base = 0;
  if (lane == leader) base = atomicAdd(count, (unsigned long long)__popc(m));
  base = __shfl_sync(0xFFFFFFFFu, base, leader);
  if (put) queue[base + __popc(m & ((1u << lane) - 1u))] = slot;
}

// Subpath bounce retire step: raytrace's per-hit block; a miss ends the subpath
struct BounceEpilogue {
  static constexpr bool kAnyHit = false;
  Scene sc;
  Subpaths sp;
  PathState *st;
  const uint32_t *queue_in;
  uint32_t *queue_out;
  unsigned long long *count_out;
  uint32_t max_bounces;
  int eye;
  __device__ __forceinline__ void operator()(bool retiring, size_t ray_idx, float t, float u, float v, uint32_t prim,
                                             float max_t, const uint32_t *) const {
    bool cont = false;
    uint32_t slot = 0;
    if (retiring && t < max_t) {
      slot = queue_in[ray_idx];
      PathState s = st[slot];
      uint32_t *np = (eye ? sp.n_eye : sp.n_light) + slot;
      uint32_t n = *np;
      cont = subpath_hit(sc, eye != 0, max_bounces, s, (eye ? sp.eye : sp.light) + (size_t)slot * sp.stride, n, t, u,
                         v, prim);
      *np = n;
      st[slot] = s;
    }
    queue_append(queue_out, count_out, cont, slot);
  }
};

}  // namespace bd

// NRT_TRAVERSE_ANY_HIT: the same retire steps on rays the kernel stops at their first hit
template <class E>
struct AnyHit : E {
  static constexpr bool kAnyHit = true;
  __host__ __device__ explicit AnyHit(const E &e) : E(e) {}
};

}  // namespace nrt
