/*
 * nanort_b200_bake.h -- texture-space baking, a C-ABI extension of nanort_b200.h: the reference's uv_raster texel cast
 * (examples/uv_raster/main.cc:687-836) and a cosine AO bake from the texels it covers.
 *
 * Kept in its own header: nanort.h, nanosg.h and nanort_b200.h are the drop-in facade that the reference's own
 * example programs are compiled against, and baking needs nothing from them beyond nanort_b200.h's types.
 */
#ifndef NANORT_B200_BAKE_H_
#define NANORT_B200_BAKE_H_

#include "nanort_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Texel cast of a UV atlas.  `uv` is a triangle accel built (nrt_build / nrt_build_ex) over the UV mesh as
 * SetupVerticesForUVRaster lays it out (main.cc:236-254): vertex k = (u_k, v_k, 0), face i = (3i, 3i+1, 3i+2).
 * Texel (x, y) casts, in float32 and in this order (main.cc:752-770),
 *   org = (r[0] + ((float)x * (r[1] - r[0]) + texel_offset[0]) / (float)width,
 *          r[2] + ((float)y * (r[3] - r[2]) + texel_offset[1]) / (float)height, 1),   r = uv_region
 *   dir = (0, 0, -1), [min_t, max_t) = [0, 1e30), default trace options
 * (the texel offset is not scaled by the region's size, as in the reference) and its record goes to texel
 * py * width + px, px = flip_x ? width - 1 - x : x, py = flip_y ? height - 1 - y : y (main.cc:779-782). */
typedef struct nrt_uv_raster_params {
  uint32_t width, height;
  float uv_region[4];    /* left, right, top, bottom */
  float texel_offset[2]; /* the reference's default is 0.5, 0.5 */
  uint32_t flip_x, flip_y;
  uint32_t flags; /* NRT_TRAVERSE_FAST / NRT_TRAVERSE_CONFORMANCE (reference visiting order), NRT_TRAVERSE_CPP03_INVERSE */
} nrt_uv_raster_params;

/* Writes every texel of d_records_16B (DEVICE, width * height nanort hit records {u, v, t, prim_id}); a texel no
 * triangle covers gets {0, 0, 1e30, 0xFFFFFFFF}.  Optional AOVs (DEVICE float[3 * width * height], NULL to skip), which
 * need `world`, a triangle accel over the mesh in object space with the same face count as `uv`:
 *   d_position_3f  (1 - u - v) v0 + u v1 + v v2 of the world triangle (main.cc:58-60, 808-829)
 *   d_normal_3f    the same interpolation of d_facevarying_normals (DEVICE float[9 * n_faces]), not normalised
 *                  (main.cc:790-806)
 * and are zero on empty texels.  *n_covered (optional; reading it synchronises the stream) receives the number of
 * covered texels.  Calls on one `uv` accel run one after the other on the device, whatever their streams. */
int nrt_uv_raster_device(const nrt_accel *uv, const nrt_accel *world, const nrt_uv_raster_params *p,
                         void *d_records_16B, float *d_position_3f, float *d_normal_3f,
                         const float *d_facevarying_normals, uint64_t *n_covered, void *stream);

/* Cosine AO from every covered texel of nrt_uv_raster_device's records, traced against `world` (the accel whose
 * triangles the records' prim_ids name).  Covered texels are taken in ascending texel order; ray slot i of the call
 * is sample sample0 + i / n_covered of the i % n_covered-th covered texel.  The ray of (texel, sample):
 *   origin     P = (1 - u - v) v0 + u v1 + v v2 of the world triangle (the position AOV)
 *   normal     the triangle's unit geometric normal normalize(cross(v1 - v0, v2 - v0)) as wound; with
 *              d_facevarying_normals (float[9 * n_faces]) flipped to the side of their interpolated value
 *   direction  the AO pass's orthonormal basis + cosine direction about that normal with
 *              u1 = rand_ps(texel, sample, 2, seed), u2 = rand_ps(texel, sample, 3, seed)
 *   range      [ao_min_t, ao_max_t)
 * d_accum[texel] (DEVICE float[width * height]) gains 1 per unoccluded ray; empty texels are not touched.
 * flags: NRT_TRAVERSE_FAST, NRT_TRAVERSE_ANY_HIT, NRT_TRAVERSE_CPP03_INVERSE (NRT_TRAVERSE_CONFORMANCE is refused).
 * The call reads the covered count back (a stream synchronisation) before its first traversal launch, and refuses
 * records whose prim_id is neither 0xFFFFFFFF nor below world's face count.  Bakes and AO / path passes on one accel
 * run one after the other on the device, whatever their streams. */
typedef struct nrt_bake_params {
  uint32_t width, height;
  uint32_t spp, sample0, seed;
  float ao_min_t, ao_max_t;
  uint32_t flags;
  const void *d_facevarying_normals; /* float[9 * n_faces] or NULL */
} nrt_bake_params;

typedef struct nrt_bake_result {
  uint64_t texels;  /* covered texels */
  uint64_t ao_rays; /* texels * spp */
  uint64_t ao_hits; /* occluded AO rays */
  float traverse_ms; /* device time inside the traversal launches (CUDA events) */
  float total_ms;    /* device time of the whole call */
  uint32_t launches, traverse_launches;
} nrt_bake_result;

/* res may be NULL (no read-back of the counters at the end). */
int nrt_bake_ao_device(const nrt_accel *world, const void *d_records_16B, const nrt_bake_params *p, float *d_accum,
                       nrt_bake_result *res, void *stream);

/* The same rays as 36-byte nanort::Ray records in slot order, to a DEVICE buffer of `capacity` records (for tests and
 * benchmarks: nrt_traverse_device or the CPU reference then trace the very same rays).  *n_rays receives
 * n_covered * spp; a call whose rays do not fit writes nothing and returns NRT_ERR_INVALID. */
int nrt_bake_ao_rays_device(const nrt_accel *world, const void *d_records_16B, const nrt_bake_params *p,
                            void *d_rays_36B, uint64_t capacity, uint64_t *n_rays, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NANORT_B200_BAKE_H_ */
