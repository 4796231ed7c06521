/*
 * nanort_b200_lightmap.h -- path-traced lightmaps of UV atlases, a C-ABI extension of nanort_b200_bake.h: the path
 * tracer's bounces (nrt_render_path_device's shading, next-event estimation and Russian roulette) started from every
 * texel that nrt_uv_raster_device's records cover.
 *
 * Kept in its own header, like nanort_b200_bake.h: nanort.h, nanosg.h and nanort_b200.h are the drop-in facade that the
 * reference's own example programs are compiled against.
 */
#ifndef NANORT_B200_LIGHTMAP_H_
#define NANORT_B200_LIGHTMAP_H_

#include "nanort_b200_bake.h"

#ifdef __cplusplus
extern "C" {
#endif

/* A lightmap bake of the covered texels of nrt_uv_raster_device's records (width * height nanort hit records), traced
 * against `world`, the triangle accel whose faces the records' prim_ids name.
 *
 * Covered texels are taken in ascending texel order; path slot i of a call is sample sample0 + i / n_covered of the
 * i % n_covered-th covered texel, and spp paths start at every covered texel.  (texel, sample) keys the random
 * numbers, rand_ps(texel, sample, dim, seed), as (pixel, sample) does in the path pass.
 *
 * Bounce 0, the texel vertex, traces no ray.  Its point P is the position AOV, (1 - u - v) v0 + u v1 + v v2 of the
 * record's world triangle; its normal n is the AO bake's: the unit geometric normal as wound, flipped to the side of the
 * interpolated face-varying normal when d_facevarying_normals is given.  It is shaded as a white Lambertian seen along
 * n: next-event estimation (MeshLight::sampleDirect) from dimensions 8 and 9, and -- when max_bounces > 1 -- a cosine
 * continuation about n from dimensions 10 and 11, the ray {P, ray_min_t} -> {dir, ray_max_t} with weight 1 that does
 * not count emission it hits.  Unlike the path tracer's |cos| at a shading point, a light sample with dot(l, n) <= 0
 * contributes nothing and spawns no shadow ray: the texel receives light from its own hemisphere only.
 * Bounces 1 .. max_bounces - 1 are nrt_render_path_device's radiance and shadow launches, unchanged.
 *
 * d_accum_rgb[3 * texel + c] (DEVICE float[3 * width * height]) gains the sum of the texel's path estimates; a texel
 * no triangle covers is not touched.  d_accum_rgb[texel] / spp estimates E / pi, the outgoing radiance of a white
 * Lambertian receiver at P (irradiance over pi), the texel's own emission not included.  Multiplied by a surface's
 * diffuse albedo it gives that surface's outgoing diffuse radiance.
 *
 * flags: NRT_TRAVERSE_FAST, NRT_TRAVERSE_ANY_HIT (shadow launches only), NRT_TRAVERSE_CPP03_INVERSE; the conformance walk
 * and other bits are refused.  Materials, material ids, emissive faces and face-varying normals are those of
 * nrt_path_params.  The calls read the covered count back (a stream synchronisation) before their first traversal
 * launch and refuse records whose prim_id is neither 0xFFFFFFFF nor below world's face count.  Bakes, AO and path
 * passes on one accel run one after the other on the device, whatever their streams. */
typedef struct nrt_lightmap_params {
  uint32_t width, height; /* the records' atlas */
  uint32_t spp, sample0, seed, max_bounces;
  float ray_min_t, ray_max_t;
  uint32_t n_materials, n_emissive;
  const void *d_materials;           /* float[16] per material, as nrt_path_params */
  const void *d_material_ids;        /* uint32 per face, or NULL (material 0) */
  const void *d_emissive_faces;      /* uint32 face ids, n_emissive of them */
  const void *d_facevarying_normals; /* float[9] per face, or NULL */
  uint32_t flags, pad;
} nrt_lightmap_params;

typedef struct nrt_lightmap_result {
  uint64_t texels;        /* covered texels */
  uint64_t paths;         /* texels * spp */
  uint64_t radiance_rays; /* continuation rays traced (bounces 1 and up) */
  uint64_t shadow_rays;
  float traverse_ms; /* device time inside the traversal launches (CUDA events) */
  float total_ms;    /* device time of the whole call */
  uint32_t launches;
  uint32_t traverse_launches; /* waves * (2 * max_bounces - 1) */
} nrt_lightmap_result;

/* The whole bake, in waves of at most 8 Mi paths.  res may be NULL (no read-back of the counters at the end). */
int nrt_bake_lightmap_device(const nrt_accel *world, const void *d_records_16B, const nrt_lightmap_params *p,
                             float *d_accum_rgb, nrt_lightmap_result *res, void *stream);

/* One bounce of the bake on caller-owned DEVICE queues, as nrt_path_bounce_device, path id = the call's slot.
 * bounce == 0: the texel vertex of paths [0, n_rays), n_rays <= n_covered * spp (the input-queue arguments are
 * ignored); bounce >= 1: traverses and shades the n_rays rays of the input queue.  Continuations go to the output queue
 * (org_tmin, dir_tmax float4 and path id per ray), light samples to the shadow queue (org_tmin, dir_tmax, contribution
 * rgb + texel), d_weight holds float4 {throughput rgb, do_emission} per path id.  Unless skip_shadow_pass, the shadow rays
 * are traced and the visible ones accumulated.  n_rays must be below 2^32, and records that cover no texel are refused
 * (n_rays == 0 returns at once). */
int nrt_bake_lightmap_bounce_device(const nrt_accel *world, const void *d_records_16B, const nrt_lightmap_params *p,
                                    uint32_t bounce, uint64_t n_rays, const void *d_org_tmin, const void *d_dir_tmax,
                                    const uint32_t *d_path_id, void *d_weight, void *d_out_org_tmin,
                                    void *d_out_dir_tmax, uint32_t *d_out_path_id, void *d_sh_org_tmin,
                                    void *d_sh_dir_tmax, void *d_sh_contrib_pix, float *d_accum_rgb,
                                    uint64_t *n_continue, uint64_t *n_shadow, int skip_shadow_pass, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NANORT_B200_LIGHTMAP_H_ */
