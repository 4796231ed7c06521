/*
 * nanort_b200_scene_bake.h -- texture-space baking of two-level scenes, a C-ABI extension of nanort_b200_lightmap.h and
 * nanort_b200_scene_path.h: the texel cast, the AO bake and the lightmap bake over an instanced scene, each instance
 * baking into its own rectangle ("chart") of one shared atlas, without flattening the scene.
 *
 * Kept in its own header, like nanort_b200_bake.h: nanort.h, nanosg.h and nanort_b200.h are the drop-in facade that the
 * reference's own example programs are compiled against.
 */
#ifndef NANORT_B200_SCENE_BAKE_H_
#define NANORT_B200_SCENE_BAKE_H_

#include "nanort_b200_lightmap.h"
#include "nanort_b200_scene_path.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One instance's chart: its rectangle of the atlas and the texel cast that fills it. */
typedef struct nrt_scene_chart {
  const nrt_accel *uv;            /* UV mesh of this instance's accel in SetupVerticesForUVRaster's layout, or NULL: no chart */
  uint32_t x0, y0, width, height; /* the chart's rectangle in the atlas, in texels */
  float uv_region[4];             /* as nrt_uv_raster_params */
  float texel_offset[2];
  uint32_t flip_x, flip_y;
} nrt_scene_chart;

/* Texel cast of an atlas of atlas_width x atlas_height texels over the scene, one chart per instance (charts: a HOST
 * array of one entry per instance).
 *   Charts   chart i's texel (x, y) casts exactly the ray nrt_uv_raster_device casts for an atlas of
 *            chart.width x chart.height with the chart's uv_region, texel_offset and flips, against chart.uv; its record
 *            goes to atlas texel (y0 + py) * atlas_width + x0 + px, px and py flipped as in that call.
 *   Records  inside a chart, nrt_uv_raster_device's records bit for bit, under NRT_TRAVERSE_FAST and
 *            NRT_TRAVERSE_CONFORMANCE: prim_id names a face of instance i's accel, and d_instance[texel] = i.
 *   Empty    a texel no chart covers, or that its chart's cast does not cover, gets {0, 0, 1e30, 0xFFFFFFFF},
 *            instance 0xFFFFFFFF and zero AOVs.  Every texel of the atlas is written.
 *   Position (d_position_3f, optional) (1 - u - v) w0 + u w1 + v w2 of the WORLD triangle, w_k = MultV(xform, v_k):
 *            each vertex moved first, then interpolated -- the position AOV of nrt_uv_raster_device over a world accel
 *            of the host-flattened triangles, bit for bit.
 *   Normal   (d_normal_3f, optional) needs `shading` (a HOST array of one entry per instance) with face-varying normals
 *            on every charted instance: each vertex normal moved to world space by the instance's inverse_transpose33
 *            (MultV order), then interpolated, not normalised.
 * d_records_16B (16-byte aligned), d_instance (uint32), d_position_3f and d_normal_3f (float3) hold one entry per atlas
 * texel.  *n_covered (optional) receives the number of covered texels.  Refused before any launch: a chart outside the
 * atlas or overlapping another, a chart whose uv accel is not a triangle accel or whose face count differs from its
 * instance's accel, a chart on a sphere or box instance, an atlas of more than 2^31 texels, a misaligned record buffer,
 * flags other than NRT_TRAVERSE_FAST / NRT_TRAVERSE_CONFORMANCE / NRT_TRAVERSE_CPP03_INVERSE.  The call owns its
 * scratch; each chart's cast is ordered on the device with the other passes of its uv accel, so calls on one scene or
 * on shared uv accels may run on several streams. */
int nrt_scene_uv_raster_device(const nrt_scene *s, const nrt_scene_chart *charts, uint32_t atlas_width,
                               uint32_t atlas_height, uint32_t flags, const nrt_scene_shading *shading,
                               void *d_records_16B, uint32_t *d_instance, float *d_position_3f, float *d_normal_3f,
                               uint64_t *n_covered, void *stream);

/* The texel point of a covered texel (record (u, v, prim), instance I), where both bakes start:
 *   P  the position AOV above;
 *   n  the unit cross(e1, e2) of the world triangle, flipped to the side of the interpolated world face-varying normal
 *      when shading[I] has normals, and otherwise flipped when I's 3x3 has a negative determinant -- mirroring reverses
 *      a triangle's winding in world space, so a mirrored instance bakes the same side as its unmirrored twin.
 * The scene walk takes an instance with the local range {0, FLT_MAX}, so min_t cannot keep a ray off its own surface:
 * rays spawned at a texel are lifted instead.
 *
 * AO bake over the scene: nrt_bake_ao_device's slots and draws (slot i is sample sample0 + i / n_covered of the
 * i % n_covered-th covered texel, direction ao_direction about n keyed by (texel, sample)) with the ray
 * origin P + ao_min_t n, range [0, ao_max_t); occluded iff the scene walk reports a hit with t < ao_max_t.
 * d_accum[texel] gains 1 per unoccluded ray.  p->d_facevarying_normals must be NULL: normals come per instance through
 * `shading` (HOST, one per instance, or NULL).  flags: NRT_TRAVERSE_FAST, NRT_TRAVERSE_CONFORMANCE (the scene walk's
 * reference-order kernel), NRT_TRAVERSE_CPP03_INVERSE; NRT_TRAVERSE_ANY_HIT is refused.  Records whose
 * (d_instance, prim_id) is not a triangle of the scene are refused after the compaction, before any walk.  The buffers
 * are the call's own, so calls may run on several streams.  res may be NULL. */
int nrt_scene_bake_ao_device(const nrt_scene *s, const void *d_records_16B, const uint32_t *d_instance,
                             const nrt_scene_shading *shading, const nrt_bake_params *p, float *d_accum,
                             nrt_bake_result *res, void *stream);
/* The same rays as 36-byte nanort::Ray records in slot order (capacity records; *n_rays = n_covered * spp); a call
 * whose rays do not fit writes nothing and returns NRT_ERR_INVALID. */
int nrt_scene_bake_ao_rays_device(const nrt_scene *s, const void *d_records_16B, const uint32_t *d_instance,
                                  const nrt_scene_shading *shading, const nrt_bake_params *p, void *d_rays_36B,
                                  uint64_t capacity, uint64_t *n_rays, void *stream);

/* Lightmap bake over the scene: nrt_bake_lightmap_device's slots, draws and estimate (d_accum_rgb[texel] / spp
 * estimates E / pi) with nrt_scene_render_path_device's inputs: one material table, material ids and LOCAL face-varying
 * normals per instance through `shading` (HOST, required, one per instance), p->d_material_ids and
 * p->d_facevarying_normals NULL, p->d_emissive_faces = {instance, face} pairs (read back once, range-checked).
 *   Bounce 0, the texel vertex, traces no ray: the texel point shaded as a white Lambertian seen along n, exactly as
 *   the flat bake (next-event estimation from dimensions 8/9, a cosine continuation from 10/11 with weight 1 that does
 *   not count emission, a light sample below n adds nothing); continuation and shadow rays are lifted as in
 *   nrt_scene_render_path_device.
 *   Bounces 1 and up are nrt_scene_render_path_device's shading and shadow stages with the texel slot map.
 * In waves of at most 8 Mi paths; each walk's ray count is read back on the host, and walks of empty queues are
 * skipped, so res->traverse_launches counts the walks actually run.  res->traverse_ms is 0: the scene walk is timed
 * as part of the call.  flags as the AO bake.  Refused before any walk: what nrt_scene_render_path_device refuses,
 * records whose (d_instance, prim_id) is not a triangle of the scene, a covered texel whose instance is 0xFFFFFFFF.
 * The buffers are the call's own, so calls may run on several streams.  res may be NULL. */
int nrt_scene_bake_lightmap_device(const nrt_scene *s, const void *d_records_16B, const uint32_t *d_instance,
                                   const nrt_lightmap_params *p, const nrt_scene_shading *shading, float *d_accum_rgb,
                                   nrt_lightmap_result *res, void *stream);
/* One bounce of it on caller-owned DEVICE queues, as nrt_bake_lightmap_bounce_device (path id = the call's slot). */
int nrt_scene_bake_lightmap_bounce_device(const nrt_scene *s, const void *d_records_16B, const uint32_t *d_instance,
                                          const nrt_lightmap_params *p, const nrt_scene_shading *shading,
                                          uint32_t bounce, uint64_t n_rays, const void *d_org_tmin,
                                          const void *d_dir_tmax, const uint32_t *d_path_id, void *d_weight,
                                          void *d_out_org_tmin, void *d_out_dir_tmax, uint32_t *d_out_path_id,
                                          void *d_sh_org_tmin, void *d_sh_dir_tmax, void *d_sh_contrib_pix,
                                          float *d_accum_rgb, uint64_t *n_continue, uint64_t *n_shadow,
                                          int skip_shadow_pass, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NANORT_B200_SCENE_BAKE_H_ */
