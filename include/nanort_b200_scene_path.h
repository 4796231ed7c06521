/*
 * nanort_b200_scene_path.h -- the path tracer over two-level scenes, a C-ABI extension of nanort_b200.h.
 *
 * Kept in its own header: nanort.h, nanosg.h and nanort_b200.h are the drop-in facade that the reference's own
 * example programs are compiled against, and this pass needs nothing from them beyond nanort_b200.h's types.
 */
#ifndef NANORT_B200_SCENE_PATH_H_
#define NANORT_B200_SCENE_PATH_H_

#include "nanort_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Path tracing over the scene: nrt_render_path_device's pass (same nrt_path_params, tile / shard slot order, camera
 * rays, random draws and shading of main.cc:826-991) with Scene::Traverse as its traversal step, as stand-alone stage
 * kernels: per wave a camera kernel, then per bounce the scene walk, the shade kernel, the scene walk over the shadow
 * rays and the accumulate kernel.  One material table (p->d_materials) for the whole scene; material ids and
 * face-varying normals come per instance in `shading` (a HOST array of one entry per instance), so two instances of
 * one accel may look different; p->d_material_ids and p->d_facevarying_normals must be NULL.
 * p->d_emissive_faces holds n_emissive pairs {instance, face} (uint32[2 * n_emissive], MeshLight's list over the
 * scene); the call reads it back once and refuses a pair out of range.
 * At a hit: P = org + t dir with the world ray and world distance (main.cc:860); the geometric normal is
 * -cross(e1, e2) of the hit triangle moved to world space by the instance's matrix (calcNormal's orientation, also for
 * a mirroring matrix); face-varying normals are moved to world space by the instance's inverse_transpose33 (as
 * nanosg.h:866-867 moves Ns), then interpolated and normalised (main.cc:862-875).  Light samples read one world-space
 * record per emissive pair (its three vertices and emission, written at pass start), so a scaled light has its world
 * area.
 * Spawned rays follow the AO pass's rule, because an instance is walked with the local range {0, FLT_MAX}: a
 * continuation ray starts at P lifted by ray_min_t along the unit geometric normal on the side its direction leaves
 * (the viewer's side for reflection and diffuse, the far side for refraction); a shadow ray starts lifted the same way
 * on the light's side, with direction, distance and contribution computed from the unlifted P; it is occluded iff it
 * hits at a reported world distance below its max_t: where the lifted ray meets the sampled light triangle's plane,
 * less 1e-5 (with dist - 1e-5 the light would occlude its own sample).
 * A continuation ray with a zero direction (total internal reflection) is counted and misses.
 * flags: NRT_TRAVERSE_FAST / NRT_TRAVERSE_CONFORMANCE (the scene walk's reference-order kernel) /
 * NRT_TRAVERSE_CPP03_INVERSE; NRT_TRAVERSE_ANY_HIT and NRT_AO_PACKED_TILES are refused.  Synchronous per bounce (the
 * ray counts are read on the host); buffers are the call's own, so calls on one scene may run on several streams. */
typedef struct nrt_scene_shading {
  const void *d_material_ids;        /* uint32 per face of the instance's accel, or NULL = material 0 */
  const void *d_facevarying_normals; /* float[9 * n_faces] in the instance's LOCAL space, or NULL */
} nrt_scene_shading;

int nrt_scene_render_path_device(const nrt_scene *s, const nrt_path_params *p, const nrt_scene_shading *shading,
                                 float *d_accum_rgb, nrt_path_result *res, void *stream);
/* One bounce of that pass on caller-owned DEVICE queues, with nrt_path_bounce_device's queues and counts. */
int nrt_scene_path_bounce_device(const nrt_scene *s, const nrt_path_params *p, const nrt_scene_shading *shading,
                                 uint32_t bounce, uint64_t n_rays, const void *d_org_tmin, const void *d_dir_tmax,
                                 const uint32_t *d_path_id, void *d_weight, void *d_out_org_tmin, void *d_out_dir_tmax,
                                 uint32_t *d_out_path_id, void *d_sh_org_tmin, void *d_sh_dir_tmax,
                                 void *d_sh_contrib_pix, float *d_accum_rgb, uint64_t *n_continue, uint64_t *n_shadow,
                                 int skip_shadow_pass, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NANORT_B200_SCENE_PATH_H_ */
