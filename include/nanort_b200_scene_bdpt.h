/*
 * nanort_b200_scene_bdpt.h -- the bidirectional path tracer (nanort_b200_bdpt.h) over two-level scenes, a C-ABI
 * extension of nanort_b200.h.
 *
 * Kept in its own header: nanort.h, nanosg.h and nanort_b200.h are the drop-in facade that the reference's own
 * example programs are compiled against, and this pass needs nothing from them beyond the types of the two headers
 * it includes.
 *
 * The pass is nrt_render_bdpt_device's: the same nrt_bdpt_params (camera, tile map, seeds, max_bounces), random
 * draws, subpaths, weightMIS and connections, the same frame layout (each pixel's samples added in ascending sample
 * order, no atomics) and the same export slot layout, with Scene::Traverse as its traversal step.  It runs as stage
 * kernels: per wave the eye bounces, the light bounces and one scene walk over all connection rays; each walk packs
 * its rays, walks the scene (the production kernel, or the reference-order kernel under NRT_TRAVERSE_CONFORMANCE)
 * and runs a stage kernel on the hit records.  The walk takes its ray count from the host, so every walk is preceded
 * by one read-back.
 *
 * What differs from the flat pass:
 *  - Per-instance shading.  One material table (p->d_materials) for the scene; p->d_material_ids and
 *    p->d_facevarying_normals must be NULL.  `shading` is a HOST array of one nrt_scene_shading per instance, and
 *    every instance must give both its material ids and its LOCAL face-varying normals (LightSampler::sample reads
 *    the normals).
 *  - The light table is LightSampler's over the {instance, face} pairs in flattened order (pair index = the sum of
 *    the face counts of the instances before it + face): LightSampler over the host-flattened mesh.  The world
 *    vertices are Matrix::MultV of the local ones (float32, nanosg's order), the area is 0.5f * |cross(v2 - v0, v1 -
 *    v0)| of the world triangle (so a scaled light has its world area), totalArea is the sequential sum in pair order
 *    and the CDF follows the (area, pair) order.
 *  - Light sample: the point on the world triangle; the face-varying normals moved to world space by the instance's
 *    inverse_transpose33, interpolated, given to directionCosTheta un-normalised and stored normalised.
 *  - Hits: P = org + t dir with the world ray (its actual, lifted origin) and the world distance.  The light's first
 *    ray is the one ray whose direction is not unit length (directionCosTheta of the un-normalised light normal), so
 *    there t is the world distance over |dir|, the ray parameter.  The shading normal is the instance's face-varying
 *    normals moved to world space, then interpolated as the flat pass does; the material comes from the instance's
 *    ids.
 *  - Spawn: the scene walks an instance with the local range {0, FLT_MAX}, so min_t cannot keep a ray off the
 *    surface it starts on.  A subpath's continuation and the light subpath's first ray start kEps (0.001) above their
 *    vertex along the unit world geometric normal, on the side the direction leaves.  Camera rays are not lifted.
 *    pdfFwd / pdfRev convert with the distances between stored (unlifted) vertex positions.
 *  - Connections (calcG): direction and dist come from the two unlifted vertices; the ray starts kEps above the eye
 *    vertex along its geometric normal, on the side of the light vertex; it is visible iff the walk reports no hit
 *    nearer than where it meets the light vertex's triangle plane (for the light-origin vertex, the sampled pair's),
 *    less 1e-5 (nanort_b200_scene_path.h's shadow rule).  G's cosines and 1 / dist^2 are calcG's, from the unlifted
 *    geometry.  The reference's |dist - t| > kEps test is not kept: a lifted ray can pass its target vertex without
 *    hitting it (at a silhouette, or near the light's edge), so the hit distance says nothing about the target.
 *  - flags: 0 or NRT_TRAVERSE_CONFORMANCE; anything else is refused.
 *  - Refused with NRT_ERR_INVALID before any traversal launch: everything nrt_render_bdpt_device refuses, a NULL
 *    shading array, an instance without material ids or normals, an instance that is not a triangle accel, a material
 *    id >= n_materials in any instance, a scene with no emissive pair and more than 2^32 - 1 pairs.  The last three
 *    are read back (a stream synchronisation) at pass start.
 *  - Buffers are the call's own, so calls on one scene may run on several streams.
 * Under NRT_TRAVERSE_CONFORMANCE with reference-built trees every hit is nanosg's, and a frame is the same from call
 * to call; the production walk may pick another surface at exactly the same distance (a shared edge).
 * res->traverse_ms is the device time inside the scene walks; res->traverse_launches counts the walks run (a walk
 * with no ray left is skipped).
 */
#ifndef NANORT_B200_SCENE_BDPT_H_
#define NANORT_B200_SCENE_BDPT_H_

#include "nanort_b200_bdpt.h"
#include "nanort_b200_scene_path.h"

#ifdef __cplusplus
extern "C" {
#endif

/* nrt_render_bdpt_device over a scene: adds each sample's connectPath colour to d_accum_rgb (DEVICE
 * float[3 * width * height]). */
int nrt_scene_render_bdpt_device(const nrt_scene *s, const nrt_bdpt_params *p, const nrt_scene_shading *shading,
                                 float *d_accum_rgb, nrt_bdpt_result *res, void *stream);

/* nrt_bdpt_export_device over a scene: the same slots and records (nrt_bdpt_vertex keeps its flat meaning; prim_id
 * is the face in its instance's accel), and per vertex record the instance of its face (d_eye_inst, d_light_inst:
 * DEVICE uint32[n_slots * (max_bounces + 1)], 0xFFFFFFFF wherever prim_id is 0xFFFFFFFF), and per slot the sampled
 * light {instance, face} (d_light_pair: DEVICE uint32[2 * n_slots], {0xFFFFFFFF, 0xFFFFFFFF} for a slot without a
 * light subpath).  Records past a subpath's length are not written. */
int nrt_scene_bdpt_export_device(const nrt_scene *s, const nrt_bdpt_params *p, const nrt_scene_shading *shading,
                                 nrt_bdpt_vertex *d_eye, nrt_bdpt_vertex *d_light, uint32_t *d_eye_inst,
                                 uint32_t *d_light_inst, uint32_t *d_light_pair, uint32_t *d_n_eye,
                                 uint32_t *d_n_light, float *d_sample_rgb, nrt_bdpt_result *res, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NANORT_B200_SCENE_BDPT_H_ */
