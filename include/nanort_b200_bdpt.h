/*
 * nanort_b200_bdpt.h -- the reference's bidirectional path tracer (examples/bidir_path_tracer/main.cc) as a
 * device-resident wavefront pass, a C-ABI extension of nanort_b200.h.
 *
 * Kept in its own header: nanort.h, nanosg.h and nanort_b200.h are the drop-in facade that the reference's own
 * example programs are compiled against, and this pass needs nothing from them beyond nanort_b200.h's types.
 *
 * One sample is the body of the reference's sample loop (main.cc:1383-1392): a xorshift128 generator `Random` seeded
 * with the sample's seed, an eye subpath (eyeSubpath + raytrace), a light subpath (LightSampler::sample,
 * directionCosTheta, raytrace) and connectPath's sum over the emission term and the MIS-weighted connections
 * (weightMIS, calcG).  All of it is restated in float32 with the reference's operation order, including the
 * subexpressions the reference evaluates in double ((1.0 - u - v), 1.0 / ior, (1.0 - fresnel), (1.0 - dissolve),
 * directionCosTheta's 2.0 * kPi * u2, sqrt(u1) and 1.0 - u1, float3::normalize's threshold and 1.0 / len).
 * directionCosTheta's two random arguments are drawn as GCC on x86-64 evaluates a call's arguments, right to left:
 * u2 first, then u1.  Its cosf / sinf are evaluated as cos / sin in double rounded to float.
 *
 * The light-origin vertex: lightSubpath leaves its material uninitialised (`Vertex vertex;`), and weightMIS reads
 * its isDelta() (main.cc:1203-1204), so the reference's result there depends on stack contents.  Here that vertex
 * (like the lens vertex) has no material (material = 0xFFFFFFFF) and is not delta -- what the reference computes
 * when its automatic variables start zeroed (GCC's -ftrivial-auto-var-init=zero).
 */
#ifndef NANORT_B200_BDPT_H_
#define NANORT_B200_BDPT_H_

#include "nanort_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nrt_bdpt_params {
  float cam[12];          /* org, right, up, forward: dir = normalize(sx*right + sy*up + forward),
                             sx = px/W - 0.5, sy = py/H - 0.5, px = x + (u0 - 0.5), py = y + (u1 - 0.5)
                             (main.cc:1022-1027; {0,5,20, 1,0,0, 0,1,0, 0,0,-1} is the reference camera, bit for bit) */
  uint32_t width, height;
  uint32_t spp, sample0, spp_total; /* samples sample0 .. sample0+spp-1 of spp_total; seed of sample i of loop pixel
                                       (x, y) = (uint32)((y*W + x)*spp_total + i)  (main.cc:1382) */
  uint32_t tile_w, tile_h, shard, n_shards;   /* the path pass's tile map and rules (tile_w % 8 == 0, tile_h % 4 == 0) */
  uint32_t max_bounces;   /* uMaxBounces (10): raytrace's loop bound AND connectPath's e + l - 2 bound; at most 64 */
  uint32_t n_materials;
  const void *d_materials;            /* 16 floats per material, as nrt_path_params: diffuse[3] specular[3]
                                         transmittance[3] emission[3] ior dissolve pad pad */
  const void *d_material_ids;         /* uint32 per face, required */
  const void *d_facevarying_normals;  /* float[9 * n_faces], required (LightSampler::sample reads them) */
  uint32_t flags;         /* 0 or NRT_TRAVERSE_CONFORMANCE; anything else is refused */
  uint32_t pad;
} nrt_bdpt_params;

typedef struct nrt_bdpt_result {
  uint64_t eye_rays;        /* closest-hit rays of the eye subpaths (camera rays included) */
  uint64_t light_rays;      /* closest-hit rays of the light subpaths */
  uint64_t connection_rays; /* calcG's rays */
  float traverse_ms;        /* device time inside the traversal launches (CUDA events) */
  float total_ms;           /* device time of the whole call */
  uint32_t launches, traverse_launches;
} nrt_bdpt_result;

/* The reference's VertexType */
#define NRT_BDPT_LIGHT 0u
#define NRT_BDPT_LENS 1u
#define NRT_BDPT_SURFACE 2u

/* One subpath vertex: the reference's Vertex with its material as an index (0xFFFFFFFF for the lens vertex and the
 * light-origin vertex) and the face it lies on (0xFFFFFFFF for the same two).  Fields a vertex never receives in the
 * reference are 0. */
typedef struct nrt_bdpt_vertex {
  float position[3];
  float original_norm[3];
  float norm[3];
  float beta[3];
  float wo[3];
  float pdf_fwd, pdf_rev;
  uint32_t type; /* NRT_BDPT_LIGHT / LENS / SURFACE */
  uint32_t material;
  uint32_t prim_id;
} nrt_bdpt_vertex; /* 80 bytes */

/* Renders samples sample0 .. sample0 + spp - 1 of every pixel of this shard's tiles and adds each sample's
 * connectPath colour to d_accum_rgb (DEVICE float[3 * width * height]) at pix = r * W + x, where the reference's loop
 * row is y = H - 1 - r: the frame is the reference's rgb array (its row flip included) before / SPP, the clamp and
 * the gamma.  A sample whose eye subpath has no vertex beyond the lens adds nothing.  Each pixel's samples are added
 * in ascending sample order, so a frame split by sample0, by shards or by tiles equals one call bit for bit.  Under
 * NRT_TRAVERSE_CONFORMANCE (the reference-order walk; with a reference-exact tree every hit is the reference's) a
 * frame is also the same from call to call; the production walk may return another of the faces a ray meets at the
 * same distance (a shared edge), as nrt_traverse does, and a sample through such a point can differ between calls.
 * Refused with NRT_ERR_INVALID before any traversal launch: NULL pointers, missing material ids or normals,
 * n_materials == 0, max_bounces outside [1, 64], flags other than NRT_TRAVERSE_CONFORMANCE, sample0 + spp > spp_total,
 * the path pass's tile rules, a material id >= n_materials and a mesh without an emissive face (max(Le) > 0.001; the
 * reference indexes cdf_[0] of an empty vector).  The last two are read back (a stream synchronisation) at pass start.
 * Passes on one accel run one after the other on the device, whatever their streams.  res may be NULL. */
int nrt_render_bdpt_device(const nrt_accel *accel, const nrt_bdpt_params *p, float *d_accum_rgb, nrt_bdpt_result *res,
                           void *stream);

/* The same pass for the call's slots (this shard's tiles, sample-major over 8x4 blocks inside each tile, as
 * nrt_render_path_device numbers them; slots outside the image have empty subpaths and colour 0), writing per slot
 * instead of a frame: both subpaths (d_eye, d_light: DEVICE nrt_bdpt_vertex[n_slots * (max_bounces + 1)]), their
 * lengths (d_n_eye, d_n_light: DEVICE uint32[n_slots]) and the sample's colour (d_sample_rgb: DEVICE
 * float[3 * n_slots]).  n_slots = (this shard's tiles) * tile_w * tile_h * spp.  Records past a subpath's length are
 * not written.  Same refusals as nrt_render_bdpt_device. */
int nrt_bdpt_export_device(const nrt_accel *accel, const nrt_bdpt_params *p, nrt_bdpt_vertex *d_eye,
                           nrt_bdpt_vertex *d_light, uint32_t *d_n_eye, uint32_t *d_n_light, float *d_sample_rgb,
                           nrt_bdpt_result *res, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NANORT_B200_BDPT_H_ */
