// Derives the private traversal layout (64-byte child-pair nodes + 48-byte packed
// triangles in leaf order) from the API-visible nanort arrays that Build or
// nrt_adopt left on the device:
//   nodes   BVHNode<float>[n_nodes]   nanort.h:498-550
//   indices uint32[n_prims]           (BVHAccel::indices_, nanort.h:855)
//   faces / verts as TriangleMesh holds them (nanort.h:925-930)
// The packed triangles remove the reference's two levels of indirection at
// intersection time (indices_ -> faces -> vertices, nanort.h:2394 + 1065-1071).
#include <string.h>

#include <algorithm>

#include "common.cuh"
#include "scan.cuh"

namespace nrt {

__global__ void pack_tris_kernel(const uint32_t *__restrict__ indices, const uint32_t *__restrict__ faces,
                                 const float *__restrict__ verts, uint32_t n, PackedTri *__restrict__ out) {
  uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= n) return;
  uint32_t prim = indices[slot];
  uint32_t f0 = faces[3 * (size_t)prim + 0], f1 = faces[3 * (size_t)prim + 1], f2 = faces[3 * (size_t)prim + 2];
  const float *p0 = verts + 3 * (size_t)f0, *p1 = verts + 3 * (size_t)f1, *p2 = verts + 3 * (size_t)f2;
  PackedTri t;
  t.a = make_float4(p0[0], p0[1], p0[2], __uint_as_float(prim));
  t.b = make_float4(p1[0], p1[1], p1[2], __uint_as_float(0u));
  t.c = make_float4(p2[0], p2[1], p2[2], 0.0f);
  out[slot] = t;
}

// Box primitives (top-level tree of a two-level scene): the same 48-byte slot carries the instance's world box,
//   bmin.xyz, instance id | bmax.xyz, last_in_leaf flag | unused
__global__ void pack_boxes_kernel(const uint32_t *__restrict__ indices, const float *__restrict__ boxes6, uint32_t n,
                                  PackedTri *__restrict__ out) {
  uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= n) return;
  const uint32_t prim = indices[slot];
  const float *b = boxes6 + 6 * (size_t)prim;
  PackedTri t;
  t.a = make_float4(b[0], b[1], b[2], __uint_as_float(prim));
  t.b = make_float4(b[3], b[4], b[5], __uint_as_float(0u));
  t.c = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  out[slot] = t;
}

__device__ __forceinline__ void invert_box(Node40 &c) {
  for (int k = 0; k < 3; k++) {
    c.bmin[k] = 3.402823466e38f;
    c.bmax[k] = -3.402823466e38f;
  }
}

__global__ void wide_nodes_kernel(const Node40 *__restrict__ nodes, uint32_t n, const uint32_t *__restrict__ widx,
                                  WideNode *__restrict__ wide, PackedTri *__restrict__ tris) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Node40 nd = nodes[i];
  if (nd.flag != 0) {
    // leaf: mark its last triangle so that the traversal needs no count
    if (nd.data[0] > 0) {
      float *w = reinterpret_cast<float *>(&tris[(size_t)nd.data[1] + nd.data[0] - 1].b) + 3;
      *w = __uint_as_float(1u);
    }
    if (i == 0) {
      // the whole tree is one leaf: a pair whose second child is empty
      WideNode w;
      w.q0 = make_float4(nd.bmin[0], nd.bmin[1], nd.bmin[2], nd.bmax[0]);
      // the empty second child carries an inverted box: it can never pass the slab test
      w.q1 = make_float4(nd.bmax[1], nd.bmax[2], 3.402823466e38f, 3.402823466e38f);
      w.q2 = make_float4(3.402823466e38f, -3.402823466e38f, -3.402823466e38f, -3.402823466e38f);
      w.q3 = make_int4(nd.data[0] ? ~(int)nd.data[1] : kEmptyLeaf, kEmptyLeaf, 0, 0);
      wide[0] = w;
    }
    return;
  }
  Node40 c0 = nodes[nd.data[0]], c1 = nodes[nd.data[1]];
  // a child leaf without primitives (reference trees built with min_leaf_primitives == 0 contain them) carries an
  // inverted box: it can never pass the slab test, so no kernel ever has to follow an empty reference
  if (c0.flag != 0 && c0.data[0] == 0) invert_box(c0);
  if (c1.flag != 0 && c1.data[0] == 0) invert_box(c1);
  WideNode w;
  w.q0 = make_float4(c0.bmin[0], c0.bmin[1], c0.bmin[2], c0.bmax[0]);
  w.q1 = make_float4(c0.bmax[1], c0.bmax[2], c1.bmin[0], c1.bmin[1]);
  w.q2 = make_float4(c1.bmin[2], c1.bmax[0], c1.bmax[1], c1.bmax[2]);
  w.q3 = make_int4(child_ref(c0, nd.data[0], widx), child_ref(c1, nd.data[1], widx), nd.axis, 0);
  wide[widx[i]] = w;
}

// ---- round-2 layout: PairNode (sign-addressed planes) and TriCM (component-major triangles), derived from the
// final WideNode / PackedTri arrays so that indices, refs and slots are shared by every kernel
__global__ void pair_from_wide_kernel(const WideNode *__restrict__ wide, uint32_t n, PairNode *__restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const WideNode w = wide[i];
  // WideNode: q0 = c0.lo.xyz, c0.hi.x | q1 = c0.hi.yz, c1.lo.xy | q2 = c1.lo.z, c1.hi.xyz
  const float lo0x = w.q0.x, lo0y = w.q0.y, lo0z = w.q0.z, hi0x = w.q0.w, hi0y = w.q1.x, hi0z = w.q1.y;
  const float lo1x = w.q1.z, lo1y = w.q1.w, lo1z = w.q2.x, hi1x = w.q2.y, hi1y = w.q2.z, hi1z = w.q2.w;
  PairNode p;
  p.x[0] = make_float4(lo0x, lo1x, hi0x, hi1x);
  p.x[1] = make_float4(hi0x, hi1x, lo0x, lo1x);
  p.y[0] = make_float4(lo0y, lo1y, hi0y, hi1y);
  p.y[1] = make_float4(hi0y, hi1y, lo0y, lo1y);
  p.z[0] = make_float4(lo0z, lo1z, hi0z, hi1z);
  p.z[1] = make_float4(hi0z, hi1z, lo0z, lo1z);
  p.r = w.q3;
  p.pad = make_int4(0, 0, 0, 0);
  out[i] = p;
}

__global__ void tris_cm_kernel(const PackedTri *__restrict__ in, uint32_t n, TriCM *__restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const PackedTri t = in[i];
  const uint32_t w = (__float_as_uint(t.a.w) & 0x7FFFFFFFu) | (__float_as_uint(t.b.w) != 0u ? 0x80000000u : 0u);
  const float wf = __uint_as_float(w);
  TriCM o;
  o.X = make_float4(t.a.x, t.b.x, t.c.x, wf);
  o.Y = make_float4(t.a.y, t.b.y, t.c.y, wf);
  o.Z = make_float4(t.a.z, t.b.z, t.c.z, wf);
  out[i] = o;
}

// Camera-relative copies: every plane and vertex coordinate minus the camera origin's component on its axis (refs,
// pad and the w words unchanged).  One IEEE subtraction gives the same bits here as in the traversal kernel, which
// subtracts the origin per ray otherwise (no contraction under --fmad=false), so every decision stays the same.
__global__ void camera_relative_kernel(const PairNode *__restrict__ pair, uint32_t n_pair, const TriCM *__restrict__ tris,
                                       uint32_t n_tris, float cx, float cy, float cz, PairNode *__restrict__ pair_rel,
                                       TriCM *__restrict__ tris_rel) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_pair) {
    PairNode p = pair[i];
    for (int k = 0; k < 2; k++) {
      p.x[k] = make_float4(p.x[k].x - cx, p.x[k].y - cx, p.x[k].z - cx, p.x[k].w - cx);
      p.y[k] = make_float4(p.y[k].x - cy, p.y[k].y - cy, p.y[k].z - cy, p.y[k].w - cy);
      p.z[k] = make_float4(p.z[k].x - cz, p.z[k].y - cz, p.z[k].z - cz, p.z[k].w - cz);
    }
    pair_rel[i] = p;
  }
  if (i < n_tris) {
    TriCM t = tris[i];
    t.X = make_float4(t.X.x - cx, t.X.y - cx, t.X.z - cx, t.X.w);
    t.Y = make_float4(t.Y.x - cy, t.Y.y - cy, t.Y.z - cy, t.Y.w);
    t.Z = make_float4(t.Z.x - cz, t.Z.y - cz, t.Z.z - cz, t.Z.w);
    tris_rel[i] = t;
  }
}

int camera_relative_layout(Accel *a, const float cam[3], cudaStream_t s) {
  uint32_t key[3];
  memcpy(key, cam, sizeof(key));  // bit patterns: -0.0 and +0.0 give different copies, NaN is a key like any other
  if (a->rel_valid && key[0] == a->rel_origin[0] && key[1] == a->rel_origin[1] && key[2] == a->rel_origin[2])
    return NRT_OK;
  a->rel_valid = false;
  if (!a->d_pair_rel) NRT_CUDA(cudaMalloc(&a->d_pair_rel, sizeof(PairNode) * a->n_wide));
  if (!a->d_tris_rel) NRT_CUDA(cudaMalloc(&a->d_tris_rel, sizeof(TriCM) * (size_t)a->n_prims));
  const uint32_t n = (uint32_t)std::max<size_t>(a->n_wide, a->n_prims);
  camera_relative_kernel<<<(n + 255) / 256, 256, 0, s>>>(a->d_pair, (uint32_t)a->n_wide, a->d_tris_cm, a->n_prims, cam[0],
                                                         cam[1], cam[2], a->d_pair_rel, a->d_tris_rel);
  NRT_CUDA(cudaGetLastError());
  memcpy(a->rel_origin, key, sizeof(key));
  a->rel_valid = true;
  return NRT_OK;
}

int derive_private_layout(Accel *a, cudaStream_t s) {
  const uint32_t n_nodes = (uint32_t)a->n_nodes;
  const uint32_t n_prims = a->n_prims;
  cudaFree(a->d_tris);
  cudaFree(a->d_wide);
  cudaFree(a->d_pair);
  cudaFree(a->d_tris_cm);
  cudaFree(a->d_pair_rel);
  cudaFree(a->d_tris_rel);
  cudaFree(a->d_face_n);
  a->d_tris = nullptr;
  a->d_wide = nullptr;
  a->d_pair = nullptr;
  a->d_tris_cm = nullptr;
  a->d_pair_rel = nullptr;
  a->d_tris_rel = nullptr;
  a->rel_valid = false;
  a->d_face_n = nullptr;
  NRT_CUDA(cudaMalloc(&a->d_tris, sizeof(PackedTri) * (size_t)n_prims));
  if (a->d_prim_boxes)
    pack_boxes_kernel<<<(n_prims + 255) / 256, 256, 0, s>>>(a->d_indices, a->d_prim_boxes, n_prims, a->d_tris);
  else
    pack_tris_kernel<<<(n_prims + 255) / 256, 256, 0, s>>>(a->d_indices, a->d_faces, a->d_verts, n_prims, a->d_tris);
  NRT_CUDA(cudaGetLastError());

  uint32_t *d_flags = nullptr, *d_widx = nullptr;
  uint32_t n_branch = 0;
  int rc = NRT_OK;
  cudaError_t e = cudaMalloc(&d_flags, sizeof(uint32_t) * (size_t)n_nodes);
  if (e == cudaSuccess) e = cudaMalloc(&d_widx, sizeof(uint32_t) * (size_t)n_nodes);
  if (e == cudaSuccess) {
    branch_flags_kernel<<<(n_nodes + 255) / 256, 256, 0, s>>>(a->d_nodes, n_nodes, d_flags);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) rc = exclusive_scan_u32(d_flags, d_widx, n_nodes, &n_branch, s);
  if (e == cudaSuccess && rc == NRT_OK) {
    a->n_wide = n_branch > 0 ? n_branch : 1;
    a->root_is_leaf = (n_branch == 0);
    e = cudaMalloc(&a->d_wide, sizeof(WideNode) * a->n_wide);
  }
  if (e == cudaSuccess && rc == NRT_OK) {
    wide_nodes_kernel<<<(n_nodes + 255) / 256, 256, 0, s>>>(a->d_nodes, n_nodes, d_widx, a->d_wide, a->d_tris);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  cudaFree(d_flags);  // every path, error or not
  cudaFree(d_widx);
  if (e != cudaSuccess) return cuda_fail(e, "derive_private_layout", __FILE__, __LINE__);
  if (rc != NRT_OK || a->d_prim_boxes) return rc;  // box accels (top level of a scene) are walked by scene.cu only
  NRT_CUDA(cudaMalloc(&a->d_pair, sizeof(PairNode) * a->n_wide));
  NRT_CUDA(cudaMalloc(&a->d_tris_cm, sizeof(TriCM) * (size_t)n_prims));
  pair_from_wide_kernel<<<((uint32_t)a->n_wide + 255) / 256, 256, 0, s>>>(a->d_wide, (uint32_t)a->n_wide, a->d_pair);
  tris_cm_kernel<<<(n_prims + 255) / 256, 256, 0, s>>>(a->d_tris, n_prims, a->d_tris_cm);
  NRT_CUDA(cudaGetLastError());
  NRT_CUDA(cudaStreamSynchronize(s));
  return NRT_OK;
}

}  // namespace nrt
