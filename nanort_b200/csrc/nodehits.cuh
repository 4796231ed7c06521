// Pieces of the reference's node-level traversal (BVHAccel::ListNodeIntersections, nanort.h:2558-2692, with the
// NodeBBoxIntersector of examples/nanosg/nanosg.h:562-640) shared by the two-level scene kernels (scene.cu) and the
// stand-alone box-primitive entry point (prims.cu: nrt_list_node_intersections).
#pragma once
#include "common.cuh"
#include "trav_common.cuh"

namespace nrt {

constexpr int kMaxNodeHits = 64;  // kMaxIntersections of nanosg::Scene::Traverse (nanosg.h:789)

struct WorldRay {
  float ox, oy, oz, dx, dy, dz, min_t, max_t;
};

__device__ __forceinline__ WorldRay load_world(const Ray36 *rays, size_t i) {
  const float *p = reinterpret_cast<const float *>(rays + i);
  WorldRay w;
  w.ox = __ldg(p + 0);
  w.oy = __ldg(p + 1);
  w.oz = __ldg(p + 2);
  w.dx = __ldg(p + 3);
  w.dy = __ldg(p + 4);
  w.dz = __ldg(p + 5);
  w.min_t = __ldg(p + 6);
  w.max_t = __ldg(p + 7);
  return w;
}

// NodeBBoxIntersector::Intersect: plain reciprocal direction, no range clamp, no widening; box = {bmin[3], bmax[3]}.
// Both distances (NodeHit::t_min / t_max).
__device__ __forceinline__ bool raw_box(const WorldRay &w, float rix, float riy, float riz, const float *box,
                                        float &tmin, float &tmax) {
  const bool sx = w.dx < 0.0f, sy = w.dy < 0.0f, sz = w.dz < 0.0f;
  const float lox = __ldg(box + 0), loy = __ldg(box + 1), loz = __ldg(box + 2);
  const float hix = __ldg(box + 3), hiy = __ldg(box + 4), hiz = __ldg(box + 5);
  const float tnx = ((sx ? hix : lox) - w.ox) * rix, tfx = ((sx ? lox : hix) - w.ox) * rix;
  const float tny = ((sy ? hiy : loy) - w.oy) * riy, tfy = ((sy ? loy : hiy) - w.oy) * riy;
  const float tnz = ((sz ? hiz : loz) - w.oz) * riz, tfz = ((sz ? loz : hiz) - w.oz) * riz;
  tmin = smax(tnz, smax(tny, tnx));
  tmax = smin(tfz, smin(tfy, tfx));
  return tmin <= tmax;
}

// ---- the reference's algorithm, one thread per ray ---------------------------------------------------------------
// std::priority_queue<NodeHit, vector, NodeHitComparator>: comp(a, b) = a.t_min < b.t_min, top = farthest.
// Sift rules of libstdc++'s __push_heap / __adjust_heap, so that entries with equal t_min leave in the same order.
struct NodeHitHeap {
  float t[kMaxNodeHits + 1];
  uint32_t id[kMaxNodeHits + 1];
  int n;
  __device__ __forceinline__ void sift_up(int hole, float vt, uint32_t vid) {
    int parent = (hole - 1) / 2;
    while (hole > 0 && t[parent] < vt) {
      t[hole] = t[parent];
      id[hole] = id[parent];
      hole = parent;
      parent = (hole - 1) / 2;
    }
    t[hole] = vt;
    id[hole] = vid;
  }
  __device__ __forceinline__ void push(float vt, uint32_t vid) {
    n++;
    sift_up(n - 1, vt, vid);
  }
  // the top moves to slot n - 1, the heap shrinks by one
  __device__ __forceinline__ void pop() {
    const int len = n - 1;
    const float vt = t[len];
    const uint32_t vid = id[len];
    t[len] = t[0];
    id[len] = id[0];
    int hole = 0, child = 0;
    while (child < (len - 1) / 2) {
      child = 2 * (child + 1);
      if (t[child] < t[child - 1]) child--;
      t[hole] = t[child];
      id[hole] = id[child];
      hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
      child = 2 * (child + 1);
      t[hole] = t[child - 1];
      id[hole] = id[child - 1];
      hole = child - 1;
    }
    n = len;
    sift_up(hole, vt, vid);
  }
};

// BVHAccel::ListNodeIntersections (nanort.h:2607-2692): the reference-order walk of a box tree over [min_t, max_t]
// (hit_t never drops), every box of a visited leaf tested with NodeBBoxIntersector and kept in the
// at-most-max_k-nearest heap, which is then sorted in place: slots 0 .. heap.n - 1 run nearest first.
// box_of(id) points at the {bmin[3], bmax[3]} of box primitive id.
template <class BoxOf>
__device__ __forceinline__ void collect_node_hits(const Node40 *nodes, const uint32_t *indices, BoxOf box_of,
                                                  const WorldRay &w, const RayCtx &c, int max_k, NodeHitHeap &heap) {
  const float rix = 1.0f / w.dx, riy = 1.0f / w.dy, riz = 1.0f / w.dz;  // NodeBBoxIntersector::PrepareTraversal
  heap.n = 0;
  reference_walk(nodes, c, w.min_t, w.max_t, [&](uint32_t first, uint32_t count, float &) {
    for (uint32_t k = 0; k < count; k++) {
      const uint32_t id = __ldg(indices + first + k);
      float tmin, tmax;
      if (!raw_box(w, rix, riy, riz, box_of(id), tmin, tmax)) continue;
      if (heap.n < max_k) {
        heap.push(tmin, id);
      } else if (tmin < heap.t[0]) {
        heap.pop();
        heap.push(tmin, id);
      }
    }
  });
  const int n_hits = heap.n;
  for (int k = 0; k < n_hits; k++) heap.pop();  // in-place heap sort
  heap.n = n_hits;
}


}  // namespace nrt
