"""Host model of the production BVH builder (csrc/build.cu, `NRT_BUILD_FAST`), restated in numpy from the code of
build.cu, build_common.cuh and radix_sort.cuh.  Given the same float32 input it returns the `Node40` array and
`indices_` that `GetNodes()` / `GetIndices()` return, bit for bit.

The library is compiled with --fmad=false and without fast-math, so every float operation of the builder is one
IEEE-rounded float32 operation, and numpy float32 reproduces it when it runs the same operations in the same order.
Three things need care:
  * float -> int conversions are CUDA's (cvt.rzi.s32.f32: truncate, NaN -> 0, saturate at the int range), which numpy's
    `astype(np.int32)` is not (`cuda_f2i`);
  * box minima / maxima are taken on ordered-uint keys (build_common.cuh:48-54, `fkey`), so -0.0 < +0.0;
  * the phases of the device (level-synchronous passes, one CTA per node, one warp per subtree, the segmented
    32-lane `small_block`) all apply one split rule; the model applies it level by level to every node at once.

The split rule of a node with box [bmin, bmax] over its primitives in the current order (build_common.cuh:79-258,
build.cu:290-362, 513-702, 723-977, 1018-1207):
  * per axis, inv = B / (bmax - bmin) if that extent is > 0, else 0 (`inv_extent`); a centroid c goes to bin
    clamp(int((c - bmin) * inv), 0, B - 1) (`bin_of`);
  * candidate boundary i in 1..B-1 splits bins [0, i) | [i, B); its cost is (float)N_L * area(L) + (float)N_R *
    area(R) with area = 2 * ((dx*dy + dy*dz) + dz*dx) of the exact union of the member boxes (`sweep_axis`,
    `box_area`); a side without primitives never wins, and a cost counts only if it is < FLT_MAX (the sweep starts
    from FLT_MAX and takes strictly smaller costs); the first minimum along an axis wins;
  * the axis: 0, then 1 if cost[0] > cost[1], then 2 if cost[ax] > cost[2] -- a tie keeps the lower axis;
  * a primitive goes left iff its bin on that axis is below the boundary; when no axis has a cost < FLT_MAX the node
    is cut at n >> 1 of its current order and labelled (ax + 2) % 3 (build.cu:311-321);
  * both partitions are stable; children are leaves iff n <= max(min_leaf_primitives, 1) or depth >= max_tree_depth
    (`child_class`, build.cu:284-287, 1282); child boxes are the exact unions of their members.
Primitive records (build.cu:50-139, prims.cu:30-44), the Morton pre-order of more than kSubtree = 128 primitives
(radix_sort.cuh:16-35, build.cu:1349-1388) and the closed-form DFS pre-order of phase C (build.cu:1209-1259) are
restated in the functions below.
"""
import numpy as np

F32 = np.float32
FLT_MAX = F32(np.finfo(np.float32).max)
K_SMALL = 32        # small_block: nodes of at most one warp of primitives (build.cu:1020)
K_SUBTREE = 128     # kSubtree: one warp per subtree; also the Morton threshold (build.cu:41, 1368)
K_MID = 2048        # kMid: one CTA per node above kSubtree (build.cu:42)
PHASES = ("level", "mid", "subtree", "small")


# ----------------------------------------------------------------------------- scalar helpers
def fkey(f):
    """build_common.cuh:48-51: order-preserving float32 -> uint32 key (-0.0 < +0.0)."""
    u = np.ascontiguousarray(f, F32).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def funkey(k):
    """build_common.cuh:52-54: the inverse of `fkey`."""
    k = np.asarray(k, np.uint32)
    return np.where(k & np.uint32(0x80000000), k ^ np.uint32(0x80000000), ~k).astype(np.uint32).view(F32)


def cuda_f2i(x):
    """(int)x of a float on the device (cvt.rzi.s32.f32): truncation toward zero, NaN -> 0, +-inf and values out of
    range saturate to INT_MAX / INT_MIN.  Returned as int64."""
    x = np.asarray(x, F32).astype(np.float64)
    with np.errstate(invalid="ignore"):
        t = np.trunc(x)
    t = np.where(np.isnan(t), 0.0, t)
    return np.clip(t, -2.0 ** 31, 2.0 ** 31 - 1).astype(np.int64)


def inv_extent(lo, hi, B):
    """build_common.cuh:93-97: B / (hi - lo) when the extent is > 0, else 0 (float32; a denormal extent gives inf)."""
    sz = np.asarray(hi, F32) - np.asarray(lo, F32)
    with np.errstate(divide="ignore", over="ignore"):
        return np.where(sz > 0, F32(B) / np.where(sz > 0, sz, F32(1)), F32(0)).astype(F32)


def bin_of(c, nmin, inv, B):
    """build_common.cuh:85-91: clamp(int((c - nmin) * inv), 0, B - 1) in float32 with CUDA's conversion."""
    with np.errstate(over="ignore", invalid="ignore"):
        q = (np.asarray(c, F32) - np.asarray(nmin, F32)) * np.asarray(inv, F32)
    return np.clip(cuda_f2i(q), 0, B - 1)


def box_area(lo, hi):
    """build_common.cuh:79-83: 2 * ((dx*dy + dy*dz) + dz*dx), float32; lo, hi: [..., 3]."""
    with np.errstate(over="ignore", invalid="ignore"):
        d = np.asarray(hi, F32) - np.asarray(lo, F32)
        dx, dy, dz = d[..., 0], d[..., 1], d[..., 2]
        return F32(2) * ((dx * dy + dy * dz) + dz * dx)


# ----------------------------------------------------------------------------- primitive records
def triangle_prims(verts, faces):
    """prim_setup_kernel (build.cu:50-71): exact box, centroid ((a + b) + c) * (1.0f / 3.0f).  `verts` are the
    float32 positions [n_verts, 3] (any stride already resolved), `faces` [n, 3]."""
    v = np.asarray(verts, F32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    a, b, cc = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    ka, kb, kc = fkey(a), fkey(b), fkey(cc)
    lo = funkey(np.minimum(ka, np.minimum(kb, kc)))
    hi = funkey(np.maximum(ka, np.maximum(kb, kc)))
    third = F32(1.0) / F32(3.0)
    with np.errstate(over="ignore", invalid="ignore"):
        c = ((a + b) + cc) * third
    return lo, hi, c


def box_prims(boxes6):
    """box_setup_kernel (build.cu:99-116): the box itself, centre (hi + lo) / 2."""
    b = np.asarray(boxes6, F32).reshape(-1, 6)
    lo, hi = b[:, :3].copy(), b[:, 3:].copy()
    with np.errstate(over="ignore", invalid="ignore"):
        c = (hi + lo) / F32(2)
    return lo, hi, c


def sphere_prims(centers, radii):
    """sphere_boxes_kernel (prims.cu:30-44): c - r, c + r, then the box rule."""
    c = np.asarray(centers, F32).reshape(-1, 3)
    r = np.asarray(radii, F32).reshape(-1, 1)
    with np.errstate(over="ignore", invalid="ignore"):
        return box_prims(np.concatenate([c - r, c + r], axis=1))


# ----------------------------------------------------------------------------- Morton pre-order
def spread_bits_10(v):
    """radix_sort.cuh:16-23."""
    v = np.asarray(v, np.uint32) & np.uint32(0x3FF)
    v = (v | (v << np.uint32(16))) & np.uint32(0x030000FF)
    v = (v | (v << np.uint32(8))) & np.uint32(0x0300F00F)
    v = (v | (v << np.uint32(4))) & np.uint32(0x030C30C3)
    v = (v | (v << np.uint32(2))) & np.uint32(0x09249249)
    return v


def morton_keys(c, smin, smax):
    """morton_kernel (radix_sort.cuh:26-35) with the host's scale (build.cu:1365-1367): (c - smin) * (1024 / extent),
    a zero scale on a flat axis, truncated and clamped to [0, 1023], interleaved x << 2 | y << 1 | z."""
    smin, smax = np.asarray(smin, F32), np.asarray(smax, F32)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        ext = smax - smin
        sinv = np.where(smax > smin, F32(1024.0) / np.where(smax > smin, ext, F32(1)), F32(0)).astype(F32)
        q = (np.asarray(c, F32) - smin) * sinv
    qi = np.clip(cuda_f2i(q), 0, 1023).astype(np.uint32)
    return (spread_bits_10(qi[:, 0]) << np.uint32(2)) | (spread_bits_10(qi[:, 1]) << np.uint32(1)) | spread_bits_10(qi[:, 2])


def morton_order(c, smin, smax):
    """build.cu:1368-1388: slot s of the builder holds primitive order[s].  More than kSubtree primitives: a stable
    sort on key bits 6..29 (radix_sort_pairs(..., 6, 30, ...)); otherwise the identity."""
    n = len(c)
    if n <= K_SUBTREE:
        return np.arange(n, dtype=np.int64)
    return np.argsort(morton_keys(c, smin, smax) >> np.uint32(6), kind="stable").astype(np.int64)


# ----------------------------------------------------------------------------- segmented helpers
def _seg_scan(keys, seg, op, reverse=False):
    """Inclusive scan of uint32 `keys` [m, k] with `op` (np.minimum / np.maximum) that restarts where the
    non-decreasing `seg` [m] changes.  The segment goes into the high 32 bits so that the scan cannot carry over a
    border: later segments get smaller high words for a minimum, larger ones for a maximum."""
    seg = seg.astype(np.uint64)
    high = seg if (op is np.maximum) != reverse else seg.max(initial=0) - seg
    v = (high[:, None] << np.uint64(32)) | keys.astype(np.uint64)
    if reverse:
        v = v[::-1]
    v = op.accumulate(v, axis=0)
    if reverse:
        v = v[::-1]
    return (v & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def _sweep(seg, bins, klo, khi, nseg, B):
    """sweep_axis (build_common.cuh:169-258) of every segment at once on one axis.  Only boundaries just above a
    non-empty bin give distinct partitions; the cost of each is the cost of every boundary up to the next non-empty
    bin, so the first minimum over them is the sweep's.  Returns (cost [nseg] float32 -- FLT_MAX without a
    candidate, cut [nseg] -- left iff bin < cut)."""
    gk = seg * B + bins
    perm = np.argsort(gk, kind="stable")
    gks = gk[perm]
    m = len(gks)
    starts = np.flatnonzero(np.r_[True, gks[1:] != gks[:-1]])
    gseg, gbin = gks[starts] // B, gks[starts] % B
    gcnt = np.diff(np.r_[starts, m])
    glo = np.minimum.reduceat(klo[perm], starts, axis=0)
    ghi = np.maximum.reduceat(khi[perm], starts, axis=0)
    pre_lo, pre_hi = _seg_scan(glo, gseg, np.minimum), _seg_scan(ghi, gseg, np.maximum)
    suf_lo, suf_hi = _seg_scan(glo, gseg, np.minimum, True), _seg_scan(ghi, gseg, np.maximum, True)
    cs = np.cumsum(gcnt)
    first = np.r_[True, gseg[1:] != gseg[:-1]]
    seg_base = np.zeros(nseg, np.int64)
    seg_base[gseg[first]] = cs[first] - gcnt[first]
    seg_tot = np.zeros(nseg, np.int64)
    np.add.at(seg_tot, gseg, gcnt)
    cand = np.flatnonzero(~first)  # group g: the boundary just below its bin
    nl = cs[cand - 1] - seg_base[gseg[cand]]
    nr = seg_tot[gseg[cand]] - nl
    with np.errstate(over="ignore", invalid="ignore"):
        cl = nl.astype(F32) * box_area(funkey(pre_lo[cand - 1]), funkey(pre_hi[cand - 1]))
        cr = nr.astype(F32) * box_area(funkey(suf_lo[cand]), funkey(suf_hi[cand]))
        cost = cl + cr
    ok = cost < FLT_MAX
    cand, cost = cand[ok], cost[ok]
    best = np.full(nseg, FLT_MAX, F32)
    cut = np.zeros(nseg, np.int64)
    if len(cand):
        cs_seg = gseg[cand]
        np.minimum.at(best, cs_seg, cost)
        hit = cost == best[cs_seg]
        s_hit, first_hit = np.unique(cs_seg[hit], return_index=True)  # candidates are in boundary order
        cut[s_hit] = gbin[cand[hit][first_hit]]
    return best, cut


# ----------------------------------------------------------------------------- the builder
def build(prims, bin_size=64, min_leaf_primitives=4, max_tree_depth=256):
    """build_on_device (build.cu:1277-1471) on primitive records (lo, hi, c) [n, 3] float32.

    Returns a dict: nodes (NODE_DTYPE), indices (uint32), stats (max_tree_depth, num_leaf_nodes, num_branch_nodes),
    branch_sizes (primitives of every branch node), median (per branch node: cut at the median index), morton
    (whether the Morton pre-order ran) and per-node size / depth / parent / is_branch in build order."""
    from nanort_b200.scenes import NODE_DTYPE

    lo, hi, c = (np.asarray(a, F32).reshape(-1, 3) for a in prims)
    n = len(lo)
    assert n >= 1
    B = int(bin_size)
    assert 2 <= B <= 256
    min_leaf = max(int(min_leaf_primitives), 1)
    max_depth = int(max_tree_depth)
    klo_p, khi_p = fkey(lo), fkey(hi)
    root_lo, root_hi = funkey(klo_p.min(axis=0)), funkey(khi_p.max(axis=0))
    order = morton_order(c, root_lo, root_hi)
    cs, klo, khi = c[order], klo_p[order], khi_p[order]
    cur = np.arange(n, dtype=np.int64)  # cur[position] = slot

    # node table, grown level by level
    N_l, N_r, N_depth = [np.array([0])], [np.array([n])], [np.array([0])]
    N_klo, N_khi = [klo_p.min(axis=0)[None]], [khi_p.max(axis=0)[None]]
    B_id, B_left, B_axis, B_median = [np.zeros(0, np.int64)], [np.zeros(0, np.int64)], [np.zeros(0, np.int64)], [np.zeros(0, bool)]
    level_ids = np.array([0])
    n_nodes = 1
    while len(level_ids):
        l = np.concatenate(N_l)[level_ids]
        r = np.concatenate(N_r)[level_ids]
        depth = np.concatenate(N_depth)[level_ids]
        split = ((r - l) > min_leaf) & (depth < max_depth)
        ids, l, r, depth = level_ids[split], l[split], r[split], depth[split]
        if not len(ids):
            break
        srt = np.argsort(l)
        ids, l, r, depth = ids[srt], l[srt], r[srt], depth[srt]
        nseg = len(ids)
        length = r - l
        seg = np.repeat(np.arange(nseg), length)
        offs = np.cumsum(length) - length
        pos = np.repeat(l, length) + (np.arange(len(seg)) - np.repeat(offs, length))
        slots = cur[pos]
        cc, kl, kh = cs[slots], klo[slots], khi[slots]
        bmin = funkey(np.concatenate(N_klo)[ids])
        bmax = funkey(np.concatenate(N_khi)[ids])
        bins = np.empty((len(seg), 3), np.int64)
        cost = np.empty((nseg, 3), F32)
        cut = np.empty((nseg, 3), np.int64)
        for a in range(3):
            inv = inv_extent(bmin[:, a], bmax[:, a], B)
            bins[:, a] = bin_of(cc[:, a], bmin[seg, a], inv[seg], B)
            cost[:, a], cut[:, a] = _sweep(seg, bins[:, a], kl, kh, nseg, B)
        ax = np.where(cost[:, 0] > cost[:, 1], 1, 0)
        ax = np.where(cost[np.arange(nseg), ax] > cost[:, 2], 2, ax)
        median = ~(cost[np.arange(nseg), ax] < FLT_MAX)
        rank = np.arange(len(seg)) - offs[seg]
        go_left = np.where(median[seg], rank < (length >> 1)[seg], bins[np.arange(len(seg)), ax[seg]] < cut[seg, ax[seg]])
        perm = np.argsort(2 * seg + (~go_left), kind="stable")  # stable partition inside every segment
        cur[pos] = slots[perm]
        nl = np.bincount(seg, weights=go_left, minlength=nseg).astype(np.int64)
        assert np.all((nl > 0) & (nl < length))
        # children: left [l, l + nl), right [l + nl, r); boxes = exact unions of the members
        c_l = np.stack([l, l + nl], 1).reshape(-1)
        c_r = np.stack([l + nl, r], 1).reshape(-1)
        starts = np.stack([offs, offs + nl], 1).reshape(-1)
        N_l.append(c_l)
        N_r.append(c_r)
        N_depth.append(np.repeat(depth + 1, 2))
        N_klo.append(np.minimum.reduceat(kl[perm], starts, axis=0))
        N_khi.append(np.maximum.reduceat(kh[perm], starts, axis=0))
        new_ids = n_nodes + np.arange(2 * nseg)
        B_id.append(ids)
        B_left.append(new_ids[0::2])
        B_axis.append(np.where(median, (ax + 2) % 3, ax))
        B_median.append(median)
        n_nodes += 2 * nseg
        level_ids = new_ids

    l = np.concatenate(N_l)
    r = np.concatenate(N_r)
    depth = np.concatenate(N_depth)
    bmin = funkey(np.concatenate(N_klo))
    bmax = funkey(np.concatenate(N_khi))
    # DFS pre-order, lower side first: a node precedes everything in its range that is deeper, and ranges that start
    # further left come first
    pre_order = np.lexsort((depth, l))
    pre = np.empty(n_nodes, np.int64)
    pre[pre_order] = np.arange(n_nodes)
    nodes = np.zeros(n_nodes, NODE_DTYPE)
    nodes["bmin"][pre] = bmin
    nodes["bmax"][pre] = bmax
    b_id = np.concatenate(B_id)
    is_branch = np.zeros(n_nodes, bool)
    left = np.zeros(n_nodes, np.int64)
    axis = np.zeros(n_nodes, np.int64)
    is_branch[b_id] = True
    left[b_id] = np.concatenate(B_left)
    axis[b_id] = np.concatenate(B_axis)
    nodes["flag"][pre] = np.where(is_branch, 0, 1)
    nodes["axis"][pre] = np.where(is_branch, axis, 0)
    d0 = np.where(is_branch, pre[left], r - l)
    d1 = np.where(is_branch, pre[np.where(is_branch, left + 1, 0)], l)
    nodes["data"][pre, 0] = d0
    nodes["data"][pre, 1] = d1
    indices = order[cur].astype(np.uint32)
    n_branch = len(b_id)
    parent = np.full(n_nodes, -1, np.int64)
    parent[left[b_id]] = b_id
    parent[left[b_id] + 1] = b_id
    return {
        "nodes": nodes,
        "indices": indices,
        "stats": {"max_tree_depth": int(depth.max()), "num_leaf_nodes": n_nodes - n_branch,
                  "num_branch_nodes": n_branch},
        "branch_sizes": (r - l)[b_id],
        "median": np.concatenate(B_median),
        "morton": n > K_SUBTREE,
        # per node, in build order (root first): primitives, depth, parent (-1 for the root), branch or leaf
        "size": r - l,
        "depth": depth,
        "parent": parent,
        "is_branch": is_branch,
    }


def phases(model):
    """Which pieces of the device builder split a node of this tree (by the node's size, build.cu:166-178, 349-358,
    926, 1020): "level" (> kMid: split_large_kernel + flag / scatter / fix_median), "mid" (kSubtree+1..kMid:
    midtree_kernel), "subtree" (K_SMALL+1..kSubtree: subtree_kernel's binned sweep), "small" (<= 32: small_block)."""
    s = model["branch_sizes"]
    out = set()
    if np.any(s > K_MID):
        out.add("level")
    if np.any((s > K_SUBTREE) & (s <= K_MID)):
        out.add("mid")
    if np.any((s > K_SMALL) & (s <= K_SUBTREE)):
        out.add("subtree")
    if np.any(s <= K_SMALL):
        out.add("small")
    return out


def build_triangles(verts, faces, **opts):
    return build(triangle_prims(verts, faces), **opts)


# ----------------------------------------------------------------------------- float64 ideal
def sah_decisions_f64(nodes, indices, prims, B):
    """For every branch node of a tree (NODE_DTYPE + indices over primitive records (lo, hi, c)), written from the
    definition of the binned SAH rather than from the model: the float32 bin of every member centroid over the node's
    box is taken as given; the cost N_L * area(L) + N_R * area(R) of every boundary with both sides non-empty, on
    every axis, is evaluated in float64 on the exact unions; the chosen partition is the node's two children.

    Returns (node index [k], chosen cost [k], optimal cost [k]) for the branch nodes that have a candidate."""
    lo, hi, c = (np.asarray(a, F32).reshape(-1, 3) for a in prims)
    lo64, hi64 = lo.astype(np.float64), hi.astype(np.float64)
    n = len(nodes)
    leaf = nodes["flag"] == 1
    # ranges of indices_ per node, bottom-up (children follow their parent)
    first = np.zeros(n, np.int64)
    count = np.zeros(n, np.int64)
    d0, d1 = nodes["data"][:, 0].astype(np.int64), nodes["data"][:, 1].astype(np.int64)
    for i in range(n - 1, -1, -1):
        if leaf[i]:
            first[i], count[i] = d1[i], d0[i]
        else:
            first[i], count[i] = first[d0[i]], count[d0[i]] + count[d1[i]]

    def area64(blo, bhi):
        d = bhi - blo
        return 2.0 * (d[..., 0] * d[..., 1] + d[..., 1] * d[..., 2] + d[..., 2] * d[..., 0])

    out_i, out_chosen, out_best = [], [], []
    for i in np.flatnonzero(~leaf):
        p = indices[first[i]:first[i] + count[i]].astype(np.int64)
        nb_min, nb_max = nodes["bmin"][i], nodes["bmax"][i]
        best = np.inf
        for a in range(3):
            b = bin_of(c[p, a], nb_min[a], inv_extent(nb_min[a], nb_max[a], B), B)
            cnt = np.bincount(b, minlength=B)
            bl = np.full((B, 3), np.inf)
            bh = np.full((B, 3), -np.inf)
            np.minimum.at(bl, b, lo64[p])
            np.maximum.at(bh, b, hi64[p])
            # boundary i: bins [0, i) | [i, B)
            nl = np.cumsum(cnt)[:-1]
            nr = len(p) - nl
            ll, lh = np.minimum.accumulate(bl)[:-1], np.maximum.accumulate(bh)[:-1]
            rl, rh = np.minimum.accumulate(bl[::-1])[::-1][1:], np.maximum.accumulate(bh[::-1])[::-1][1:]
            ok = (nl > 0) & (nr > 0)
            if np.any(ok):
                with np.errstate(invalid="ignore", over="ignore"):
                    cost = nl[ok] * area64(ll[ok], lh[ok]) + nr[ok] * area64(rl[ok], rh[ok])
                best = min(best, float(cost.min()))
        if not np.isfinite(best):
            continue
        L, R = d0[i], d1[i]
        chosen = count[L] * area64(nodes["bmin"][L].astype(np.float64), nodes["bmax"][L].astype(np.float64)) + \
            count[R] * area64(nodes["bmin"][R].astype(np.float64), nodes["bmax"][R].astype(np.float64))
        out_i.append(i)
        out_chosen.append(float(chosen))
        out_best.append(best)
    return np.array(out_i, np.int64), np.array(out_chosen), np.array(out_best)


def sah_cost_f64(nodes):
    """SAH cost of a tree in float64 with unit traversal and intersection costs: (sum of branch areas + sum of leaf
    area * primitive count) / root area."""
    d = nodes["bmax"].astype(np.float64) - nodes["bmin"].astype(np.float64)
    area = 2.0 * (d[:, 0] * d[:, 1] + d[:, 1] * d[:, 2] + d[:, 2] * d[:, 0])
    leaf = nodes["flag"] == 1
    w = np.where(leaf, nodes["data"][:, 0].astype(np.float64), 1.0)
    return float((area * w).sum() / area[0])
