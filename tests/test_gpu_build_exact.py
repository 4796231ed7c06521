"""The production builder (`NRT_BUILD_FAST`, csrc/build.cu) against its host model (`tests/build_model.py`): the node
array, `indices_` and the statistics must equal the model's bit for bit.  Hits do not depend on topology, so this is
what catches a builder that takes a valid but different split (wrong axis, wrong tie, wrong candidate plane, wrong
centroid arithmetic, wrong median index, wrong Morton order).

Every case first asserts which pieces of the device builder it reaches, from the model's node sizes:
"level" (> 2048 primitives: split_large_kernel, flag / scatter_large_kernel, fix_median_kernel), "mid" (129..2048:
midtree_kernel), "subtree" (33..128: subtree_kernel's binned sweep) and "small" (<= 32: small_block)."""
import numpy as np
import pytest

import build_model as M
from helpers import degenerate_mesh, random_soup

pytestmark = pytest.mark.gpu

ALL = {"level", "mid", "subtree", "small"}


def _same_bits(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def assert_tree_equal(got_nodes, got_idx, model):
    """Every field of every node and every index, bit for bit; a mismatch names the first differing node."""
    want = model["nodes"]
    assert len(got_nodes) == len(want), (len(got_nodes), len(want))
    for k in ("bmin", "bmax", "flag", "axis", "data"):
        bad = np.flatnonzero((got_nodes[k].view(np.uint32) != want[k].view(np.uint32)).reshape(len(want), -1).any(1))
        assert len(bad) == 0, (k, int(bad[0]), got_nodes[bad[0]], want[bad[0]], len(bad))
    bad = np.flatnonzero(got_idx != model["indices"])
    assert len(bad) == 0, ("indices", int(bad[0]), len(bad))


def assert_stats_equal(got, model):
    for k, v in model["stats"].items():
        assert got[k] == v, (k, got, model["stats"])


def depth_limited_phases(model, max_depth, min_leaf):
    """Pieces whose splits made a leaf only because of the depth limit."""
    lim = (~model["is_branch"]) & (model["depth"] >= max_depth) & (model["size"] > max(min_leaf, 1))
    par = model["parent"][lim]
    return M.phases({"branch_sizes": model["size"][par[par >= 0]]})


# ------------------------------------------------------------------------------------------- geometry
def _soup(n, seed):
    return random_soup(np.random.default_rng(seed), n)


def _tris(c, size, rng):
    """Triangles of the given half-size around centres c [n, 3] (float64)."""
    t = c[:, None, :] + rng.uniform(-1, 1, (len(c), 3, 3)) * np.asarray(size)[..., None, None]
    return t.reshape(-1, 3).astype(np.float32), np.arange(3 * len(c), dtype=np.uint32).reshape(-1, 3)


def _geometry(kind):
    rng = np.random.default_rng(77)
    if kind.startswith("soup:"):
        _, n, seed = kind.split(":")
        return _soup(int(n), int(seed))
    if kind.startswith("deg:"):
        return degenerate_mesh(kind[4:])
    if kind == "plane":  # every vertex in z = 0: centroids in a plane, zero extent on z (inv = 0)
        v, f = _soup(3000, 5)
        v[:, 2] = 0.0
        return v, f
    if kind == "line_y":  # centroids on a line along y, boxes of varying width
        k = 2500
        y = np.arange(k, dtype=np.float64) * 0.37
        c = np.stack([np.zeros(k), y, np.zeros(k)], 1)
        v, f = _tris(c, 0.0, rng)
        v = v.reshape(-1, 3, 3)
        v[:, 1, 0] += (np.arange(k) % 7).astype(np.float32)  # boxes differ, centroids move only on x by a bounded amount
        v[:, 2, 0] -= (np.arange(k) % 7).astype(np.float32)
        return v.reshape(-1, 3), f
    if kind == "morton_cluster":
        # 3000 triangles inside ONE cell of the top 24 Morton bits (1/256 of the scene box per axis) but spread over
        # its 4x4x4 sub-cells in a scrambled order, plus 2000 spread over the box: which of them share a leaf or a
        # median half depends on the sort being stable on bits 6..29 only
        c0 = rng.uniform(0, 256, (2000, 3))
        c0[0], c0[1] = 0.0, 256.0
        cell = (np.floor(rng.uniform(0, 4, (3000, 3))) + 0.5) * 0.25 + 100.0  # sub-cells of the cell [100, 101)
        c = np.concatenate([cell, c0])
        v, f = _tris(c, np.r_[np.full(3000, 1e-3), np.full(2000, 0.5)], rng)
        return v, f
    if kind.startswith("sweep_tie:"):
        # three clusters of m copies along x, mirror-symmetric in their BOXES, so {A} | {B, C} and {A, B} | {C} cost
        # exactly the same; B's centroid sits just left of the middle (bin 31 of 64), so the first partition spans
        # boundaries 1..31 and the second 32..63, and only the first-minimum rule picks {A} | {B, C}
        m = int(kind.split(":")[1])
        ta = [[-16, 0, 0], [-16, 1, 0], [-15, 0.5, 1]]
        tb = [[-1, 0, 0], [1, 1, 0], [-0.5, 0.5, 1]]
        tc = [[16, 0, 0], [16, 1, 0], [15, 0.5, 1]]
        v = np.array(ta * m + tb * m + tc * m, np.float32)
        return v, np.arange(len(v), dtype=np.uint32).reshape(-1, 3)
    if kind == "signed_zero":  # coordinates that are exactly -0.0 and +0.0 in every axis
        v, f = _soup(4000, 9)
        z = rng.random(v.shape) < 0.3
        v[z] = np.where(rng.random(int(z.sum())) < 0.5, np.float32(-0.0), np.float32(0.0))
        return v, f
    if kind == "huge":  # around 1e19: box areas overflow to inf near the root, so those nodes fall back to median cuts
        v, f = _soup(6000, 3)
        v = v / np.maximum(np.abs(v).max(), 1e-30) * np.float32(3e19)
        v[:3000] *= np.float32(1e-6)  # small nodes lower down split by SAH again
        return v.astype(np.float32), f
    if kind == "denormal":  # a cluster whose x extent is denormal (B / extent = inf) inside a normal scene
        v, f = _soup(3000, 4)
        d, fd = _tris(rng.uniform(0, 1, (1500, 3)), 0.01, rng)
        d[:, 0] = (rng.integers(0, 64, len(d)) * 2.0 ** -149).astype(np.float32)  # 0 .. 63 denormal steps
        return np.concatenate([v, d]), np.concatenate([f, fd + len(v)])
    if kind == "denormal_scene":  # the whole scene's x extent is denormal: the Morton scale on x is inf too
        d, fd = _tris(rng.uniform(0, 1, (2500, 3)), 0.01, rng)
        d[:, 0] = (rng.integers(0, 64, len(d)) * 2.0 ** -149).astype(np.float32)
        return d, fd
    from nanort_b200 import scenes as S

    name, _, arg = kind.partition(":")  # "terrain:96" is terrain(n=96)
    return S.make_scene(name, **(dict(n=int(arg)) if arg else {}))


# (geometry, build options, pieces the tree must reach)
CASES = [
    # sizes at every class border
    ("soup:1:1", dict(min_leaf_primitives=0), set()),
    ("soup:2:2", dict(min_leaf_primitives=1), {"small"}),
    ("soup:3:3", dict(min_leaf_primitives=0), {"small"}),
    ("soup:31:4", dict(min_leaf_primitives=1), {"small"}),
    ("soup:32:5", dict(min_leaf_primitives=1), {"small"}),
    ("soup:33:6", dict(min_leaf_primitives=1), {"subtree", "small"}),
    ("soup:127:7", {}, {"subtree", "small"}),
    ("soup:128:8", {}, {"subtree", "small"}),
    ("soup:129:9", {}, {"mid", "subtree", "small"}),
    ("soup:2047:10", {}, {"mid", "subtree", "small"}),
    ("soup:2048:11", {}, {"mid", "subtree", "small"}),
    ("soup:2049:12", {}, ALL),
    ("sphere_grid", {}, ALL),
    ("terrain", {}, ALL),
    # bin counts, including ones that are not a multiple of 32 (uneven per-lane chunks in sweep_axis)
    ("soup:6000:20", dict(bin_size=2), ALL),
    ("soup:6000:21", dict(bin_size=3), ALL),
    ("soup:6000:22", dict(bin_size=33), ALL),
    ("soup:6000:23", dict(bin_size=100), ALL),
    ("soup:6000:24", dict(bin_size=255), ALL),
    ("soup:6000:25", dict(bin_size=256), ALL),
    # leaf sizes; 200 > kSubtree: leaves straight out of the level-synchronous and the middle phase
    ("soup:6000:30", dict(min_leaf_primitives=0), ALL),
    ("soup:6000:31", dict(min_leaf_primitives=1), ALL),
    ("soup:6000:32", dict(min_leaf_primitives=13), ALL),
    ("soup:6000:33", dict(min_leaf_primitives=200), {"level", "mid"}),
    ("terrain:96", dict(min_leaf_primitives=200), {"level", "mid"}),
    # depth limits
    ("soup:6000:40", dict(max_tree_depth=0), set()),
    ("soup:6000:41", dict(max_tree_depth=1), {"level"}),
    # geometry
    ("deg:one", {}, set()),
    ("deg:five", dict(min_leaf_primitives=1), {"small"}),
    ("deg:identical", {}, ALL),
    ("deg:line", dict(min_leaf_primitives=2), {"mid", "subtree", "small"}),
    ("line_y", {}, ALL),
    ("plane", {}, ALL),
    ("morton_cluster", {}, ALL),
    ("sweep_tie:8", dict(min_leaf_primitives=1), {"small"}),
    ("sweep_tie:20", {}, {"subtree", "small"}),
    ("sweep_tie:300", {}, {"mid", "subtree", "small"}),
    ("sweep_tie:1000", {}, ALL),
    ("signed_zero", {}, ALL),
    ("huge", {}, ALL),
    ("denormal", {}, ALL),
    ("denormal_scene", dict(min_leaf_primitives=1), ALL),
]

# the depth limit reached inside each piece: (geometry, max_tree_depth, piece whose splits hit it)
DEPTH_CASES = [
    ("soup:9000:50", 2, "level"),
    ("soup:9000:51", 5, "mid"),
    ("soup:9000:52", 10, "subtree"),
    ("soup:9000:53", 12, "small"),
]


def _build_and_compare(v, f, okw, model=None, stride_floats=3):
    from nanort_b200 import api

    if model is None:
        model = M.build_triangles(v, f, **okw)
    buf = v
    if stride_floats != 3:
        buf = np.full((len(v), stride_floats), np.float32(-7.5e8), np.float32)  # junk in the padding
        buf[:, :3] = v
    acc = api.BVHAccel()
    assert acc.Build(len(f), buf, f, api.BVHBuildOptions(**okw), vertex_stride_bytes=4 * stride_floats)
    assert_tree_equal(acc.GetNodes(), acc.GetIndices(), model)
    assert_stats_equal(acc.GetStatistics(), model)
    bmin, bmax = acc.BoundingBox()
    assert _same_bits(bmin, model["nodes"]["bmin"][0]) and _same_bits(bmax, model["nodes"]["bmax"][0])
    return model


@pytest.mark.parametrize("kind,okw,reach", CASES, ids=[f"{c[0]}-{'-'.join(f'{k}={v}' for k, v in c[1].items())}"
                                                      for c in CASES])
def test_triangle_tree_equals_the_model(kind, okw, reach):
    v, f = _geometry(kind)
    model = M.build_triangles(v, f, **okw)
    assert M.phases(model) == reach, (M.phases(model), reach)
    assert model["morton"] == (len(f) > 128)
    if kind in ("deg:identical", "huge"):
        assert model["median"].any()
    if kind.startswith("sweep_tie:"):
        m = len(f) // 3
        assert model["size"][1:3].tolist() == [m, 2 * m]
    _build_and_compare(v, f, okw, model)


@pytest.mark.parametrize("kind,depth,piece", DEPTH_CASES)
def test_depth_limit_inside_each_piece(kind, depth, piece):
    v, f = _geometry(kind)
    okw = dict(max_tree_depth=depth, min_leaf_primitives=1)
    model = M.build_triangles(v, f, **okw)
    assert piece in depth_limited_phases(model, depth, 1), depth_limited_phases(model, depth, 1)
    _build_and_compare(v, f, okw, model)


@pytest.mark.parametrize("stride_floats", [4, 5])
def test_vertex_strides(stride_floats):
    v, f = _geometry("terrain:40")
    model = M.build_triangles(v, f)
    assert M.phases(model) == ALL
    _build_and_compare(v, f, {}, model, stride_floats=stride_floats)


def test_spheres_equal_the_model():
    from nanort_b200 import api

    rng = np.random.default_rng(5)
    c = rng.uniform(-20, 20, (6000, 3)).astype(np.float32)
    c[:500] = c[500:1000]  # coincident centres
    r = rng.uniform(0.0, 0.5, 6000).astype(np.float32)
    model = M.build(M.sphere_prims(c, r))
    assert M.phases(model) == ALL
    acc = api.BVHAccel()
    assert acc.BuildSpheres(c, r)
    assert_tree_equal(acc.GetNodes(), acc.GetIndices(), model)
    assert_stats_equal(acc.GetStatistics(), model)


@pytest.mark.parametrize("okw", [{}, dict(min_leaf_primitives=1, bin_size=33)])
def test_boxes_equal_the_model(okw):
    from nanort_b200 import api

    rng = np.random.default_rng(6)
    lo = rng.uniform(-50, 50, (5000, 3)).astype(np.float32)
    ext = rng.exponential(1.0, (5000, 3)).astype(np.float32)
    ext[:400] = 0.0  # point boxes
    boxes = np.concatenate([lo, lo + ext], axis=1)
    model = M.build(M.box_prims(boxes), **okw)
    assert M.phases(model) == ALL
    acc = api.BVHAccel()
    assert acc.BuildBoxes(boxes, api.BVHBuildOptions(**okw))
    assert_tree_equal(acc.GetNodes(), acc.GetIndices(), model)
    assert_stats_equal(acc.GetStatistics(), model)


@pytest.mark.parametrize("n,reach", [(24, {"small"}), (300, {"mid", "subtree", "small"})])
def test_scene_top_level_equals_the_model(n, reach):
    """Scene::Commit(BUILD_FAST): the top level is the production builder over the instances' world boxes with
    min_leaf_primitives = 1 (nanosg.h:731-732)."""
    from nanort_b200 import api, scenes as S

    insts = S.instances_mixed(n=n)
    accels, sc = {}, api.Scene()
    for v, f, x in insts:
        key = (v.ctypes.data, f.ctypes.data)
        if key not in accels:
            a = api.BVHAccel()
            a.Build(len(f), v, f)
            accels[key] = a
        sc.AddNode(accels[key], x)
    assert sc.Commit(api.BUILD_FAST)
    st = sc.InstanceStates()
    model = M.build(M.box_prims(np.concatenate([st["xbmin"], st["xbmax"]], axis=1)), min_leaf_primitives=1)
    assert M.phases(model) == reach
    tn, ti = sc.GetTopLevel()
    assert_tree_equal(tn, ti, model)


def test_f64_accel_topology_equals_the_model():
    """BVHAccelF64.Build: the production tree over the float-rounded vertices, boxes refitted as exact double unions
    by f64_refit_kernel (whose arrival order at each branch varies; the result must not)."""
    from nanort_b200 import api, scenes as S

    v32, f = S.sphere_grid(nx=6, nz=6)
    rng = np.random.default_rng(8)
    v = v32.astype(np.float64) + rng.uniform(-1e-9, 1e-9, v32.shape)  # doubles that are not floats
    model = M.build_triangles(v.astype(np.float32), f)
    assert M.phases(model) == ALL
    acc = api.BVHAccelF64()
    assert acc.Build(len(f), v, f)
    nodes, idx = acc.GetNodes(), acc.GetIndices()
    want = model["nodes"]
    assert len(nodes) == len(want)
    for k in ("flag", "axis", "data"):
        assert _same_bits(nodes[k], want[k]), k
    assert _same_bits(idx, model["indices"])
    # exact double unions, bottom-up over the same topology
    tri = v[f.astype(np.int64)]
    lo, hi = tri.min(axis=1), tri.max(axis=1)
    bmin, bmax = np.zeros((len(want), 3)), np.zeros((len(want), 3))
    d0, d1 = want["data"][:, 0].astype(np.int64), want["data"][:, 1].astype(np.int64)
    for i in range(len(want) - 1, -1, -1):
        if want["flag"][i]:
            p = model["indices"][d1[i]:d1[i] + d0[i]]
            bmin[i], bmax[i] = lo[p].min(axis=0), hi[p].max(axis=0)
        else:
            bmin[i], bmax[i] = np.minimum(bmin[d0[i]], bmin[d1[i]]), np.maximum(bmax[d0[i]], bmax[d1[i]])
    assert _same_bits(nodes["bmin"], bmin) and _same_bits(nodes["bmax"], bmax)
    assert_stats_equal(acc.GetStatistics(), model)


@pytest.mark.parametrize("name", ["sphere_grid", "terrain"])
def test_production_tree_is_no_worse_than_the_reference_tree(name):
    """DESIGN.md §5: binning all three axes makes a better SAH tree than the reference-exact build (x only)."""
    from nanort_b200 import api, scenes as S

    v, f = S.make_scene(name)
    costs = {}
    for flags in (api.BUILD_FAST, api.BUILD_REFERENCE_TREE):
        acc = api.BVHAccel()
        assert acc.Build(len(f), v, f, flags=flags)
        costs[flags] = M.sah_cost_f64(acc.GetNodes())
    assert costs[api.BUILD_FAST] <= costs[api.BUILD_REFERENCE_TREE], costs
