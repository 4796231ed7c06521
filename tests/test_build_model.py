"""The host model of the production builder (`tests/build_model.py`) on its own, without a GPU: its trees are valid
nanort trees, its split choices are near-optimal by a float64 evaluation of the binned SAH written from the
definition, and its Morton key and float -> int conversion behave as the device's."""
import numpy as np
import pytest

import build_model as M
from helpers import check_tree_structure, degenerate_mesh, random_soup

INT_MAX, INT_MIN = 2 ** 31 - 1, -2 ** 31


def _scene(name, kw):
    from nanort_b200 import scenes as S

    if name.startswith("deg:"):
        return degenerate_mesh(name[4:])
    return S.make_scene(name, **kw)


@pytest.mark.parametrize("name,kw,okw", [
    ("cornell", {}, {}),
    ("cornell", {}, dict(min_leaf_primitives=1, bin_size=3)),
    ("sphere_grid", dict(nx=3, nz=3), {}),
    ("sphere_grid", {}, {}),
    ("terrain", dict(n=96), dict(bin_size=16)),
    ("terrain", dict(n=300), {}),
    ("terrain", dict(n=96), dict(max_tree_depth=9)),
    ("deg:one", {}, {}),
    ("deg:five", {}, dict(min_leaf_primitives=1)),
    ("deg:identical", {}, {}),
    ("deg:line", {}, dict(min_leaf_primitives=2)),
])
def test_model_tree_is_valid(name, kw, okw):
    v, f = _scene(name, kw)
    m = M.build_triangles(v, f, **okw)
    opts = {"min_leaf_primitives": 4, "max_tree_depth": 256, **okw}
    st = check_tree_structure(m["nodes"], m["indices"], v, f, min_leaf=max(opts["min_leaf_primitives"], 1),
                              max_depth=opts["max_tree_depth"])
    assert st == m["stats"]
    if name == "deg:identical":  # no plane separates the centroids: median cuts labelled (0 + 2) % 3
        assert m["median"].all() and np.all(m["nodes"]["axis"][m["nodes"]["flag"] == 0] == 2)


@pytest.mark.parametrize("seed", range(12))
def test_model_tree_is_valid_on_clustered_soups(seed):
    rng = np.random.default_rng(2000 + seed)
    n = [2, 31, 33, 127, 129, 2047, 2049, 5000][seed % 8] if seed < 8 else int(rng.integers(2, 12000))
    v, f = random_soup(rng, n)
    okw = dict(min_leaf_primitives=int(rng.choice([0, 1, 4, 13])), bin_size=int(rng.choice([2, 3, 33, 64, 255])),
               max_tree_depth=int(rng.choice([1, 8, 256])))
    m = M.build_triangles(v, f, **okw)
    st = check_tree_structure(m["nodes"], m["indices"], v, f, min_leaf=max(okw["min_leaf_primitives"], 1),
                              max_depth=okw["max_tree_depth"])
    assert st == m["stats"]


@pytest.mark.parametrize("name,kw,okw", [
    ("cornell", {}, dict(min_leaf_primitives=1)),
    ("sphere_grid", dict(nx=3, nz=3), {}),
    ("terrain", dict(n=64), dict(bin_size=16)),
    ("soup", dict(n=3000, seed=1), dict(bin_size=33)),
    ("soup", dict(n=3000, seed=2), dict(min_leaf_primitives=1)),
])
def test_model_choices_are_near_the_f64_optimum(name, kw, okw):
    """On every branch node with a candidate plane, the partition the model picks costs at most 4 float32 roundings
    more than the best candidate evaluated in float64 -- and never less, which would mean the f64 search missed the
    model's candidate."""
    if name == "soup":
        v, f = random_soup(np.random.default_rng(kw["seed"]), kw["n"])
    else:
        v, f = _scene(name, kw)
    m = M.build_triangles(v, f, **okw)
    prims = M.triangle_prims(v, f)
    B = okw.get("bin_size", 64)
    idx, chosen, best = M.sah_decisions_f64(m["nodes"], m["indices"], prims, B)
    assert len(idx) == m["stats"]["num_branch_nodes"] - int(m["median"].sum())
    assert np.all(chosen >= best * (1 - 1e-12)), np.max(best / chosen)
    rel = chosen / best - 1
    assert np.all(rel <= 4 * 2.0 ** -24), (float(rel.max()), int(idx[np.argmax(rel)]))


def test_cuda_float_to_int():
    x = np.array([np.nan, np.inf, -np.inf, 2.5, -2.5, 0.99999994, -0.0, 3e9, -3e9, 2147483520.0, -2147483648.0],
                 np.float32)
    assert M.cuda_f2i(x).tolist() == [0, INT_MAX, INT_MIN, 2, -2, 0, 0, INT_MAX, INT_MIN, 2147483520, INT_MIN]


def test_bin_of_edges():
    B = 64
    # a denormal extent: B / extent overflows to inf; (c - min) * inf is inf (-> B - 1) or NaN at c == min (-> 0)
    lo, hi = np.float32(0), np.float32(2.0 ** -140)
    inv = M.inv_extent(lo, hi, B)
    assert np.isinf(inv)
    assert M.bin_of(np.array([0, 2.0 ** -145, 2.0 ** -140], np.float32), lo, inv, B).tolist() == [0, B - 1, B - 1]
    # a flat axis: inv = 0, every centroid in bin 0
    assert M.inv_extent(np.float32(3), np.float32(3), B) == 0
    assert M.bin_of(np.array([3, 4], np.float32), np.float32(3), np.float32(0), B).tolist() == [0, 0]
    # the box max lands in the last bin, centroids below the box (rounding) in the first
    inv = M.inv_extent(np.float32(-1), np.float32(1), B)
    assert M.bin_of(np.array([1, -1.0000001, 0.0], np.float32), np.float32(-1), inv, B).tolist() == [B - 1, 0, B // 2]


def test_ordered_keys():
    x = np.array([-np.inf, -3.0, -1e-45, -0.0, 0.0, 1e-45, 2.0, np.inf], np.float32)
    k = M.fkey(x)
    assert np.all(np.diff(k.astype(np.int64)) > 0)  # -0.0 sorts below +0.0
    assert M.funkey(k).tobytes() == x.tobytes()


def test_morton_key_bits_and_clamping():
    smin, smax = np.zeros(3, np.float32), np.full(3, 1024, np.float32)
    c = np.array([[1023, 0, 0], [0, 1023, 0], [0, 0, 1023], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    assert M.morton_keys(c, smin, smax).tolist() == [0x24924924, 0x12492492, 0x09249249, 4, 2, 1]
    # the box max maps to 1024 and is clamped to 1023; below the box clamps to 0; NaN -> 0
    c = np.array([[1024, 1024, 1024], [-5, -5, -5], [np.nan, 0, 0]], np.float32)
    assert M.morton_keys(c, smin, smax).tolist() == [0x3FFFFFFF, 0, 0]
    # a flat axis gets a zero scale
    flat_max = np.array([1024, 0, 1024], np.float32)
    assert M.morton_keys(np.array([[512, 0, 0]], np.float32), smin, flat_max).tolist() == [M.spread_bits_10(512) << 2]
    # an extent of one denormal step: the scale is inf, so the axis is 0 or 1023
    tiny = np.array([2.0 ** -149, 1024, 1024], np.float32)
    keys = M.morton_keys(np.array([[0, 0, 0], [2.0 ** -149, 0, 0]], np.float32), smin, tiny)
    assert keys.tolist() == [0, 0x24924924]


def test_morton_order_is_stable_on_the_top_24_bits():
    rng = np.random.default_rng(3)
    # 64 cells of 1/256 of the box, each holding ~16 centroids spread over its 4x4x4 sub-cells
    c = (rng.integers(0, 4, (1000, 3)) / 4 + rng.uniform(0, 1 / 300, (1000, 3))).astype(np.float32)
    c[0], c[1] = 0.0, 1.0
    order = M.morton_order(c, np.zeros(3, np.float32), np.ones(3, np.float32))
    k = M.morton_keys(c, np.zeros(3, np.float32), np.ones(3, np.float32)) >> 6
    assert np.all(np.diff(k[order].astype(np.int64)) >= 0)
    same = np.flatnonzero(np.diff(k[order].astype(np.int64)) == 0)
    assert len(same) > 900 and np.all(order[same] < order[same + 1])  # equal prefixes keep the input order
    full = M.morton_keys(c, np.zeros(3, np.float32), np.ones(3, np.float32))
    assert not np.all(np.diff(full[order].astype(np.int64)) >= 0)  # ... which is not the order of the full key
    # at most kSubtree primitives: the identity
    assert M.morton_order(c[:128], np.zeros(3, np.float32), np.ones(3, np.float32)).tolist() == list(range(128))


def test_primitive_records():
    a = np.array([[1, 2, 3]], np.float32)
    b = np.array([[0.1, -0.0, 7]], np.float32)
    c = np.array([[0.2, 0.0, 5]], np.float32)
    lo, hi, cen = M.triangle_prims(np.concatenate([a, b, c]), np.array([[0, 1, 2]]))
    third = np.float32(1) / np.float32(3)
    assert cen.tobytes() == (((a + b) + c) * third).tobytes()
    assert lo.tobytes() == np.array([[0.1, -0.0, 3]], np.float32).tobytes()
    assert hi.tobytes() == np.array([[1, 2, 7]], np.float32).tobytes()
    lo, hi, cen = M.sphere_prims(np.array([[1, 2, 3]], np.float32), np.array([0.5], np.float32))
    assert lo.tolist() == [[0.5, 1.5, 2.5]] and hi.tolist() == [[1.5, 2.5, 3.5]] and cen.tolist() == [[1, 2, 3]]
