"""The sphere kind (csrc/prims.cu, traverse_spheres_kernel) ray by ray against the reference's own intersector walking
the DEVICE's tree: `orc.ReferenceSpheres.adopt(acc.GetNodes(), acc.GetIndices(), ...)` loads the device's arrays into
the unmodified BVHAccel<float> of examples/particle_primitive/main.cc, whose Traverse then runs its own
SphereIntersector over them.  Both walks test a leaf's slots in `indices_` order with the same arithmetic; they differ
only in the order they visit leaves (the reference: near child by direction sign; the device: by entry distance).
`classify_sphere_hits` asserts, with no budget:
  * the same hit mask;
  * every device record is `test_prim(ray, its prim)`, the reference's Intersect + PostTraversal for that pick: t and
    prim_id bit for bit, u / v bit for bit except one float ulp where the exact double atan2 / acos value lies within
    a few double ulps of a float32 rounding midpoint (a CUDA-versus-glibc last-ulp straddle, counted);
  * the same pick gives the whole record;
  * a different pick is (a) an exact t tie (equal values, so -0.0 and +0.0 tie) between spheres in different leaves, or (b) a below-min_t early stop: the
    reference's sphere test has no min_t, so a hit below min_t is accepted whenever its leaf's box passes the slab test
    over [min_t, best], after which best < min_t fails every further box -- which one is kept depends on the order.
Rays with a NaN / inf component, or for which some sphere yields a NaN t, are checked on their own (a NaN t is
accepted and later replaced, so the reference's own answer depends on its order): every device hit is
test_prim-consistent, and the mask is the reference's wherever no sphere yields a NaN t.
Each family first asserts, with the oracle, that it reaches what it is there to test."""
import threading

import numpy as np
import pytest

from edge_cases import hostile_rays
from nanort_b200 import api, scenes as S
from oracle import orc

pytestmark = pytest.mark.gpu

F32 = np.float32
EPS = np.finfo(np.float32).eps
STATS = {}  # scene -> class counts, printed by the last test (pytest -s)


def _have(cpp11=True):
    return orc.ReferenceSpheres.exact_available(cpp11)


def _need(cpp11=True):
    if not _have(cpp11):
        pytest.skip("oracle/_ref/libprim_ref{,03}.so not built from the current oracle/prim_ref_shim.cc "
                    "(no reference tree at build time)")


def _flags(cpp11):
    return 0 if cpp11 else api.TRAVERSE_CPP03_INVERSE


# ---------------------------------------------------------------------------------------------------- host restatements
def _normal(rays, rec, centers):
    """SphereIntersector::PostTraversal's normal in float32, the reference's operation order (main.cc:272-274)."""
    t = rec["t"].astype(F32)[:, None]
    n = (rays["org"] + t * rays["dir"]) - centers[rec["prim_id"]]
    ln = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    big = np.abs(ln) > EPS
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = (F32(1.0) / np.where(big, ln, F32(1.0))).astype(F32)
    return np.where(big[:, None], n * inv[:, None], n).astype(F32)


def _near_midpoint(d, k=4):
    """the double d lies within k double ulps of a float32 rounding midpoint"""
    f = d.astype(F32)
    out = np.zeros(len(d), bool)
    for nb in (np.nextafter(f, F32(np.inf)), np.nextafter(f, F32(-np.inf))):
        mid = (f.astype(np.float64) + nb.astype(np.float64)) / 2.0
        out |= np.abs(d - mid) <= k * np.spacing(np.abs(d))
    return out


def _uv_straddle(rays, rec, centers):
    n = _normal(rays, rec, centers).astype(np.float64)
    with np.errstate(invalid="ignore"):
        return (_near_midpoint(np.arctan2(n[:, 0], n[:, 2]) + np.pi),
                _near_midpoint(np.arccos(n[:, 1]) / np.pi))


def _disc(rays, prims, centers, radii):
    """SphereIntersector::Intersect's discriminant (main.cc:182-188) in float32, for the families' reach checks"""
    d, oc = rays["dir"], rays["org"] - centers[prims]
    with np.errstate(all="ignore"):
        a = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        b = F32(2.0) * ((d[:, 0] * oc[:, 0] + d[:, 1] * oc[:, 1]) + d[:, 2] * oc[:, 2])
        c = ((oc[:, 0] * oc[:, 0] + oc[:, 1] * oc[:, 1]) + oc[:, 2] * oc[:, 2]) - radii[prims] * radii[prims]
        return b * b - (F32(4.0) * a) * c


def _ulps(a, b):
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


# ---------------------------------------------------------------------------------------------------- the classifier
def classify_sphere_hits(ref, rays, got_h, got_m, centers, radii, topts=None, nan_t=None, root_leaf=False):
    """Device hits (got_h, got_m) vs the reference `ref` (ReferenceSpheres.adopt of the device's own tree), ray by ray;
    see the module docstring.  nan_t: rays for which some sphere yields a NaN t (ReferenceSpheres.nan_rays), None when
    the scene is built so that none can.  root_leaf: one leaf, one visiting order -- every pick must be the
    reference's.  Returns ({"hits", "same", "ties", "below_min_t", "uv_straddles", "relaxed"} counts, reference hits)."""
    centers = np.ascontiguousarray(centers, F32).reshape(-1, 3)
    wh, wm = ref.traverse(rays, topts=topts)
    gm, wm = np.asarray(got_m).astype(bool), wm.astype(bool)
    with np.errstate(invalid="ignore"):
        finite = np.isfinite(rays["org"]).all(axis=1) & np.isfinite(rays["dir"]).all(axis=1)
    nan_t = np.zeros(len(rays), bool) if nan_t is None else np.asarray(nan_t, bool)
    strict = finite & ~nan_t
    bad = np.flatnonzero((gm != wm) & ~nan_t)
    assert len(bad) == 0, f"hit mask differs on {len(bad)} rays, first {bad[:8]}: got {got_h[bad[:3]]} want {wh[bad[:3]]}"
    # every device record is the reference's record for the device's own pick
    hit = np.flatnonzero(gm)
    g = got_h[hit]
    rec, ok = ref.test_prim(rays[hit], g["prim_id"], topts=topts)
    assert ok.all(), f"the reference's Intersect refuses the device's pick on rays {hit[~ok][:8]}"
    same_t = (rec["t"].view(np.uint32) == g["t"].view(np.uint32)) & (rec["prim_id"] == g["prim_id"])
    assert same_t.all(), f"t differs from test_prim on rays {hit[~same_t][:8]}: got {g[~same_t][:3]} want {rec[~same_t][:3]}"
    out = {"hits": len(hit), "same": 0, "ties": 0, "below_min_t": 0, "uv_straddles": 0,
           "relaxed": int((~strict).sum())}
    uv_bad = (rec["u"].view(np.uint32) != g["u"].view(np.uint32)) | (rec["v"].view(np.uint32) != g["v"].view(np.uint32))
    if uv_bad.any():
        k = np.flatnonzero(uv_bad)
        su, sv = _uv_straddle(rays[hit[k]], rec[k], centers)
        du, dv = _ulps(rec["u"][k], g["u"][k]), _ulps(rec["v"][k], g["v"][k])
        fine = ((du == 0) | ((du == 1) & su)) & ((dv == 0) | ((dv == 1) & sv))
        assert fine.all(), f"u / v differ from test_prim outside a last-ulp straddle on rays {hit[k[~fine]][:8]}: " \
            f"got {g[k[~fine]][:3]} want {rec[k[~fine]][:3]}"
        out["uv_straddles"] = len(k)
    # picks against the reference's own walk, on the strict rays
    hs = np.flatnonzero(gm & strict)
    g, w, r = got_h[hs], wh[hs], ref.test_prim(rays[hs], got_h["prim_id"][hs], topts=topts)[0]
    same = g["prim_id"] == w["prim_id"]
    assert r[same].tobytes() == w[same].tobytes()
    out["same"] = int(same.sum())
    leaf = ref.leaf_of()
    unexplained = []
    for j in np.flatnonzero(~same):
        i = hs[j]
        tg, tw, pg, pw = F32(g["t"][j]), F32(w["t"][j]), int(g["prim_id"][j]), int(w["prim_id"][j])
        if not root_leaf and tg == tw and leaf[pg] != leaf[pw]:
            out["ties"] += 1  # (a); -0.0 ties +0.0 too: `t > *t_inout` is false either way
            continue
        mt = F32(rays["min_t"][i])
        below = [p for t, p in ((tg, pg), (tw, pw)) if t < mt]
        if not root_leaf and any(ref.box_hit(rays[i], leaf[p]) for p in below):
            out["below_min_t"] += 1  # (b)
            continue
        unexplained.append((int(i), g[j], w[j], int(leaf[pg]), int(leaf[pw])))
    assert not unexplained, f"{len(unexplained)} picks differ outside the two classes, first (ray, got, want, " \
        f"leaves): {unexplained[:3]}"
    return out, wh


def _check(name, acc, centers, radii, rays, topts=None, cpp11=True, nan_t="auto"):
    """Device Traverse of `rays` classified against the reference on the device's tree; returns (counts, device hits,
    device mask, reference hits)."""
    ref = orc.ReferenceSpheres.adopt(acc.GetNodes(), acc.GetIndices(), centers, radii, cpp11=cpp11)
    gh, gm = acc.Traverse(rays, options=topts, flags=_flags(cpp11))
    if isinstance(nan_t, str):
        nan_t = ref.nan_rays(rays, topts=topts) if len(radii) * len(rays) <= 4e8 else None
    res, wh = classify_sphere_hits(ref, rays, gh, gm, centers, radii, topts=topts, nan_t=nan_t,
                                   root_leaf=len(acc.GetNodes()) == 1)
    key = f"{name}{'' if cpp11 else ' cpp03'}"
    tot = STATS.setdefault(key, {})
    for k, v in res.items():
        tot[k] = tot.get(k, 0) + v
    return res, gh, gm, wh


# ---------------------------------------------------------------------------------------------------- sphere sets
def _random(n, seed, lo=-6.0, hi=6.0, rmax=None):
    rng = np.random.default_rng(seed)
    c = rng.uniform(lo, hi, size=(n, 3)).astype(F32)
    rmax = rmax or max(0.02, 2.0 * (hi - lo) / np.cbrt(n) / 3.0)
    return c, rng.uniform(0.2 * rmax, rmax, size=n).astype(F32)


def _scene(name):
    """(centers, radii, build options or None)"""
    if name == "one":
        return np.float32([[0.5, -0.25, 1.0]]), np.float32([1.0]), None
    if name == "two":
        return np.float32([[0, 0, 0], [0.75, 0.5, 0]]), np.float32([1.0, 0.75]), None
    if name == "three":
        return np.float32([[0, 0, 0], [0, 0, 0], [1.5, 0, 0]]), np.float32([1.0, 0.5, 1.0]), None
    if name.startswith("random"):
        n = int(name[6:])
        c, r = _random(n, seed=n)
        return c, r, None
    if name == "dup_one_leaf":  # 40 positions x 4 exact copies, all in one leaf: in-leaf ties, last slot wins
        c, r = _random(40, seed=5, rmax=0.8)
        return np.repeat(c, 4, axis=0), np.repeat(r, 4), api.BVHBuildOptions(min_leaf_primitives=200)
    if name == "dup_spread":  # 3000 positions x 3 copies, one sphere per leaf where the builder can split
        c, r = _random(3000, seed=6, rmax=0.5)
        return np.tile(c, (3, 1)), np.tile(r, 3), api.BVHBuildOptions(min_leaf_primitives=1)
    if name == "nested":  # concentric shells and overlapping offset spheres
        g = np.stack(np.meshgrid(*[np.arange(-4, 5, 2.0)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(F32)
        c = np.concatenate([g, g, g, g + F32(0.4)])
        r = np.concatenate([np.full(len(g), 0.3), np.full(len(g), 0.6), np.full(len(g), 0.9), np.full(len(g), 0.5)])
        return c.astype(F32), r.astype(F32), None
    if name == "zero_radius":
        c, r = _random(500, seed=8, rmax=0.6)
        r[::3] = 0.0
        return c, r, None
    if name == "tiny_radius":  # r*r = 1e-40 (denormal) and 0 (underflow); near-origin rays take the tangent branch
        g = np.stack(np.meshgrid(*[np.arange(-3, 4, 1.0)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(F32)
        r = np.where(np.arange(len(g)) % 2 == 0, 1e-20, 1e-23).astype(F32)
        return np.concatenate([g, g + F32(0.5)]), np.concatenate([r, np.full(len(g), 1e-4, F32)]), None
    if name == "huge_radius":  # r*r near 1e38 and overflowing to inf
        c, r = _random(64, seed=9, lo=-1e3, hi=1e3, rmax=1.0)
        r[:16] = np.float32(1e19) * (1 + np.arange(16, dtype=F32) / 16)
        r[16:20] = np.float32(3e19)
        return c, r, None
    if name == "far_centres":  # centres near 1e6, where org - center cancels
        c, r = _random(2000, seed=10, lo=1e6 - 50, hi=1e6 + 50, rmax=2.0)
        return c, r, None
    raise KeyError(name)


def _build(centers, radii, options=None, stride=12):
    acc = api.BVHAccel()
    assert acc.BuildSpheres(centers, radii, options=options, center_stride_bytes=stride)
    return acc


# ---------------------------------------------------------------------------------------------------- ray families
def _box(centers, radii):
    """the region the rays start in: around the spheres, huge radii left out"""
    r = np.minimum(radii, 4 * np.median(radii))[:, None]
    lo, hi = (centers - r).min(axis=0), (centers + r).max(axis=0)
    ext = np.maximum(hi - lo, F32(1.0))
    return (lo - 0.2 * ext).astype(F32), (hi + 0.2 * ext).astype(F32)


def _random_rays(centers, radii, n, seed):
    lo, hi = _box(centers, radii)
    r = S.incoherent_rays(lo, hi, n, seed=seed, axis_parallel_fraction=1.0 / 32)
    r["min_t"] = 0.0
    return r


def _unit(rng, n):
    d = rng.normal(size=(n, 3))
    return (d / np.linalg.norm(d, axis=1)[:, None]).astype(F32)


def _inside_min_t(centers, radii, n, seed):
    """from inside spheres with min_t past the sphere's own exit: the reference accepts that hit below min_t whenever
    the leaf's box reaches past min_t; max_t a little further, so that a kernel that rejected t < min_t would miss"""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, len(radii), n)
    r = np.zeros(n, S.RAY_DTYPE)
    r["dir"] = _unit(rng, n)
    r["org"] = centers[k] + (rng.uniform(-0.3, 0.3, (n, 1)) * radii[k, None] * r["dir"]).astype(F32)
    r["min_t"] = (radii[k] * rng.uniform(1.02, 2.0, n)).astype(F32)
    r["max_t"] = np.where(rng.uniform(size=n) < 0.5, r["min_t"] * F32(1.5), F32(1e30))
    return r


def _tangent(centers, radii, n, seed):
    """exact tangents: origin at centre + r e_a - s e_b, direction e_b (|disc| = 0 in float); and grazing rays with a
    random offset (the branch |disc| < FLT_EPSILON where B*B is small)"""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, len(radii), n)
    a = rng.integers(0, 3, n)
    b = (a + rng.integers(1, 3, n)) % 3
    s = F32(2.0) ** rng.integers(-2, 3, n).astype(F32)
    sign = np.where(rng.uniform(size=n) < 0.5, F32(-1.0), F32(1.0))
    r = np.zeros(n, S.RAY_DTYPE)
    idx = np.arange(n)
    org = centers[k].copy()
    org[idx, a] += radii[k]
    org[idx, b] -= sign * s
    r["org"] = org
    r["dir"][idx, b] = sign
    r["max_t"] = 1e30
    m = n // 2  # grazing, random
    e = _unit(rng, m)
    d = _unit(rng, m)
    perp = np.cross(d, e)
    perp /= np.linalg.norm(perp, axis=1)[:, None]
    r["org"][:m] = (centers[k[:m]] + perp * radii[k[:m], None] * rng.uniform(0.999, 1.001, (m, 1)) - d * s[:m, None]).astype(F32)
    r["dir"][:m] = d
    return r


def _on_surface(centers, radii, n, seed):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, len(radii), n)
    r = np.zeros(n, S.RAY_DTYPE)
    u = _unit(rng, n)
    r["org"] = (centers[k] + u * radii[k, None]).astype(F32)
    r["dir"] = np.where((rng.uniform(size=n) < 0.5)[:, None], -u, _unit(rng, n))
    r["max_t"] = 1e30
    return r


def _axis_zero(centers, radii, n, seed):
    """axis-parallel rays whose origin sits in a sphere box's plane, with +-0.0 in the other two components: the two
    vsafe_inverse conventions (copysign vs +inf for -0.0) pass different boxes"""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, len(radii), n)
    a = rng.integers(0, 3, n)
    r = np.zeros(n, S.RAY_DTYPE)
    idx = np.arange(n)
    org = centers[k] + (rng.uniform(-0.5, 0.5, (n, 3)) * radii[k, None]).astype(F32)
    face = rng.integers(0, 2, n)
    o2 = (a + 1) % 3
    org[idx, o2] = np.where(face == 0, centers[k, o2] - radii[k], centers[k, o2] + radii[k])  # in a box plane
    org[idx, a] = centers[k, a] - np.where(rng.uniform(size=n) < 0.5, 3, -3) * radii[k]
    r["org"] = org
    zeros = np.where(rng.uniform(size=(n, 3)) < 0.5, F32(-0.0), F32(0.0))
    r["dir"] = zeros
    r["dir"][idx, a] = np.where(org[idx, a] < centers[k, a], F32(1.0), F32(-1.0))
    r["max_t"] = 1e30
    return r


def _hostile_ranges(centers, radii, n, seed):
    """NaN min_t, NaN max_t, inverted ranges, zero ranges"""
    r = _random_rays(centers, radii, n, seed)
    c = np.arange(n) % 4
    r["min_t"][c == 0] = np.nan
    r["max_t"][c == 1] = np.nan
    r["min_t"][c == 2], r["max_t"][c == 2] = 5.0, 1.0
    r["max_t"][c == 3] = 0.0
    return r


def _max_t_exact(ref, centers, radii, n, seed):
    """max_t set to exactly the reference's t: `t < max_t` fails, not a hit"""
    rays = _random_rays(centers, radii, 4 * n, seed)
    h, m = ref.traverse(rays)
    k = np.flatnonzero(m)[:n]
    out = rays[k].copy()
    out["max_t"] = h["t"][k]
    return out


def _families(name, acc, centers, radii, n, seed):
    ref = orc.ReferenceSpheres.adopt(acc.GetNodes(), acc.GetIndices(), centers, radii)
    fam = {
        "random": _random_rays(centers, radii, n, seed),
        "inside_min_t": _inside_min_t(centers, radii, n // 2, seed + 1),
        "tangent": _tangent(centers, radii, n // 4, seed + 2),
        "on_surface": _on_surface(centers, radii, n // 4, seed + 3),
        "axis_zero": _axis_zero(centers, radii, n // 4, seed + 4),
        "ranges": _hostile_ranges(centers, radii, n // 8, seed + 5),
        "max_t_exact": _max_t_exact(ref, centers, radii, n // 8, seed + 6),
    }
    for s in (1e-3, 1e3):
        r = _random_rays(centers, radii, n // 4, seed + 7)
        r["dir"] *= F32(s)
        fam[f"dir_x{s:g}"] = r
    z = _random_rays(centers, radii, 64, seed + 8)
    z["dir"] = 0.0
    fam["zero_dir"] = z
    lo, hi = _box(centers, radii)
    fam["hostile"] = hostile_rays(lo, hi, n // 8, seed=seed + 9)
    return fam


REACH = {"one", "two", "three", "random7", "dup_one_leaf", "nested", "zero_radius", "random5000", "dup_spread"}


def _reach(fam_name, acc, centers, radii, rays, res, gh, gm, wh, scene):
    """what each family is there to test actually happens (checked with the oracle's records); the geometric families
    are checked on the scenes of ordinary radii and coordinates"""
    hit = gm.astype(bool)
    if scene not in REACH and fam_name in ("inside_min_t", "tangent", "on_surface"):
        return
    if fam_name == "inside_min_t":
        assert ((wh["t"] < rays["min_t"]) & hit).any(), "no hit below min_t"
    elif fam_name == "max_t_exact":
        assert not hit.any()
    elif fam_name == "tangent":
        k = np.flatnonzero(hit)
        assert (np.abs(_disc(rays[k], gh["prim_id"][k], centers, radii)) < EPS).any(), "tangent branch not reached"
    elif fam_name == "on_surface":
        near = gh["t"] <= F32(1e-4) * radii[np.minimum(gh["prim_id"], len(radii) - 1)]
        assert (hit & near).any() and (hit & ~near).any()
    elif fam_name == "ranges":
        assert not hit.any()
    elif fam_name == "zero_dir":
        assert res["relaxed"] == len(rays)


# ---------------------------------------------------------------------------------------------------- the matrix
SMALL = ["one", "two", "three", "random7", "dup_one_leaf", "nested", "zero_radius", "tiny_radius", "huge_radius"]


@pytest.mark.parametrize("name", SMALL + ["random5000", "dup_spread", "far_centres"])
def test_sphere_families_match_the_reference_on_the_device_tree(name):
    _need(True)
    _need(False)
    centers, radii, opts = _scene(name)
    acc = _build(centers, radii, opts)
    nodes = acc.GetNodes()
    if name in ("one", "two", "three", "dup_one_leaf"):
        assert len(nodes) == 1 and nodes["flag"][0] == 1, "the root must be a leaf"
    fam = _families(name, acc, centers, radii, 8000 if name in SMALL else 40000, seed=len(radii))
    differ = 0
    for fname, rays in fam.items():
        for cpp11 in (True, False):
            res, gh, gm, wh = _check(name, acc, centers, radii, rays, cpp11=cpp11)
            if cpp11:
                _reach(fname, acc, centers, radii, rays, res, gh, gm, wh, name)
                first = gm
            elif fname == "axis_zero":
                differ += int((gm != first).sum())
    assert differ > 0, "the two vsafe_inverse conventions never disagreed on the axis-parallel +-0.0 rays"
    ref = orc.ReferenceSpheres.adopt(nodes, acc.GetIndices(), centers, radii)
    all_rays = np.concatenate(list(fam.values()))
    _, wm = ref.traverse(all_rays)
    assert wm.sum() > 10
    if name == "dup_one_leaf":  # ties inside the one leaf resolve to the last copy in slot order, as the reference
        h, m = acc.Traverse(fam["random"])
        slot = np.argsort(acc.GetIndices())
        p = h["prim_id"][m.astype(bool)]
        assert len(p) > 100
        copies = (p // 4)[:, None] * 4 + np.arange(4)[None, :]
        assert (slot[p] == slot[copies].max(axis=1)).all(), "an in-leaf tie did not keep the last tested copy"
    if name == "huge_radius":
        assert _check(name, acc, centers, radii, fam["random"])[0]["relaxed"] > 0  # r*r = inf gives NaN t
    if name == "tiny_radius":
        assert np.any(radii * radii == 0) and np.any((radii * radii > 0) & (radii * radii < np.finfo(F32).tiny))
        h, m = acc.Traverse(fam["tangent"])
        p = h["prim_id"][m.astype(bool)]
        assert (radii[p] < 1e-19).any(), "no hit on a sphere of radius 1e-20"


@pytest.mark.parametrize("opt", [dict(min_leaf_primitives=1), dict(min_leaf_primitives=8),
                                 dict(min_leaf_primitives=200), dict(bin_size=3), dict(bin_size=256),
                                 dict(max_tree_depth=2), dict(max_tree_depth=500)])
def test_sphere_build_options(opt):
    _need(True)
    centers, radii, _ = _scene("random5000")
    acc = _build(centers, radii, api.BVHBuildOptions(**opt))
    st = acc.GetStatistics()
    nodes = acc.GetNodes()
    leaf_sizes = nodes["data"][nodes["flag"] == 1, 0]
    if "max_tree_depth" in opt:
        assert st["max_tree_depth"] <= opt["max_tree_depth"]
    if opt.get("max_tree_depth") == 2:
        assert leaf_sizes.max() > 200
    if opt.get("min_leaf_primitives") == 200:
        assert leaf_sizes.max() > 8
    if opt.get("min_leaf_primitives") == 1:
        assert leaf_sizes.min() == 1
    name = "opts " + ",".join(f"{k}={v}" for k, v in opt.items())
    for rays in (_random_rays(centers, radii, 30000, 1), _inside_min_t(centers, radii, 20000, 2)):
        for cpp11 in (True, False):
            _check(name, acc, centers, radii, rays, cpp11=cpp11, nan_t=None)


@pytest.mark.parametrize("stride", [16, 20])
def test_sphere_centre_strides(stride):
    """centres `stride` bytes apart with junk in the padding: the same tree and the same hits as stride 12"""
    centers, radii, _ = _scene("random5000")
    w = stride // 4
    padded = np.full((len(radii), w), np.nan, F32)
    padded[:, 3:] = np.float32(1e30) * np.arange(1, w - 2, dtype=F32)
    padded[:, 3] = -7.0
    padded[:, :3] = centers
    a12, aw = _build(centers, radii), _build(padded, radii, stride=stride)
    assert aw.GetNodes().tobytes() == a12.GetNodes().tobytes() and np.array_equal(aw.GetIndices(), a12.GetIndices())
    rays = _random_rays(centers, radii, 30000, 3)
    h12, m12 = a12.Traverse(rays)
    hw, mw = aw.Traverse(rays)
    assert np.array_equal(mw, m12) and hw.tobytes() == h12.tobytes() and mw.sum() > 1000
    if _have():
        _check(f"stride {stride}", aw, centers, radii, rays)


def test_sphere_prim_id_windows():
    _need(True)
    centers, radii, _ = _scene("random5000")
    acc = _build(centers, radii)
    rays = np.concatenate([_random_rays(centers, radii, 30000, 4), _inside_min_t(centers, radii, 10000, 5)])
    counts = {}
    for lo, hi in [(7, 7), (1234, 1235), (0, len(radii)), (0, 0x7FFFFFFF), (2500, 0xFFFFFFFF)]:
        topts = api.BVHTraceOptions(prim_ids_range=(lo, hi))
        res, gh, gm, _ = _check("prim_ids_range", acc, centers, radii, rays, topts=topts, nan_t=None)
        p = gh["prim_id"][gm.astype(bool)]
        assert ((p >= lo) & (p < hi)).all()
        counts[(lo, hi)] = res["hits"]
    assert counts[(7, 7)] == 0 and counts[(1234, 1235)] > 0 and counts[(0, len(radii))] == counts[(0, 0x7FFFFFFF)]


@pytest.mark.parametrize("n", [200000, 1000000])
def test_large_sphere_sets(n):
    """200 K and 1 M random spheres; the 1 M set with one batch of 2^20 + 777 rays (more than one host-path chunk)"""
    _need(True)
    centers, radii, _ = _scene(f"random{n}")
    acc = _build(centers, radii)
    m = (1 << 20) + 777 if n == 1000000 else 200000
    rays = np.concatenate([_random_rays(centers, radii, m - m // 4, 11), _inside_min_t(centers, radii, m // 4, 12)])
    res, gh, gm, _ = _check(f"random{n}", acc, centers, radii, rays, nan_t=None)
    assert res["hits"] > m // 4
    if n == 1000000:  # the rays of the second chunk are right too: same records as launched alone
        tail = rays[1 << 20:]
        th, tm = acc.Traverse(tail)
        assert np.array_equal(tm, gm[1 << 20:]) and th.tobytes() == gh[1 << 20:].tobytes()


def test_small_batches_from_threads_and_traverse_device():
    """the <= 64-ray zero-copy path from 8 host threads, batches of 1..65 rays, and TraverseDevice: the records of the
    classified large batch, bit for bit"""
    import torch

    centers, radii, _ = _scene("random5000")
    acc = _build(centers, radii)
    rays = np.concatenate([_random_rays(centers, radii, 3000, 21), _inside_min_t(centers, radii, 1000, 22)])
    if _have():
        _, gh, gm, _ = _check("paths", acc, centers, radii, rays)
    else:
        gh, gm = acc.Traverse(rays)
    assert gm.sum() > 1000
    errors = []

    def work(t):
        try:
            for k in range(1, 66):
                s = (t * 977 + k * 53) % (len(rays) - k)
                h, m = acc.Traverse(rays[s:s + k])
                if not (np.array_equal(m, gm[s:s + k]) and h.tobytes() == gh[s:s + k].tobytes()):
                    errors.append((t, k, s))
        except Exception as e:  # noqa: BLE001 -- reported below
            errors.append(repr(e))

    th = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors[:4]
    d_rays = torch.from_numpy(rays.view(np.uint8).copy()).cuda()
    d_hits = torch.zeros(len(rays) * 16, dtype=torch.uint8, device="cuda")
    d_mask = torch.zeros(len(rays), dtype=torch.uint8, device="cuda")
    acc.TraverseDevice(d_rays.data_ptr(), len(rays), d_hits.data_ptr(), d_mask.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(d_mask.cpu().numpy(), gm)
    assert d_hits.cpu().numpy().tobytes() == gh.tobytes()


def test_conformance_and_any_hit_flags_are_ignored_on_sphere_accels():
    centers, radii, _ = _scene("random5000")
    acc = _build(centers, radii)
    rays = np.concatenate([_random_rays(centers, radii, 20000, 31), _inside_min_t(centers, radii, 5000, 32)])
    for base in (0, api.TRAVERSE_CPP03_INVERSE):
        h0, m0 = acc.Traverse(rays, flags=base)
        for extra in (api.TRAVERSE_CONFORMANCE, api.TRAVERSE_ANY_HIT, api.TRAVERSE_CONFORMANCE | api.TRAVERSE_ANY_HIT):
            h, m = acc.Traverse(rays, flags=base | extra)
            assert np.array_equal(m, m0) and h.tobytes() == h0.tobytes(), (base, extra)


def test_counting_entry_points_refuse_non_triangle_accels():
    import torch

    centers, radii, _ = _scene("random7")
    sph = _build(centers, radii)
    box = api.BVHAccel()
    assert box.BuildBoxes(np.concatenate([centers - 1, centers + 1], axis=1))
    rays = _random_rays(centers, radii, 256, 41)
    d_rays = torch.from_numpy(rays.view(np.uint8).copy()).cuda()
    for acc in (sph, box):
        for flags in (api.TRAVERSE_FAST, api.TRAVERSE_CONFORMANCE):
            with pytest.raises(api.NanortB200Error, match="triangle accel"):
                acc.CountDevice(d_rays.data_ptr(), len(rays), flags=flags)
            with pytest.raises(api.NanortB200Error, match="triangle accel"):
                acc.LaneStatsDevice(d_rays.data_ptr(), len(rays), flags=flags)
    # a triangle accel still counts
    v, f = S.make_scene("sphere_grid", nx=2, nz=2)
    tri = api.BVHAccel()
    assert tri.Build(len(f), v, f)
    b, p = tri.CountDevice(d_rays.data_ptr(), len(rays), flags=api.TRAVERSE_CONFORMANCE)
    assert b > 0


def test_zz_report_class_counts():
    """prints the per-scene counts of classes (a) and (b) and of u / v straddles (pytest -s)"""
    for k, v in sorted(STATS.items()):
        print(f"{k:32s} hits {v['hits']:8d} same {v['same']:8d} (a) ties {v['ties']:5d} (b) below min_t "
              f"{v['below_min_t']:5d} u/v straddles {v['uv_straddles']:3d} relaxed rays {v['relaxed']:6d}")
