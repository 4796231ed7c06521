"""The bidirectional path tracer (include/nanort_b200_bdpt.h) where tests/test_gpu_bdpt.py does not reach:
  * calls cut into several waves of whole tiles (render and export, a partial last wave, partial edge tiles): a frame
    equals its shard, sample-range and repeated calls bit for bit, and every exported slot equals the same (pixel,
    sample) of single-wave shard exports;
  * a light table of thousands of faces over several sort tiles (the many-light panel scene of bdpt_helpers), and of
    one face: the reference's light picks, pdfPos and connections bit for bit;
  * max_bounces other than the reference's 10: device colours against the float64 connectPath of bdpt_model.py, which
    tests/test_bdpt_model.py checks against the reference's own; subpaths at 10 are prefixes of those at 64.
The wave count of a call is traverse_launches / (2 * max_bounces + 1): every wave runs max_bounces eye and light bounce
launches and one connection launch.  Each test asserts the wave count it relies on."""
import numpy as np
import pytest

import bdpt_helpers as H
import bdpt_model as M
from bdpt_helpers import MB, Setup, _bits, _compare_samples, frame_from_samples, slot_map

pytestmark = pytest.mark.gpu

SORT_TILE = 1024  # radix_sort.cuh: 256 threads x 4 keys


@pytest.fixture(scope="module")
def ref_mod():
    from oracle import bdpt_ref, orc

    if not bdpt_ref.available() or not orc.Reference.available(True):
        pytest.skip("oracle/_ref not built (no reference tree at build time)")
    return bdpt_ref


def _with_model(setup):
    setup.total = M.light_total_area(setup.v, setup.f, setup.mats, setup.ids)[0]
    setup.trace = H.reference_trace(setup.v, setup.f)
    return setup


@pytest.fixture(scope="module")
def cornell(ref_mod):
    from nanort_b200 import scenes as S

    v, f, mats, ids, _ = S.cornell_with_materials()
    return _with_model(Setup(ref_mod, v, f, mats, ids))


@pytest.fixture(scope="module")
def many(ref_mod):
    v, f, mats, ids, info = H.many_lights_scene()
    s = _with_model(Setup(ref_mod, v, f, mats, ids))
    s.info = info
    return s


def waves(res, B=MB):
    assert res.traverse_launches % (2 * B + 1) == 0, res.traverse_launches
    return res.traverse_launches // (2 * B + 1)


def tiles_per_wave(p, export):
    """run_bdpt's wave size: the tiles whose scratch fits 512 MB (PathState, both subpaths unless exported, lengths,
    colour, two queues, count, offset, emission, B(B+1)/2 24-byte records and scan scratch per slot)"""
    B = p.max_bounces
    per_slot = 64 + (0 if export else 2 * (B + 1) * 80 + 8 + 12) + 8 + 4 + 4 + 12 + B * (B + 1) // 2 * 24 + 8
    return max(1, (512 << 20) // (per_slot * p.tile_w * p.tile_h * p.spp))


def n_tiles(p):
    return -(-p.width // p.tile_w) * -(-p.height // p.tile_h)


def _differing_pixels(a, b):
    return int(np.count_nonzero(np.any(a.reshape(-1, 3) != b.reshape(-1, 3), axis=1)))


def _same_frame(flags, got, want):
    """bit for bit under the conformance walk; the production walk may pick either face at a shared edge (see
    test_gpu_bdpt.py), so at most 1 % of its pixels may differ"""
    got, want = got.cpu().numpy(), want.cpu().numpy()
    if flags:
        return np.array_equal(_bits(got), _bits(want))
    return _differing_pixels(got, want) <= 0.01 * (len(got) // 3)


# ---------------------------------------------------------------- waves
@pytest.mark.parametrize("flags", [1, 0], ids=["conformance", "production"])
def test_render_across_waves(cornell, flags):
    """330 x 250 at 4 spp: 21 x 32 = 672 tiles of 16 x 8, partial in both directions, over at least three waves with
    a partial last one; against three single-wave shards, a sample-range split and a second call"""
    import torch

    W, Ht, spp = 330, 250, 4
    p = cornell.params(W, Ht, spp, flags=flags)
    frame, r = cornell.render(p)
    nw = waves(r)
    tpw = tiles_per_wave(p, export=False)
    print(f"bdpt render {W}x{Ht}x{spp} ({'conformance' if flags else 'production'}): {n_tiles(p)} tiles, "
          f"{nw} waves of {tpw} tiles")
    assert nw >= 3 and nw == -(-n_tiles(p) // tpw) and n_tiles(p) % tpw != 0
    got = frame.cpu().numpy()
    assert np.all(np.isfinite(got)) and np.count_nonzero(got) > 0.2 * got.size  # rows past the box stay black
    # shards, each one wave; every pixel written by exactly one shard
    acc = torch.zeros_like(frame)
    totals = np.zeros(3, np.int64)
    for sh in range(3):
        one, rs = cornell.render(cornell.params(W, Ht, spp, shard=sh, n_shards=3, flags=flags))
        assert waves(rs) == 1
        assert not bool(((acc != 0) & (one != 0)).any())
        acc += one
        totals += (rs.eye_rays, rs.light_rays, rs.connection_rays)
    assert _same_frame(flags, acc, frame)
    if flags:
        assert tuple(totals) == (r.eye_rays, r.light_rays, r.connection_rays)
    # sample ranges into one frame
    acc = torch.zeros_like(frame)
    for s0, n in ((0, 1), (1, 3)):
        cornell.render(cornell.params(W, Ht, n, sample0=s0, spp_total=spp, flags=flags), acc)
    assert _same_frame(flags, acc, frame)
    again, r2 = cornell.render(p)
    assert _same_frame(flags, again, frame)
    if flags:
        assert (r2.eye_rays, r2.light_rays, r2.connection_rays) == (r.eye_rays, r.light_rays, r.connection_rays)


def _row_bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(len(a), -1)


def test_export_across_waves(cornell):
    """400 x 400 at 4 spp: 1250 tiles over at least two export waves.  Every slot equals, bit for bit, the same (pixel,
    sample) of single-wave shard exports; the reference's connectPath gives each wave's colours bit for bit; the last
    wave's whole samples are the reference's.  Slots run top row first, and the reference camera sees nothing in the
    bottom sixth of the frame (below the box's open front), so the frame is tall enough for the last wave to reach
    the box."""
    W, Ht, spp = 400, 400, 4
    p = cornell.params(W, Ht, spp)
    ex = cornell.export(p)
    nw = waves(ex["res"])
    tpw = tiles_per_wave(p, export=True)
    print(f"bdpt export {W}x{Ht}x{spp}: {n_tiles(p)} tiles, {nw} waves of {tpw} tiles")
    assert nw >= 2 and nw == -(-n_tiles(p) // tpw)
    pix, smp, valid = slot_map(p)
    n = len(pix)
    inv = np.full(W * Ht * spp, -1, np.int64)
    inv[pix[valid] * spp + smp[valid]] = np.nonzero(valid)[0]
    assert np.all(ex["ne"][~valid] == 0) and np.all(ex["ne"][valid] >= 1)
    for sh in range(nw):
        q = cornell.params(W, Ht, spp, shard=sh, n_shards=nw)
        part = cornell.export(q)
        assert waves(part["res"]) == 1
        qp, qs, qv = slot_map(q)
        idx = inv[qp[qv] * spp + qs[qv]]
        assert np.all(idx >= 0)
        assert np.array_equal(part["ne"][qv], ex["ne"][idx]) and np.array_equal(part["nl"][qv], ex["nl"][idx])
        assert np.array_equal(_bits(part["rgb"][qv]), _bits(ex["rgb"][idx]))
        for k in ("eye", "light"):
            assert np.array_equal(_row_bytes(part[k][qv]), _row_bytes(ex[k][idx])), (sh, k)
        del part
    # connectPath of the reference over each wave's subpaths
    cap = tpw * p.tile_w * p.tile_h * spp
    rng = np.random.default_rng(3)
    live = ex["ne"] > 1
    last_tile = np.arange(n - p.tile_w * p.tile_h * spp, n)
    last_tile = last_tile[valid[last_tile]]  # lens-only slots too: their colour is 0 in both
    checked = 0
    for w in range(nw):
        in_wave = np.nonzero(live[w * cap:min(n, (w + 1) * cap)])[0] + w * cap
        assert len(in_wave) >= 2000
        slots = rng.choice(in_wave, 2000, replace=False)
        if w == nw - 1:
            slots = np.union1d(slots, last_tile)
        bad = [int(i) for i in slots if not np.array_equal(
            _bits(cornell.ref.connect(ex["eye"][i, :ex["ne"][i]], ex["light"][i, :ex["nl"][i]])), _bits(ex["rgb"][i]))]
        assert not bad, (w, len(bad), bad[:5])
        checked += len(slots)
    # whole samples of the last wave
    last = np.arange((nw - 1) * cap, n)
    slots = rng.choice(last[valid[last]], 600, replace=False)
    same, diverged, value_bad = _compare_samples(cornell, p, ex, slots)
    print(f"bdpt export waves: {checked} slots connect bit for bit; last wave {same}/{same + len(diverged)} "
          f"samples structurally identical, {len(value_bad)} value mismatches")
    assert same + len(diverged) >= 500 and same >= 0.99 * (same + len(diverged)), diverged[:10]
    assert not value_bad, value_bad[:10]


# ---------------------------------------------------------------- the light table
def _light_faces(setup, ex):
    """the panel face of each live slot's light-origin vertex"""
    live = np.nonzero(ex["ne"] > 1)[0]
    assert np.all(ex["nl"][live] >= 1)
    faces = H.panel_faces_of(ex["light"][live, 0]["position"], setup.info)
    return live, faces


def test_many_lights_whole_samples(many):
    p = many.params(64, 64, 4)
    ex = many.export(p)
    assert waves(ex["res"]) == 1
    same, diverged, value_bad = _compare_samples(many, p, ex, np.arange(len(ex["ne"])))
    total = same + len(diverged)
    live, faces = _light_faces(many, ex)
    # pdfPos = 1 / totalArea, totalArea summed in face order
    assert np.array_equal(_bits(ex["light"][live, 0]["pdf_fwd"]), np.full(len(live), _bits(np.float32(1) / many.total)))
    # coverage of the table: picks in every sort tile and in a tie group across two sort tiles
    _, area, lit = M.light_total_area(many.v, many.f, many.mats, many.ids)
    order = np.lexsort((lit, area))
    rank = np.empty(len(order), np.int64)
    rank[order] = np.arange(len(order))
    assert np.all(faces >= 0), "a light origin off the panel"
    assert not np.any(faces == many.info["threshold"])
    pos = rank[np.searchsorted(lit, faces)]
    assert np.array_equal(lit[np.searchsorted(lit, faces)], faces), "a light origin on a face that is not a light"
    tiles = pos // SORT_TILE
    s = area[order].view(np.uint32)
    first = np.searchsorted(s, s[pos], side="left") // SORT_TILE
    last = (np.searchsorted(s, s[pos], side="right") - 1) // SORT_TILE
    n_tiles_table = -(-len(lit) // SORT_TILE)
    spanning = int(np.count_nonzero(first != last))
    # the max(Le) == kEps face ends eye subpaths without being a light
    ends = [(ex["eye"][i, ex["ne"][i] - 1]["prim_id"], ex["eye"][i, ex["ne"][i] - 1]["type"]) for i in live]
    thr = [t for f_, t in ends if f_ == many.info["threshold"]]
    print(f"bdpt many lights: {len(lit)} lights over {n_tiles_table} sort tiles; {len(live)} light picks in tiles "
          f"{np.bincount(tiles, minlength=n_tiles_table).tolist()}, {spanning} in tie groups across tiles; "
          f"{len(thr)} eye subpaths end on the max(Le) = kEps face; {same}/{total} samples structurally identical")
    assert n_tiles_table >= 3 and set(tiles.tolist()) == set(range(n_tiles_table))
    assert spanning > 0
    assert len(thr) > 0 and all(t == H.LIGHT for t in thr)
    assert same >= 0.99 * total, diverged[:10]
    assert not value_bad, value_bad[:10]


@pytest.mark.parametrize("flags", [1, 0], ids=["conformance", "production"])
def test_many_lights_connections_bit_for_bit(many, flags):
    p = many.params(64, 64, 4, flags=flags)
    ex = many.export(p)
    live = np.nonzero(ex["ne"] > 1)[0]
    assert len(live) > 1000
    bad = [int(i) for i in live if not np.array_equal(
        _bits(many.ref.connect(ex["eye"][i, :ex["ne"][i]], ex["light"][i, :ex["nl"][i]])), _bits(ex["rgb"][i]))]
    assert not bad, (len(bad), bad[:5])
    assert np.count_nonzero(ex["rgb"][live].sum(axis=1)) > 100


def test_single_light_face(ref_mod):
    """n_lights = 1: the Cornell box with one of its two light triangles dark"""
    from nanort_b200 import scenes as S

    v, f, mats, ids, emissive = S.cornell_with_materials()
    ids = ids.copy()
    ids[emissive[1]] = 0
    one = Setup(ref_mod, v, f, mats, ids)
    total, area, lit = M.light_total_area(one.v, one.f, one.mats, one.ids)
    assert list(lit) == [emissive[0]] and total == area[0]
    p = one.params(32, 32, 4)
    ex = one.export(p)
    live = np.nonzero(ex["ne"] > 1)[0]
    assert len(live) > 500
    l0 = ex["light"][live, 0]
    assert np.array_equal(_bits(l0["pdf_fwd"]), np.full(len(live), _bits(np.float32(1) / total)))
    tri = one.v[one.f[emissive[0]]].astype(np.float64)
    # barycentrics in the light's (x, z) plane
    d = l0["position"].astype(np.float64)[:, [0, 2]] - tri[0, [0, 2]]
    e1, e2 = tri[1, [0, 2]] - tri[0, [0, 2]], tri[2, [0, 2]] - tri[0, [0, 2]]
    det = e1[0] * e2[1] - e1[1] * e2[0]
    b1, b2 = (d[:, 0] * e2[1] - d[:, 1] * e2[0]) / det, (e1[0] * d[:, 1] - e1[1] * d[:, 0]) / det
    assert np.all((b1 >= -1e-6) & (b2 >= -1e-6) & (b1 + b2 <= 1 + 1e-6))
    bad = [int(i) for i in live if not np.array_equal(
        _bits(one.ref.connect(ex["eye"][i, :ex["ne"][i]], ex["light"][i, :ex["nl"][i]])), _bits(ex["rgb"][i]))]
    assert not bad, bad[:5]
    same, diverged, value_bad = _compare_samples(one, p, ex, np.arange(len(ex["ne"])))
    assert same >= 0.99 * (same + len(diverged)) and not value_bad, (diverged[:10], value_bad[:10])


# ---------------------------------------------------------------- max_bounces
def _pairs(ne, nl, B):
    """connectPath's (e, l) pairs of one sample within e + l - 2 <= B, before its delta and L == 0 skips"""
    return sum(max(0, min(int(nl), B + 2 - e)) for e in range(2, int(ne) + 1))


@pytest.mark.parametrize("B", [1, 2, 3, 5, 16, 64])
def test_colours_against_the_model(cornell, B):
    """All live slots of 32 x 32 x 2 for B <= 5; for B = 16 and 64, the 300 live slots of the longest subpaths.  The
    model's terms reach past e + l - 2 = 10 there, which a skip at the reference's constant would drop."""
    p = cornell.params(32, 32, 2, max_bounces=B)
    ex = cornell.export(p)
    assert waves(ex["res"], B) == 1
    live = np.nonzero(ex["ne"] > 1)[0]
    assert np.all(np.isfinite(ex["rgb"])) and np.all(ex["ne"] <= B + 1) and np.all(ex["nl"] <= B + 1)
    if B <= 5:
        slots = live
    else:
        slots = live[np.argsort(-(ex["ne"][live] + ex["nl"][live]), kind="stable")[:300]]
    assert len(slots) >= min(300, len(live)) and len(slots) >= 300
    bad, worst, beyond = [], 0.0, 0
    for i in slots:
        eye, light = ex["eye"][i, :ex["ne"][i]], ex["light"][i, :ex["nl"][i]]
        terms = M.connection_terms(eye, light, cornell.mats, cornell.total, B, cornell.trace)
        want = np.sum([t for _, _, t in terms], axis=0) if terms else np.zeros(3)
        mag = np.sum([np.abs(t) for _, _, t in terms], axis=0) if terms else np.zeros(3)
        err = np.abs(ex["rgb"][i].astype(np.float64) - want)
        if np.any(err > 1e-4 * mag + 1e-30):
            bad.append((int(i), ex["rgb"][i], want))
        worst = max(worst, float(np.max(err / np.maximum(mag, 1e-30))))
        beyond += any(e + l - 2 > MB and np.any(t != 0) for e, l, t in terms)
    cand = sum(_pairs(a, b, B) for a, b in zip(ex["ne"][live], ex["nl"][live]))
    print(f"bdpt max_bounces {B}: {len(slots)} slots against the model (worst {worst:.2e} sum|term|), longest eye / "
          f"light subpaths {ex['ne'].max()} / {ex['nl'].max()}, {ex['res'].connection_rays} connection rays of {cand} "
          f"pairs, {beyond} slots with terms past e + l - 2 = {MB}")
    assert not bad, (len(bad), bad[:5])
    assert 0 < ex["res"].connection_rays <= cand
    if B > MB:
        assert beyond > 0
    if B == 64:
        assert ex["ne"].max() > MB + 1 and ex["nl"].max() > MB + 1


def test_subpaths_are_prefixes_of_max_bounces_64(cornell):
    """Eye subpaths at 10 are prefixes of those at 64; so are light subpaths where the eye subpath ended below 11
    vertices (the light subpath then starts from the same generator state).  The last vertex's pdf_rev is written by the
    next bounce, which a cut subpath does not trace."""
    short = cornell.export(cornell.params(32, 32, 2, max_bounces=MB))
    full = cornell.export(cornell.params(32, 32, 2, max_bounces=64))
    assert np.all(short["ne"] == np.minimum(full["ne"], MB + 1))
    fields = H.FIELDS + ("type", "prim_id", "material")
    same_start = (short["ne"] > 1) & (short["ne"] < MB + 1)
    assert np.all(short["nl"][same_start] == np.minimum(full["nl"][same_start], MB + 1))
    n_light = 0
    for k, cnt, rows in (("eye", "ne", np.nonzero(short["ne"] > 0)[0]), ("light", "nl", np.nonzero(same_start)[0])):
        for i in rows:
            n = short[cnt][i]
            a, c = short[k][i, :n], full[k][i, :n]
            for key in fields:
                x, y = a[key], c[key]
                if key == "pdf_rev":
                    x, y = x[:-1], y[:-1]
                assert np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32)), (k, i, key)
        n_light += len(rows) if k == "light" else 0
    assert n_light > 500
    assert np.count_nonzero(full["nl"][same_start] > MB + 1) > 0  # light subpaths the cut did shorten


def test_render_max_bounces_64_across_waves(cornell):
    """160 x 96 x 1 at B = 64: 120 tiles over at least two waves against single-wave shards"""
    import torch

    B = 64
    p = cornell.params(160, 96, 1, max_bounces=B)
    frame, r = cornell.render(p)
    nw = waves(r, B)
    print(f"bdpt render 160x96x1 at max_bounces {B}: {n_tiles(p)} tiles, {nw} waves of {tiles_per_wave(p, False)}")
    assert nw >= 2 and nw == -(-n_tiles(p) // tiles_per_wave(p, export=False))
    got = frame.cpu().numpy()
    assert np.all(np.isfinite(got)) and np.count_nonzero(got) > 0
    acc = torch.zeros_like(frame)
    for sh in range(nw):
        one, rs = cornell.render(cornell.params(160, 96, 1, shard=sh, n_shards=nw, max_bounces=B))
        assert waves(rs, B) == 1
        acc += one
    assert np.array_equal(_bits(acc.cpu().numpy()), _bits(got))
    ex = cornell.export(p)
    assert np.array_equal(_bits(frame_from_samples(p, ex).reshape(-1)), _bits(got))
