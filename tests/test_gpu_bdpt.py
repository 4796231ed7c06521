"""The bidirectional path tracer (include/nanort_b200_bdpt.h) against the reference's own code
(oracle/_ref/libbdpt_ref.so = the unmodified examples/bidir_path_tracer/main.cc):
  * connections bit for bit: connectPath of the reference (its weightMIS and calcG over its own tree) over the
    device's exported subpaths equals the device's sample colour, under the conformance walk and the production walk;
  * whole samples: the reference's generator, subpaths and connections for the same pixel and seed give the device's
    subpaths and colours (structure for at least 99 % of the samples, values to a relative 1e-4 / 1e-3);
  * frames: the frame is the ordered sum of the exported sample colours, deterministic, and splits into sample ranges,
    shards and partial tiles equal one call bit for bit; eye subpaths at smaller max_bounces are prefixes;
  * the 1 M-triangle terrain under an area light; refusals launch nothing; two streams on one accel."""
import numpy as np
import pytest

import bdpt_model as M
from bdpt_helpers import FIELDS, MB, Setup, _bits, _compare_samples, frame_from_samples, slot_map

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref_mod():
    from oracle import bdpt_ref

    if not bdpt_ref.available():
        pytest.skip("oracle/_ref/libbdpt_ref.so not built (no reference tree at build time)")
    return bdpt_ref


@pytest.fixture(scope="module")
def cornell(ref_mod):
    from nanort_b200 import scenes as S

    v, f, mats, ids, _ = S.cornell_with_materials()
    return Setup(ref_mod, v, f, mats, ids)


@pytest.mark.parametrize("flags", [1, 0], ids=["conformance", "production"])
def test_connections_bit_for_bit(cornell, flags):
    """calcG reads only the nearest distance, and the production walk's distance to a given triangle is the
    reference's bit for bit (tests/test_gpu_traverse.py), so both walks must give the reference's colours exactly."""
    p = cornell.params(64, 64, 4, flags=flags)
    ex = cornell.export(p)
    live = np.nonzero(ex["ne"] > 1)[0]
    assert len(live) > 1000
    bad = []
    for i in live:
        want = cornell.ref.connect(ex["eye"][i, :ex["ne"][i]], ex["light"][i, :ex["nl"][i]])
        if not np.array_equal(_bits(want), _bits(ex["rgb"][i])):
            bad.append((int(i), want, ex["rgb"][i]))
    assert not bad, (len(bad), bad[:5])
    assert np.count_nonzero(ex["rgb"][live].sum(axis=1)) > 100  # the frame is not black


def test_whole_samples_against_the_reference(cornell):
    """Structure identical for >= 99 % of the samples.  The expected divergence is directionCosTheta's cosf / sinf
    (the device rounds cos / sin evaluated in double; glibc's are within an ulp of that), which moves later vertices by
    an ulp or two of the scene's coordinates and, rarely, to another face.  Measured on an H100 (80GB HBM3): 16337 of
    16384 samples (99.71 %) structurally identical."""
    p = cornell.params(64, 64, 4)
    ex = cornell.export(p)
    slots = np.nonzero(ex["ne"] >= 0)[0]
    same, diverged, value_bad = _compare_samples(cornell, p, ex, slots)
    total = same + len(diverged)
    print(f"bdpt whole samples: {same}/{total} structurally identical ({100.0 * same / total:.3f} %), "
          f"{len(value_bad)} value mismatches")
    assert same >= 0.99 * total, (same, total, diverged[:10])
    assert not value_bad, value_bad[:10]


def test_frame_is_the_ordered_sum_of_the_samples(cornell):
    """Under the conformance walk, bit for bit and from call to call.  The production walk may return another of the
    faces a ray meets at the same distance (an edge shared by two faces), as nrt_traverse does, so its samples can
    differ between two calls there: its frame is held to the exported sum on all but a few pixels."""
    import torch

    for flags in (1, 0):
        p = cornell.params(64, 64, 4, flags=flags)
        ex = cornell.export(p)
        frame, r = cornell.render(p)
        got = frame.cpu().numpy().reshape(-1, 3)
        assert np.all(np.isfinite(got)) and got.sum() > 0
        want = frame_from_samples(p, ex)
        if flags:
            assert np.array_equal(_bits(got), _bits(want))
            again, _ = cornell.render(p)
            assert torch.equal(frame, again)
        else:
            assert np.count_nonzero(np.any(got != want, axis=1)) <= 0.01 * len(got)
        # ray counts: every subpath ray is one Traverse; a subpath of n vertices traced n - 1 or n rays
        pix, smp, valid = slot_map(p)
        ne, nl = ex["ne"][valid], ex["nl"][valid]
        assert np.sum(ne - 1) <= ex["res"].eye_rays <= np.sum(ne)
        live = ne > 1
        assert np.sum(nl[live] - 1) <= ex["res"].light_rays <= np.sum(nl[live])
        cand = sum(max(0, min(int(a) - 1, MB)) * int(b) for a, b in zip(ne[live], nl[live]))
        assert 0 < ex["res"].connection_rays <= cand
        if flags:
            er = ex["res"]
            assert (er.eye_rays, er.light_rays, er.connection_rays) == (r.eye_rays, r.light_rays, r.connection_rays)


def test_frame_splits_are_bit_identical(cornell):
    import torch

    W, H, spp = 61, 45, 4  # partial tiles
    whole, _ = cornell.render(cornell.params(W, H, spp, tile=(16, 8)))
    want = whole.cpu().numpy()
    # sample ranges
    acc = torch.zeros_like(whole)
    for s0, n in ((0, 1), (1, 2), (3, 1)):
        cornell.render(cornell.params(W, H, n, sample0=s0, spp_total=spp), acc)
    assert np.array_equal(_bits(acc.cpu().numpy()), _bits(want))
    # shards: every pixel written by exactly one shard
    acc = torch.zeros_like(whole)
    for sh in range(3):
        one, _ = cornell.render(cornell.params(W, H, spp, shard=sh, n_shards=3))
        o = one.cpu().numpy()
        assert not np.any((acc.cpu().numpy() != 0) & (o != 0))
        acc += one
    assert np.array_equal(_bits(acc.cpu().numpy()), _bits(want))
    # other tiles
    for tile in ((8, 4), (64, 64), (24, 12)):
        other, _ = cornell.render(cornell.params(W, H, spp, tile=tile))
        assert np.array_equal(_bits(other.cpu().numpy()), _bits(want)), tile


def test_eye_subpaths_are_prefixes_across_max_bounces(cornell):
    full = cornell.export(cornell.params(32, 32, 2))
    for b in range(1, MB):
        ex = cornell.export(cornell.params(32, 32, 2, max_bounces=b))
        assert np.all(ex["ne"] <= b + 1) and np.all(ex["ne"] <= full["ne"])
        assert np.all((ex["ne"] == b + 1) | (ex["ne"] == full["ne"]))
        for i in np.nonzero(ex["ne"] > 0)[0]:
            n = ex["ne"][i]
            a, c = ex["eye"][i, :n], full["eye"][i, :n]
            for k in FIELDS + ("type", "prim_id", "material"):
                x, y = a[k], c[k]
                if k == "pdf_rev":  # the last vertex's pdfRev is written by the next bounce
                    x, y = x[:-1], y[:-1]
                assert np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32)), (b, i, k)
        assert all(np.all(np.isfinite(ex[k]["position"][ex["ne" if k == "eye" else "nl"][:, None] >
                                                      np.arange(b + 1)[None, :]])) for k in ("eye", "light"))


@pytest.fixture(scope="module")
def terrain(ref_mod):
    from nanort_b200 import scenes as S

    v, f = S.make_scene("terrain")
    v, f, l0, ln = S.with_area_light(v, f, (0.0, 3.0, 0.0), 1.0, 1.0)
    mats = np.concatenate([S.material(diffuse=(0.7, 0.6, 0.5)), S.material(emission=(20.0, 20.0, 20.0))])
    ids = np.zeros(len(f), np.uint32)
    ids[l0:l0 + ln] = 1
    return Setup(ref_mod, v, f, mats, ids)


def test_terrain_samples_against_the_reference(terrain):
    p = terrain.params(128, 128, 1)  # the reference camera sees the terrain nearly edge-on: ~7 % of the pixels
    ex = terrain.export(p)
    live = np.nonzero(ex["ne"] > 1)[0]
    assert len(live) > 300
    slots = np.random.default_rng(11).choice(live, 300, replace=False)
    same, diverged, value_bad = _compare_samples(terrain, p, ex, slots)
    print(f"bdpt terrain samples: {same}/{same + len(diverged)} structurally identical")
    assert same >= 0.99 * (same + len(diverged)), diverged[:10]
    assert not value_bad, value_bad[:10]
    for flags in (1, 0):  # the production walk: see test_frame_is_the_ordered_sum_of_the_samples
        q = terrain.params(64, 64, 1, flags=flags)
        e = terrain.export(q)
        frame, _ = terrain.render(q)
        got = frame.cpu().numpy().reshape(-1, 3)
        assert np.all(np.isfinite(got)) and got.sum() > 0
        want = frame_from_samples(q, e)
        if flags:
            assert np.array_equal(_bits(got), _bits(want))
        else:
            assert np.count_nonzero(np.any(got != want, axis=1)) <= 0.01 * len(got)


def test_refusals_launch_nothing(cornell):
    import torch

    from nanort_b200 import api

    def refused(p, accel=None):
        acc = torch.full((3 * p.width * p.height,), 7.0, device="cuda:0")
        with pytest.raises(api.NanortB200Error):
            cornell.render(p, acc, accel=accel)
        torch.cuda.synchronize()
        assert bool((acc == 7.0).all())

    base = lambda **kw: cornell.params(16, 16, 1, **kw)
    for field in ("d_materials", "d_material_ids", "d_facevarying_normals"):
        p = base()
        setattr(p, field, None)
        refused(p)
    p = base()
    p.n_materials = 0
    refused(p)
    refused(base(flags=api.TRAVERSE_ANY_HIT))
    refused(base(flags=1 | api.TRAVERSE_CPP03_INVERSE))
    refused(base(sample0=1, spp_total=1))
    refused(base(tile=(12, 8)))
    refused(base(tile=(16, 6)))
    refused(base(max_bounces=0))
    refused(base(shard=2, n_shards=2))
    # a material id past n_materials, and a mesh without an emissive face (both read back at pass start)
    p = base()
    p.n_materials = 5  # the light (5) and the floor (6) now lie past the table
    refused(p)
    dark = torch.from_numpy(np.where(cornell.ids == 5, 0, cornell.ids).astype(np.int32)).to("cuda:0")
    p = base()
    p.d_material_ids = dark.data_ptr()
    refused(p)
    with pytest.raises(api.NanortB200Error):
        cornell.conf.ExportBDPT(base(), 0, 0, 0, 0, 0)
    with pytest.raises(api.NanortB200Error):
        cornell.conf.RenderBDPT(base(), 0)


def test_two_streams_on_one_accel(cornell):
    import torch

    pa, pb = cornell.params(48, 40, 2), cornell.params(48, 40, 2, sample0=2, spp_total=4)
    want_a, _ = cornell.render(pa)
    want_b, _ = cornell.render(pb)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a = torch.zeros_like(want_a)
    b = torch.zeros_like(want_b)
    torch.cuda.synchronize()
    cornell.conf.RenderBDPT(pa, a.data_ptr(), s1.cuda_stream)
    cornell.conf.RenderBDPT(pb, b.data_ptr(), s2.cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(a, want_a) and torch.equal(b, want_b)
