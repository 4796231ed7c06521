"""The float64 connectPath of tests/bdpt_model.py against the reference's own (oracle/_ref/libbdpt_ref.so, the unmodified
examples/bidir_path_tracer/main.cc) at its uMaxBounces = 10, on whole reference samples of the Cornell box and of the
many-light panel scene.  No GPU: this validates the model before tests/test_gpu_bdpt_slots.py judges the device with
it at other max_bounces."""
import numpy as np
import pytest

import bdpt_helpers as H
import bdpt_model as M

W = H_IMG = 64
M_B = 10  # the reference's uMaxBounces


@pytest.fixture(scope="module")
def ref_mod():
    from oracle import bdpt_ref, orc

    if not bdpt_ref.available() or not orc.Reference.available(True):
        pytest.skip("oracle/_ref not built (no reference tree at build time)")
    return bdpt_ref


def _scene(ref_mod, v, f, mats, ids):
    from nanort_b200 import api

    v, f = np.ascontiguousarray(v, np.float32), np.ascontiguousarray(f, np.uint32)
    mats = np.ascontiguousarray(np.asarray(mats).view(np.float32).reshape(-1, 16))
    ids = np.ascontiguousarray(ids, np.uint32)
    ref = ref_mod.BdptReference(v, f, ids, mats, M.flat_normals(v, f), api.BDPT_VERTEX_DTYPE)
    return ref, mats, M.light_total_area(v, f, mats, ids), H.reference_trace(v, f)


def _reference_samples(ref, n):
    """n samples of the reference with a vertex beyond the lens, from pixels all over a 64 x 64 frame at spp_total 4"""
    out = []
    for k in np.random.default_rng(5).permutation(W * H_IMG * 4):
        x, y, i = (k // 4) % W, (k // 4) // W, k % 4
        eye, light, _ = ref.sample(x, y, W, H_IMG, M.seed(x, y, W, 4, i))
        if len(eye) > 1:
            out.append((eye, light))
        if len(out) == n:
            break
    assert len(out) == n
    return out


def _check(ref_mod, scene, n=2000):
    ref, mats, (total, _, _), trace = scene
    samples = _reference_samples(ref, n)
    worst, terms, lit = 0.0, 0, 0
    for eye, light in samples:
        assert np.array_equal(H._bits(light[0]["pdf_fwd"]), H._bits(np.float32(1.0) / total))  # pdfPos = 1 / totalArea
        want = ref.connect(eye, light).astype(np.float64)
        got, mag = M.connect_path(eye, light, mats, total, M_B, trace)
        err = np.abs(got - want)
        assert np.all(err <= 1e-4 * mag + 1e-30), (eye, light, got, want, mag)
        worst = max(worst, float(np.max(err / np.maximum(mag, 1e-30))))
        terms += len(M.connection_terms(eye, light, mats, total, M_B, trace))
        lit += bool(np.any(want > 0))
    print(f"bdpt model: {n} samples, {terms} terms, {lit} non-black, worst |model - reference| = {worst:.2e} sum|term|")
    assert terms > 2 * n and lit > n // 5
    return samples


def test_model_matches_reference_connect_cornell(ref_mod):
    from nanort_b200 import scenes as S

    v, f, mats, ids, _ = S.cornell_with_materials()
    _check(ref_mod, _scene(ref_mod, v, f, mats, ids))


def test_model_matches_reference_connect_many_lights(ref_mod):
    v, f, mats, ids, info = H.many_lights_scene()
    scene = _scene(ref_mod, v, f, mats, ids)
    samples = _check(ref_mod, scene)
    # the reference's light origins lie on panel lights, never on the max(Le) == kEps wall
    faces = H.panel_faces_of(np.array([light[0]["position"] for _, light in samples]), info)
    assert np.all(faces >= 0)
    assert np.all(scene[2][2][np.searchsorted(scene[2][2], faces)] == faces)  # every picked face is in the table


def test_many_light_scene_shape():
    """The panel scene exercises what the light table can get wrong: more than two sort tiles of lights, a tie group
    across tile boundaries, distinct jittered areas, a face-order total that a sorted-order sum would not give, and the
    kEps threshold on both sides."""
    v, f, mats, ids, info = H.many_lights_scene()
    mats16 = np.asarray(mats).view(np.float32).reshape(-1, 16)
    total, area, lit = M.light_total_area(v, f, mats16, ids)
    assert len(lit) > 2048
    assert info["threshold"] not in lit and info["just"] in lit and info["blue"] in lit
    assert np.max(mats16[ids[info["threshold"]], 9:12]) == np.float32(0.001)
    order = np.lexsort((lit, area))  # std::sort's (area, face)
    s = area[order]
    tile = np.arange(len(s)) // 1024
    groups = np.split(np.arange(len(s)), np.nonzero(np.diff(s.view(np.uint32)))[0] + 1)
    assert any(tile[g[0]] != tile[g[-1]] for g in groups)  # a tie group spans sort tiles
    assert len(groups) >= 5  # jittered faces with distinct areas
    sorted_total = np.float32(0.0)
    for x in s:
        sorted_total = np.float32(sorted_total + x)
    assert sorted_total != total
    cross = np.cross(v[f[info["base"]:, 2]] - v[f[info["base"]:, 0]], v[f[info["base"]:, 1]] - v[f[info["base"]:, 0]])
    assert np.all(cross != 0)
