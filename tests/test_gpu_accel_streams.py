"""Many launches and passes of ONE accel in flight at once, on many streams, against the oracle and against serial runs.

nrt_traverse_device, nrt_traverse_f64_device and the AO / path / sharded passes are asynchronous with no limit on how
many calls a renderer keeps in flight.  Their persistent kernels draw rays from a device cursor, and the passes keep
queues and counters in per-accel (or per-communicator) scratch.  Every test here holds its launches back behind one
gate -- a stream that spins, then records the event every worker stream waits on -- so that all of them are enqueued
before any starts, and sizes them so that all can be resident together: a launch that shared a cursor or scratch
with another would process only part of its rays, or add another launch's work to its own.

Outputs are prefilled with 0xFF bytes: a ray no launch processed leaves a mask byte outside {0, 1}, which every test
asserts first."""
import numpy as np
import pytest

from helpers import assert_parity, compare_hits

pytestmark = pytest.mark.gpu

GATE_CYCLES = 100_000_000  # ~60 ms at H100 clocks: far longer than enqueueing everything behind the gate takes
N_RAYS = 2048              # 16 CTAs of 128 threads: 48 such launches stay under 132 SMs x 10 CTAs


def _gated_streams(torch, k):
    """k distinct worker streams, all waiting on one gate that has not opened yet.  torch hands streams out round-robin
    from a pool of 32 per priority, so the 33rd stream of one priority would be the first again and its launches would
    run after the first one's instead of beside them: the gate and 31 workers come from the default pool, the other
    workers from the high-priority one."""
    gate = torch.cuda.Stream()
    streams = [torch.cuda.Stream(priority=0 if i < 31 else -1) for i in range(k)]
    assert len({s.cuda_stream for s in streams} - {gate.cuda_stream}) == k
    with torch.cuda.stream(gate):
        torch.cuda._sleep(GATE_CYCLES)
    ev = torch.cuda.Event()
    ev.record(gate)
    for s in streams:
        s.wait_event(ev)
    return streams


def _filled(torch, *shape):
    return torch.full(shape, 0xFF, dtype=torch.uint8, device="cuda")


def _assert_no_holes(mask, what):
    bad = int(((mask != 0) & (mask != 1)).sum())
    assert bad == 0, f"{what}: {bad} rays were never written"


# ------------------------------------------------------------------ triangle accels: the ray-cursor ring
def _launch_kinds(api):
    """(flags, trace option set) of the launches, in turn: the default fast launch, any-hit, 32-byte records, the
    reference-order walk (no cursor), and two trace option sets"""
    from test_gpu_trav_variants import TRACE_OPTION_SETS

    return [(0, None), (api.TRAVERSE_ANY_HIT, None), (api.TRAVERSE_RAY32, None), (api.TRAVERSE_CONFORMANCE, None),
            (0, TRACE_OPTION_SETS[1]), (0, TRACE_OPTION_SETS[4])]


class _Launch:
    """one TraverseDevice call with its own rays and prefilled outputs"""

    def __init__(self, torch, rays, flags, tkw):
        from nanort_b200 import api

        self.rays, self.flags, self.tkw = rays, flags, tkw
        raw = np.ascontiguousarray(rays).view(np.uint8).reshape(-1, 36)
        if flags & api.TRAVERSE_RAY32:  # 16-byte aligned 32-byte records (torch allocations are 512-byte aligned)
            raw = np.ascontiguousarray(raw[:, :32])
        self.d_rays = torch.from_numpy(raw.copy()).cuda()
        self.d_hits = _filled(torch, len(rays), 16)
        self.d_mask = _filled(torch, len(rays))

    def enqueue(self, acc, stream):
        from nanort_b200 import api

        acc.TraverseDevice(self.d_rays.data_ptr(), len(self.rays), self.d_hits.data_ptr(), self.d_mask.data_ptr(),
                           options=None if self.tkw is None else api.BVHTraceOptions(**self.tkw), flags=self.flags,
                           stream=stream.cuda_stream)

    def check(self, port, acc, nodes, idx, v, f, what):
        """against the oracle walking the accel's own tree"""
        from nanort_b200 import api, scenes as S
        from oracle import orc

        m = self.d_mask.cpu().numpy()
        _assert_no_holes(m, what)
        h = self.d_hits.cpu().numpy().reshape(-1).view(S.HIT_DTYPE)
        topts = None if self.tkw is None else orc.trace_options(**self.tkw)
        want_h, want_m = port.traverse(nodes, idx, v, f, self.rays, topts=topts, threads=8)
        hit = want_m.astype(bool)
        if self.flags & api.TRAVERSE_CONFORMANCE:  # the reference's visiting order: bit-exact, ties included
            assert np.array_equal(m, want_m), what
            assert np.array_equal(h[hit].view(np.uint32), want_h[hit].view(np.uint32)), what
        elif self.flags & api.TRAVERSE_ANY_HIT:
            # the closest-hit mask; every record that is not the closest hit is a genuine hit of its own triangle
            assert np.array_equal(m, want_m), what
            assert np.all(h["prim_id"][~hit] == 0xFFFFFFFF), what
            assert np.all(h["t"][hit] >= want_h["t"][hit]) and np.all(h["t"][hit] < self.rays["max_t"][hit]), what
            other = np.flatnonzero(hit & (h["prim_id"] != want_h["prim_id"]))
            for i in other[:: max(1, len(other) // 32)]:
                o = api.BVHTraceOptions(prim_ids_range=(int(h["prim_id"][i]), int(h["prim_id"][i]) + 1))
                h1, m1 = acc.Traverse(self.rays[i:i + 1], options=o)
                assert m1[0] == 1 and h1.tobytes() == h[i:i + 1].tobytes(), (what, i)
        else:  # exact t / u / v; a different triangle only at exactly the same t
            assert_parity(compare_hits(port, v, f, self.rays, h, m, want_h, want_m, topts=topts))
        return int(hit.sum())


def _many_launches(torch, port, acc, v, f, k, seed0):
    """k gated TraverseDevice launches on k streams, each with its own rays and one of the launch kinds in turn.  The
    first k - 32 launches, whose cursors the last k - 32 come round to, carry three times the rays (48 CTAs), so that
    they are still running when the later launches start: 16 x 48 + 32 x 16 CTAs are still resident together."""
    from nanort_b200 import api, scenes as S

    lo, hi = v.min(axis=0), v.max(axis=0)
    kinds = _launch_kinds(api)
    launches = [_Launch(torch, S.incoherent_rays(lo, hi, N_RAYS * (3 if i < k - 32 else 1), seed=seed0 + i),
                        *kinds[i % len(kinds)]) for i in range(k)]
    torch.cuda.synchronize()
    for ln, s in zip(launches, _gated_streams(torch, k)):
        ln.enqueue(acc, s)
    return launches


def _check_all(port, acc, launches, v, f):
    nodes, idx = acc.GetNodes(), acc.GetIndices()
    hits = [ln.check(port, acc, nodes, idx, v, f, f"launch {i} (flags {ln.flags:#x}, options {ln.tkw})")
            for i, ln in enumerate(launches)]
    assert min(hits) >= 16 and sum(hits) > len(launches) * N_RAYS // 5, hits  # every launch has hits to lose


@pytest.mark.parametrize("tree", ["production", "reference"])
def test_more_traversal_launches_in_flight_than_the_cursor_ring_has_slots(port, tree):
    """48 launches of one accel on 48 streams, more than the 32 cursors of the accel's ring: every launch's records
    are the oracle's.  The production-built sphere grid walks the 64-entry stack; the reference-built terrain (depth
    > 64) the 512-entry one."""
    import torch
    from nanort_b200 import api, scenes as S
    from test_gpu_trav_variants import _deep

    if tree == "production":
        v, f = S.make_scene("sphere_grid", nx=4, nz=4)
        acc = api.BVHAccel()
        assert acc.Build(len(f), v, f)
        assert not _deep(acc)
    else:
        v, f = S.make_scene("terrain", n=128)
        acc = api.BVHAccel()
        assert acc.Build(len(f), v, f, flags=api.BUILD_REFERENCE_TREE)
        assert _deep(acc), acc.GetStatistics()["max_tree_depth"]
    launches = _many_launches(torch, port, acc, v, f, 48, seed0=1000)
    torch.cuda.synchronize()
    _check_all(port, acc, launches, v, f)


# ------------------------------------------------------------------ double-precision accels
def test_more_f64_launches_in_flight_than_the_cursor_ring_has_slots():
    """12 launches of one BVHAccelF64 on 12 streams, more than its 8 cursors: each equals the reference-order walk of
    the same rays (pinned to the reference's BVHAccel<double> by test_gpu_f64.py)."""
    import torch
    from nanort_b200 import api
    from test_gpu_f64 import _assert_fast_equals_conformance, _rays64, _scene64

    v64, f = _scene64(seed=21)
    acc = api.BVHAccelF64()
    assert acc.Build(len(f), v64, f)
    rays = [_rays64(v64, N_RAYS, seed=300 + i) for i in range(12)]
    acc.Traverse(rays[0][:64])  # derives the fast layout before the gate
    d_rays = [torch.from_numpy(np.ascontiguousarray(r).view(np.uint8).copy()).cuda() for r in rays]
    outs = [(_filled(torch, N_RAYS, 32), _filled(torch, N_RAYS)) for _ in rays]
    torch.cuda.synchronize()
    for r, (h, m), s in zip(d_rays, outs, _gated_streams(torch, len(rays))):
        acc.TraverseDevice(r.data_ptr(), N_RAYS, h.data_ptr(), m.data_ptr(), stream=s.cuda_stream)
    torch.cuda.synchronize()
    for i, (r, (h, m)) in enumerate(zip(rays, outs)):
        fm = m.cpu().numpy()
        _assert_no_holes(fm, f"launch {i}")
        fh = h.cpu().numpy().reshape(-1).view(api.HIT64_DTYPE)
        ch, cm = acc.Traverse(r, flags=api.TRAVERSE_CONFORMANCE)
        assert cm.sum() > N_RAYS // 20
        _assert_fast_equals_conformance(r, fh, fm, ch, cm)


# ------------------------------------------------------------------ passes
def _ao_params(api, S, scene, W, H, spp, cam=None):
    p = api.AoParams()
    cam = S.scene_camera(scene, W, H) if cam is None else cam
    for i in range(12):
        p.cam[i] = float(cam[i])
    p.width, p.height, p.spp, p.sample0, p.seed = W, H, spp, 0, 1
    p.tile_w, p.tile_h, p.shard, p.n_shards = 64, 8, 0, 1
    p.ray_min_t, p.ray_max_t, p.ao_min_t, p.ao_max_t = 1e-3, 1e30, 1e-3, 2.0
    return p


def _serial_ao(torch, acc, p):
    accum = torch.zeros(p.width * p.height, dtype=torch.float32, device="cuda")
    r = acc.RenderAO(p, accum.data_ptr())
    torch.cuda.synchronize()
    return accum, (r.primary_rays, r.ao_rays, r.ao_hits)


def test_ao_pass_next_to_traversals_that_wrap_the_cursor_ring(port):
    """An asynchronous AO pass (camera launch + AO launch, two cursors of the ring) and 40 traversal launches enqueued
    after it on 40 other streams, enough to come round to the pass's cursors: the frame equals the serial frame bit for
    bit, its visibility sum is the serial pass's primary minus AO hits, and every traversal's records are the oracle's."""
    import torch
    from nanort_b200 import api, scenes as S

    v, f = S.make_scene("sphere_grid", nx=4, nz=4)
    acc = api.BVHAccel()
    assert acc.Build(len(f), v, f)
    p = _ao_params(api, S, "sphere_grid", 64, 32, 1)  # 2048 camera rays: 16 CTAs per launch
    want, counts = _serial_ao(torch, acc, p)
    assert counts[0] == 64 * 32 and counts[1] > 0

    lo, hi = v.min(axis=0), v.max(axis=0)
    kinds = _launch_kinds(api)
    launches = [_Launch(torch, S.incoherent_rays(lo, hi, N_RAYS, seed=2000 + i), *kinds[i % len(kinds)])
                for i in range(40)]
    accum = torch.zeros(64 * 32, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    streams = _gated_streams(torch, 41)
    acc.RenderAO(p, accum.data_ptr(), stream=streams[0].cuda_stream, want_result=False)
    for ln, s in zip(launches, streams[1:]):
        ln.enqueue(acc, s)
    torch.cuda.synchronize()
    assert torch.equal(accum, want), int((accum != want).sum().item())
    assert float(accum.sum().item()) == float(counts[0] - counts[2])
    again, counts2 = _serial_ao(torch, acc, p)
    assert counts2 == counts and torch.equal(again, want)
    _check_all(port, acc, launches, v, f)


def _rel_pixels(got, want):
    """pixels whose radiance differs by more than 1e-5 relative (floor 1)"""
    g, w = got.cpu().numpy().astype(np.float64).reshape(-1, 3), want.cpu().numpy().astype(np.float64).reshape(-1, 3)
    rel = np.max(np.abs(g - w) / np.maximum(np.abs(w), 1.0), axis=1)
    return int(np.count_nonzero(rel > 1e-5))


def _path_scene(torch):
    from nanort_b200 import api, scenes as S
    from test_gpu_path import _setup

    v, f, mats, ids, emissive = S.cornell_with_materials()
    W, H = 64, 48
    acc, p, cam, keep = _setup(torch, api, S, v, f, mats, ids, emissive, None, W, H, 4, 6, 5)
    return acc, p, keep, W, H


def test_path_passes_and_an_ao_pass_on_three_streams_equal_serial_runs():
    """Two asynchronous path passes with different seeds and an AO pass, all on one accel and three streams: each path
    frame equals its serial frame up to the exact-distance ties of test_gpu_path (at most 4 pixels), the AO frame bit
    for bit."""
    import torch
    from nanort_b200 import api, scenes as S

    acc, p1, keep, W, H = _path_scene(torch)
    p2 = api.PathParams.from_buffer_copy(p1)
    p2.seed = 11
    pa = _ao_params(api, S, "cornell", W, H, 2)
    pa.ao_max_t = 5.0

    def path_frame():
        return torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")

    serial = []
    for p in (p1, p2):
        a = path_frame()
        r = acc.RenderPath(p, a.data_ptr())
        assert r.camera_rays == W * H * 4
        serial.append(a)
    want_ao, _ = _serial_ao(torch, acc, pa)
    assert not torch.equal(serial[0], serial[1])

    got = [path_frame(), path_frame()]
    got_ao = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    s1, s2, s3 = _gated_streams(torch, 3)
    acc.RenderPath(p1, got[0].data_ptr(), stream=s1.cuda_stream, want_result=False)
    acc.RenderPath(p2, got[1].data_ptr(), stream=s2.cuda_stream, want_result=False)
    acc.RenderAO(pa, got_ao.data_ptr(), stream=s3.cuda_stream, want_result=False)
    torch.cuda.synchronize()
    for k in range(2):
        assert _rel_pixels(got[k], serial[k]) <= 4, k
    assert torch.equal(got_ao, want_ao), int((got_ao != want_ao).sum().item())


def test_path_bounce_right_after_an_asynchronous_path_pass_equals_a_serial_bounce():
    """nrt_path_bounce_device on one stream while a path pass enqueued just before it on another stream has not
    finished: the same counts, the same set of continuing path ids and the same continuation rays (matched by path
    id, 1e-5) as the same bounce run alone."""
    import torch
    from nanort_b200 import dist as nd, scenes as S
    from test_gpu_path import TILE, _rel

    acc, p, keep, W, H = _path_scene(torch)
    spp = p.spp
    pix_of_slot, smp_of_slot = nd.slot_pixels(W, H, TILE[0], TILE[1], 0, 1, spp)
    valid = np.nonzero(pix_of_slot >= 0)[0]
    order = np.argsort(pix_of_slot[valid] * spp + smp_of_slot[valid], kind="stable")
    rays0 = S.primary_rays(S.scene_camera("cornell", W, H), W, H, spp=spp, seed=p.seed)
    pid = valid[order].astype(np.int32)
    n = len(pid)

    def f4(xyz, w):
        return torch.as_tensor(np.concatenate([xyz, np.full((len(xyz), 1), w, np.float32)], axis=1).astype(np.float32),
                               device="cuda")

    d_o, d_d, d_pid = f4(rays0["org"], 1e-3), f4(rays0["dir"], 1e30), torch.as_tensor(pid, device="cuda")

    def buffers():
        out = [torch.zeros((n, 4), device="cuda"), torch.zeros((n, 4), device="cuda"),
               torch.full((n,), -1, dtype=torch.int32, device="cuda")]
        sh = [torch.zeros((n, 4), device="cuda") for _ in range(3)]
        weight = torch.ones((len(pix_of_slot), 4), dtype=torch.float32, device="cuda")
        accum = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")
        return out, sh, weight, accum

    def bounce(bufs, stream=None):
        out, sh, weight, accum = bufs
        nc, ns = acc.PathBounce(p, 0, n, d_o.data_ptr(), d_d.data_ptr(), d_pid.data_ptr(), weight.data_ptr(),
                                out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), sh[0].data_ptr(),
                                sh[1].data_ptr(), sh[2].data_ptr(), accum.data_ptr(),
                                stream=stream.cuda_stream if stream is not None else None)
        torch.cuda.synchronize()
        return nc, ns, [t.cpu().numpy() for t in out]

    want_bufs, got_bufs = buffers(), buffers()
    frame = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    want_nc, want_ns, want = bounce(want_bufs)
    assert want_nc > n // 4 and want_ns > 0
    sa, sb = _gated_streams(torch, 2)
    acc.RenderPath(p, frame.data_ptr(), stream=sa.cuda_stream, want_result=False)
    nc, ns, got = bounce(got_bufs, sb)
    assert (nc, ns) == (want_nc, want_ns)
    gp, wp = got[2][:nc], want[2][:nc]
    assert np.array_equal(np.sort(gp), np.sort(wp)), "different set of continuing paths"
    gs, ws = np.argsort(gp), np.argsort(wp)
    for k in range(2):  # continuation origins, directions
        assert _rel(got[k][:nc][gs][:, :3], want[k][:nc][ws][:, :3]) <= 1e-5, k


# ------------------------------------------------------------------ sharded passes
def test_two_sharded_passes_on_one_communicator_equal_their_render_ao_frames():
    """Two asynchronous nrt_render_ao_sharded calls with different cameras on one communicator of one rank and two
    streams: each frame equals the RenderAO frame of its camera exactly."""
    import torch
    from nanort_b200 import api, scenes as S

    v, f = S.make_scene("sphere_grid", nx=4, nz=4)
    acc = api.BVHAccel()
    assert acc.Build(len(f), v, f)
    W, H = 128, 96
    params = [_ao_params(api, S, "sphere_grid", W, H, 2),
              _ao_params(api, S, "sphere_grid", W, H, 2, cam=S.look_at((4.0, 3.0, 7.0), (0.0, 0.2, 0.0),
                                                                         fov_y_deg=40.0, aspect=W / H))]
    want = [_serial_ao(torch, acc, p)[0] for p in params]
    assert not torch.equal(want[0], want[1])
    try:
        comm = api.Comm(api.Comm.unique_id(), 0, 1)
    except api.NanortB200Error as e:
        pytest.skip(str(e))
    try:
        warm = torch.zeros(W * H, dtype=torch.float32, device="cuda")
        comm.RenderAO(acc, params[0], warm.data_ptr())  # sizes the gather buffer before the gate
        torch.cuda.synchronize()
        assert torch.equal(warm, want[0])
        frames = [torch.full((W * H,), float("nan"), dtype=torch.float32, device="cuda") for _ in params]
        torch.cuda.synchronize()
        for p, fr, s in zip(params, frames, _gated_streams(torch, 2)):
            comm.RenderAO(acc, p, fr.data_ptr(), stream=s.cuda_stream, want_result=False)
        torch.cuda.synchronize()
        for k in range(2):
            assert torch.equal(frames[k], want[k]), (k, int((frames[k] != want[k]).sum().item()))
    finally:
        comm.free()
