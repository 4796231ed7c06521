"""CPU: the wavefront passes' host plumbing (nanort_b200/csrc/pass_host.cuh), compiled into a small host program that
runs without a GPU.  The scratch carver must measure exactly what it hands out, on 256-byte boundaries and without
overlap; the shard and wave arithmetic must deal out tiles as a plain restatement of the round-robin rule does; a pass
clock that is off (the caller passed no result struct) must make no CUDA call and read zero times."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "nanort_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

PROGRAM = r"""
#include <stdio.h>
#include <string.h>

#include "pass_host.cuh"

namespace nrt {
void set_error(const std::string &) {}
int cuda_fail(cudaError_t, const char *, const char *, int) { return NRT_ERR_CUDA; }
}  // namespace nrt
using namespace nrt;

// a 256-byte aligned base address the carver only does arithmetic on
static char *const kBase = reinterpret_cast<char *>((size_t)1 << 40);

static void buf(const void *p, size_t bytes) {
  printf("buf %zu %zu\n", (size_t)(static_cast<const char *>(p) - kBase), bytes);
}

int main() {
  char cmd[16];
  while (scanf("%15s", cmd) == 1) {
    if (!strcmp(cmd, "queues")) {  // carve_path_queues(cap)
      size_t cap;
      if (scanf("%zu", &cap) != 1) return 2;
      Carver measure, c(kBase);
      carve_path_queues(measure, cap);
      const PathQueues q = carve_path_queues(c, cap);
      printf("size %zu %zu\n", measure.size(), c.size());
      for (int k = 0; k < 2; k++) {
        buf(q.org_tmin[k], 16 * cap);
        buf(q.dir_tmax[k], 16 * cap);
        buf(q.path_id[k], 4 * cap);
      }
      buf(q.sh_org_tmin, 16 * cap);
      buf(q.sh_dir_tmax, 16 * cap);
      buf(q.sh_contrib_pix, 16 * cap);
      buf(q.weight, 16 * cap);
    } else if (!strcmp(cmd, "bytes")) {  // n buffers of the given byte sizes, then 3-float records of the last size
      int n;
      if (scanf("%d", &n) != 1) return 2;
      size_t sizes[64];
      for (int i = 0; i < n; i++)
        if (scanf("%zu", &sizes[i]) != 1) return 2;
      Carver measure, c(kBase);
      for (int i = 0; i < n; i++) measure.take<unsigned char>(sizes[i]);
      measure.take<float3>(sizes[n - 1]);
      void *p[65];
      for (int i = 0; i < n; i++) p[i] = c.take<unsigned char>(sizes[i]);
      p[n] = c.take<float3>(sizes[n - 1]);
      printf("size %zu %zu\n", measure.size(), c.size());
      for (int i = 0; i < n; i++) buf(p[i], sizes[i]);
      buf(p[n], 12 * sizes[n - 1]);
    } else if (!strcmp(cmd, "clock_off")) {  // a pass with no result struct: no event, no CUDA call, zero times
      PassClock clock(false);
      int rc = clock.start(nullptr);
      for (int tag = 0; tag < 2; tag++) {
        rc |= clock.begin(nullptr);
        rc |= clock.end(nullptr, tag);
      }
      rc |= clock.stop(nullptr);
      float total = -1.0f, span[2] = {-1.0f, -1.0f};
      rc |= clock.read(&total, span);
      printf("clock %d %g %g %g\n", rc, total, span[0], span[1]);
      continue;
    } else if (!strcmp(cmd, "shard")) {  // width height tile_w tile_h spp shard n_shards budget
      unsigned w, h, tw, th, spp, shard, n;
      unsigned long long budget;
      if (scanf("%u %u %u %u %u %u %u %llu", &w, &h, &tw, &th, &spp, &shard, &n, &budget) != 8) return 2;
      const ShardSlots s = shard_slots(w, h, tw, th, spp, shard, n);
      printf("shard %llu %llu %llu %llu\n", s.tiles, s.per_tile, s.total, s.wave(budget));
      continue;
    } else {
      return 2;
    }
    printf("end\n");
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def program(tmp_path_factory):
    if not os.path.exists(NVCC) and not shutil.which("nvcc"):
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("pass_host")
    src = d / "pass_host_check.cu"
    src.write_text(PROGRAM)
    exe = d / "pass_host_check"
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-Xcompiler", "-Wall",
                        f"-I{CSRC}", str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return str(exe)


def run(program, lines):
    r = subprocess.run([program], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    return r.stdout.split("\n")


def layouts(program, lines):
    """[(measured size, carved size, [(offset, bytes), ...]), ...] per carving command"""
    out, cur = [], None
    for line in run(program, lines):
        f = line.split()
        if not f:
            continue
        if f[0] == "size":
            cur = (int(f[1]), int(f[2]), [])
        elif f[0] == "buf":
            cur[2].append((int(f[1]), int(f[2])))
        elif f[0] == "end":
            out.append(cur)
    return out


def check_layout(measured, carved, bufs):
    assert measured == carved
    for off, nbytes in bufs:
        assert off % 256 == 0
        assert 0 <= off and off + nbytes <= carved
    spans = sorted(bufs)
    for (o0, n0), (o1, _) in zip(spans, spans[1:]):
        assert o0 + n0 <= o1, "buffers overlap"
    # nothing but the rounding of each buffer up to 256 bytes is added
    assert carved == sum((n + 255) // 256 * 256 for _, n in bufs)


@pytest.mark.parametrize("cap", [0, 1, 7, 32, 4096, 1000003, 8 << 20])
def test_path_queues_layout(program, cap):
    [(measured, carved, bufs)] = layouts(program, [f"queues {cap}"])
    assert len(bufs) == 10
    check_layout(measured, carved, bufs)


@pytest.mark.parametrize("sizes", [[1], [0, 0, 5], [255, 256, 257, 1], [4, 12, 4096, 3, 100000, 64]])
def test_carver_layout(program, sizes):
    [(measured, carved, bufs)] = layouts(program, [f"bytes {len(sizes)} " + " ".join(map(str, sizes))])
    assert len(bufs) == len(sizes) + 1
    check_layout(measured, carved, bufs)


def shard_ref(w, h, tw, th, spp, shard, n, budget):
    """this shard's tiles dealt round-robin, and a wave of whole tiles: at most budget slots, at least one tile"""
    n_tiles = -(-w // tw) * -(-h // th)
    tiles = len(range(shard, n_tiles, n))
    per_tile = tw * th * spp
    total = tiles * per_tile
    return tiles, per_tile, total, min(total, max(1, budget // per_tile) * per_tile)


SHARD_CASES = [
    (64, 32, 8, 4, 1, 0, 1, 16 << 20),          # whole tiles only
    (100, 50, 8, 4, 3, 0, 1, 16 << 20),         # partial edge tiles
    (100, 50, 16, 8, 7, 0, 1, 1000),            # several waves, partial edge tiles
    (8, 4, 8, 4, 1, 3, 4, 8 << 20),             # shard >= n_tiles: nothing to do
    (10, 10, 8, 4, 2, 5, 6, 8 << 20),           # 6 tiles, the last shard's one
    (64, 64, 64, 64, 4096, 0, 1, 1 << 22),      # one tile larger than the wave budget
    (1920, 1080, 32, 16, 16, 0, 1, 4 << 20),
    (3840, 2160, 64, 32, 64, 0, 1, 16 << 20),   # the AO pass's budget
    (4096, 4096, 256, 256, 1024, 0, 1, (512 << 20) // 2000),  # a BDPT-like byte budget over a large per-slot size
]
SHARD_CASES += [(1000, 700, 16, 8, 5, k, 3, 8 << 20) for k in range(3)]   # several shards
SHARD_CASES += [(257, 129, 8, 4, 2, k, 8, 1 << 22) for k in range(8)]


def test_shard_slots_against_restatement(program):
    lines = ["shard " + " ".join(map(str, c)) for c in SHARD_CASES]
    got = [tuple(map(int, line.split()[1:])) for line in run(program, lines) if line.startswith("shard")]
    assert got == [shard_ref(*c) for c in SHARD_CASES]
    for (w, h, tw, th, spp, shard, n, budget), (tiles, per_tile, total, wave) in zip(SHARD_CASES, got):
        if total:
            assert wave % per_tile == 0 and 0 < wave <= total


def test_shards_cover_every_tile_once(program):
    w, h, tw, th, spp, n = 1000, 700, 16, 8, 5, 3
    lines = [f"shard {w} {h} {tw} {th} {spp} {k} {n} {8 << 20}" for k in range(n)]
    tiles = [int(line.split()[1]) for line in run(program, lines) if line.startswith("shard")]
    assert sum(tiles) == -(-w // tw) * -(-h // th)


def test_pass_clock_off_reads_zero_without_cuda(program):
    # off, the clock touches no CUDA API: this runs on a machine with no GPU and no driver
    [line] = [ln for ln in run(program, ["clock_off"]) if ln.startswith("clock")]
    assert line.split()[1:] == ["0", "0", "0", "0"]
