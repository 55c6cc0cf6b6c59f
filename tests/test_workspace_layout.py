"""Workspace carving (CPU only, needs g++ and the CUDA headers): cg_ws_carve / cg_io_carve of cg_common.cuh.

Every library entry point that needs scratch memory describes its pieces once, as a layout of cg_arena::take calls.
The helper runs the layout over a measuring arena (base nullptr), reserves exactly the bytes it measured, and runs it
again over the reserved arena.  This test compiles a small host program against cg_common.cuh, with host stand-ins for
the two reservations of cg_api.cu, and checks for layouts with odd piece sizes (12 P + 4 bytes, 1-byte and empty
pieces) that
- the measuring run returns null pointers and reports the size the carve ends at,
- each helper reserves exactly that size, and the carved offsets are the expected ones, each a multiple of 256,
- a layout that takes a different size on its second run is refused with CG_EINVAL instead of writing past the arena.

Seeded mutation aimed at: a measuring arena that skips the 256-byte rounding (it under-reports every layout whose
pieces are not multiples of 256 bytes).
"""
import os
import shutil
import subprocess

import pytest

from catgrasp_b200 import build

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUDA_INCLUDE = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(NVCC))), "include")
CXX = os.environ.get("CXX", "g++")
pytestmark = pytest.mark.skipif(shutil.which(CXX) is None or not os.path.exists(os.path.join(CUDA_INCLUDE, "cuda_runtime.h")),
                                reason="no host C++ compiler or CUDA headers")

PROGRAM = r"""
#include <stdlib.h>
#include "cg_common.cuh"

// host stand-ins for cg_api.cu: record the request and hand out a 256-aligned host block (grow-only)
static size_t requested[2];
static int reserve(void **arena, size_t *cur, size_t bytes, int which) {
  requested[which] = bytes;
  if (bytes > *cur) {
    free(*arena);
    *arena = aligned_alloc(256, (bytes + 255) / 256 * 256);
    *cur = bytes;
  }
  return CG_OK;
}
int cg_ws_reserve(cg_ctx *ctx, size_t bytes) { return reserve(&ctx->ws, &ctx->ws_bytes, bytes, 0); }
int cg_io_reserve(cg_ctx *ctx, size_t bytes) { return reserve(&ctx->io, &ctx->io_bytes, bytes, 1); }

struct Piece { char type; size_t n; };

// argv: pieces as <type>:<count>, type c (1 byte), f (float), d (double)
int main(int argc, char **argv) {
  std::vector<Piece> pieces;
  for (int i = 1; i < argc; i++) pieces.push_back({argv[i][0], strtoull(argv[i] + 2, nullptr, 10)});
  std::vector<void *> got(pieces.size());
  auto layout = [&](cg_arena &ar) {
    for (size_t i = 0; i < pieces.size(); i++) {
      const Piece &p = pieces[i];
      got[i] = p.type == 'c' ? (void *)ar.take<char>(p.n) : p.type == 'f' ? (void *)ar.take<float>(p.n)
                                                                           : (void *)ar.take<double>(p.n);
    }
  };
  cg_arena measure(nullptr);
  layout(measure);
  int nonnull = 0;
  for (void *p : got) nonnull += p != nullptr;
  printf("measure %zu %d\n", measure.off, nonnull);
  cg_ctx ctx;
  for (int io = 0; io < 2; io++) {
    const int rc = io ? cg_io_carve(&ctx, layout) : cg_ws_carve(&ctx, layout);
    const char *base = static_cast<const char *>(io ? ctx.io : ctx.ws);
    printf("%s %d %zu", io ? "io" : "ws", rc, requested[io]);
    for (void *p : got) printf(" %td", static_cast<const char *>(p) - base);
    printf("\n");
  }
  int runs = 0;
  const int rc = cg_ws_carve(&ctx, [&](cg_arena &ar) { ar.take<char>(runs++ ? 257 : 1); });
  printf("unstable %d %d %s\n", rc, runs, ctx.err.c_str());
  free(ctx.ws);
  free(ctx.io);
  return 0;
}
"""

SIZE = {"c": 1, "f": 4, "d": 8}


@pytest.fixture(scope="module")
def program(tmp_path_factory):
    d = tmp_path_factory.mktemp("layout")
    src, exe = d / "layout.cpp", d / "layout"
    src.write_text(PROGRAM)
    p = subprocess.run([CXX, "-std=c++17", "-O2", "-I", build.CSRC, "-I", CUDA_INCLUDE, str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    return str(exe)


def _expected(pieces):
    off, offsets = 0, []
    for t, n in pieces:
        off = (off + 255) // 256 * 256
        offsets.append(off)
        off += n * SIZE[t]
    return off, offsets


def _filter_staging(P):
    """the shape of cg_filter_grasp_pose_host's io carve: two (P,3) float point sets with one spare float each
    (12 P + 4 bytes), 1-byte status and offset arrays, empty and boundary-sized pieces"""
    return [("f", 3 * P + 1), ("f", 3 * P + 1), ("c", 1), ("c", 1), ("c", 0), ("d", P), ("c", 255), ("c", 256),
            ("c", 257), ("f", 3 * P + 1)]


CASES = {**{f"filter_P{P}": _filter_staging(P) for P in (1, 2, 63, 64, 65, 4096, 100003)},
         "one_byte": [("c", 1)], "empty": [("c", 0)], "five_bytes": [("c", 1)] * 5}


@pytest.mark.parametrize("pieces", list(CASES.values()), ids=list(CASES))
def test_measured_layout_matches_carve(program, pieces):
    out = subprocess.run([program] + [f"{t}:{n}" for t, n in pieces], capture_output=True, text=True, check=True)
    lines = {ln.split()[0]: ln.split()[1:] for ln in out.stdout.splitlines()}
    size, offsets = _expected(pieces)
    measured, nonnull = map(int, lines["measure"])
    assert measured == size
    assert nonnull == 0                    # a measuring arena hands out no pointers
    for arena in ("ws", "io"):
        rc, reserved, *carved = map(int, lines[arena])
        assert rc == 0
        assert reserved == size            # exactly the measured bytes, no slack
        assert carved == offsets
        assert all(o % 256 == 0 for o in carved)
        assert carved[-1] + pieces[-1][1] * SIZE[pieces[-1][0]] == size


def test_unstable_layout_refused(program):
    out = subprocess.run([program, "c:1"], capture_output=True, text=True, check=True)
    rc, runs, *err = out.stdout.splitlines()[-1].split()[1:]
    assert int(rc) == -1                   # CG_EINVAL
    assert int(runs) == 2
    assert "internal error" in " ".join(err)
