"""Workspace carving and host staging (CPU only, needs g++ and the CUDA headers): cg_ws_carve / cg_io_carve /
cg_io_stage of cg_common.cuh.

Every library entry point that needs scratch memory describes its pieces once, as a layout of cg_arena::take calls.
The helper runs the layout over a measuring arena (base nullptr), reserves exactly the bytes it measured, and runs it
again over the reserved arena.  Every *_host entry point stages through cg_io_stage: its layout's pieces are carved
over the io arena the same way, then inputs are copied in, the compute step runs, and outputs are copied out.  This
test compiles a small host program against cg_common.cuh, with host stand-ins for the two reservations of cg_api.cu
and for the CUDA runtime calls of cg_io_stage (plain memcpy, each call logged), and checks
- for layouts with odd piece sizes (12 P + 4 bytes, 1-byte and empty pieces): the measuring run returns null pointers
  and reports the size the carve ends at, each arena reserves exactly that size, and the carved offsets are the
  expected ones, each a multiple of 256;
- that a layout that takes a different size on its second run is refused with CG_EINVAL instead of writing past the
  arena;
- that cg_io_stage copies inputs in declaration order before the compute step, copies back only the outputs with a
  host pointer after it, and synchronises last; that empty inputs and outputs take an aligned piece and copy nothing;
- that a failing compute step returns its status with nothing copied back or synchronised, and that a compute step
  which carves the io arena is refused with CG_EINVAL while one that carves ws is not.

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

// host stand-ins for the runtime calls of cg_io_stage: copies are memcpy, and each call is logged with the io offset
static std::string trace;
static const char *io_base;
static std::string at(const void *p) { return std::to_string(static_cast<const char *>(p) - io_base); }
cudaError_t cudaSetDevice(int) { return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void *dst, const void *src, size_t n, cudaMemcpyKind kind, cudaStream_t) {
  memcpy(dst, src, n);
  trace += kind == cudaMemcpyHostToDevice ? " h2d@" + at(dst) : " d2h@" + at(src);
  trace += ":" + std::to_string(n);
  return cudaSuccess;
}
cudaError_t cudaStreamSynchronize(cudaStream_t) { trace += " sync"; return cudaSuccess; }
const char *cudaGetErrorString(cudaError_t) { return "stand-in"; }

// argv[2]: ok, fail (the compute step returns CG_ECUDA), carve_io / carve_ws (it carves that arena), stage_io (it
// runs a stage of its own)
static int stage(const std::string &mode) {
  cg_ctx ctx;
  reserve(&ctx.io, &ctx.io_bytes, 4096, 1);   // a fixed base for the offsets in the log
  io_base = static_cast<const char *>(ctx.io);
  const double a[3] = {1.5, 2.5, 3.5};
  const int32_t b[5] = {4, 5, 6, 7, 8};
  float out[4] = {0, 0, 0, 0}, empty_out[1] = {-1};
  void *p[8];
  bool seen = false;
  const int rc = cg_io_stage(&ctx, [&](cg_io_pieces &io) {
    p[0] = io.in(a, 3);
    p[1] = io.in<float>(nullptr, 0);         // an empty input, as from a null, empty point set
    p[2] = io.in(b, 5);
    p[3] = io.take<char>(0);
    p[4] = io.out(out, 4);
    p[5] = io.out<int32_t>(nullptr, 2);      // an output the caller does not want
    p[6] = io.out(empty_out, 0);
    p[7] = io.take<double>(7);
  }, [&] {
    trace += " compute";
    seen = !memcmp(p[0], a, sizeof(a)) && !memcmp(p[2], b, sizeof(b));
    for (int i = 0; i < 4; i++) static_cast<float *>(p[4])[i] = 9.f + i;
    if (mode == "fail") return CG_ECUDA;
    if (mode == "carve_io") return cg_io_carve(&ctx, [](cg_arena &ar) { ar.take<char>(1); });
    if (mode == "stage_io") return cg_io_stage(&ctx, [](cg_io_pieces &io) { io.take<char>(1); }, [] { return CG_OK; });
    if (mode == "carve_ws") return cg_ws_carve(&ctx, [](cg_arena &ar) { ar.take<char>(1); });
    return CG_OK;
  });
  printf("rc %d\nseen %d\nheld %d\ntrace%s\n", rc, (int)seen, (int)ctx.io_held, trace.c_str());
  printf("pieces");
  for (void *q : p) printf(" %s", at(q).c_str());
  printf("\nout %g %g %g %g %g\nerr %s\n", out[0], out[1], out[2], out[3], empty_out[0], ctx.err.c_str());
  free(ctx.ws);
  free(ctx.io);
  return 0;
}

struct Piece { char type; size_t n; };

// argv: pieces as <type>:<count>, type c (1 byte), f (float), d (double); or stage <mode>
int main(int argc, char **argv) {
  if (argc == 3 && !strcmp(argv[1], "stage")) return stage(argv[2]);
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

SIZE = {"c": 1, "i": 4, "f": 4, "d": 8}


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
    """odd piece sizes: (P,3) float point sets with one spare float each (12 P + 4 bytes), 1-byte status and offset
    arrays, empty and boundary-sized pieces"""
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


# the stage program's layout: in (3,) double, empty in, in (5,) int32, empty scratch, out (4,) float, out without a
# host pointer, empty out, scratch (7,) double
STAGE_PIECES = [("d", 3), ("f", 0), ("i", 5), ("c", 0), ("f", 4), ("i", 2), ("f", 0), ("d", 7)]
H2D = " h2d@0:24 h2d@256:20 compute"


@pytest.mark.parametrize("mode, rc, trace", [
    ("ok", 0, H2D + " d2h@512:16 sync"),
    ("carve_ws", 0, H2D + " d2h@512:16 sync"),      # a compute step may carve ws
    ("fail", -2, H2D),                               # its status as it is, nothing copied back, no synchronisation
    ("carve_io", -1, H2D),                           # CG_EINVAL: the pieces it works on live in io
    ("stage_io", -1, H2D),                           # a stage of its own carves io too
])
def test_io_stage(program, mode, rc, trace):
    out = subprocess.run([program, "stage", mode], capture_output=True, text=True, check=True)
    lines = {ln.split()[0]: ln.split(maxsplit=1)[1:] for ln in out.stdout.splitlines()}
    assert int(lines["rc"][0]) == rc
    assert " " + lines["trace"][0] == trace           # inputs in declaration order, then compute, outputs, sync
    assert lines["seen"] == ["1"]                     # the compute step saw every input on the device
    assert lines["held"] == ["0"]
    pieces = list(map(int, lines["pieces"][0].split()))
    assert pieces == _expected(STAGE_PIECES)[1]
    assert all(o % 256 == 0 for o in pieces)
    spans = sorted((o, o + n * SIZE[t]) for o, (t, n) in zip(pieces, STAGE_PIECES))
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
    values = lines["out"][0].split()
    assert values == (["9", "10", "11", "12"] if rc == 0 else ["0"] * 4) + ["-1"]
    assert ("internal error" in " ".join(lines["err"])) == mode.endswith("_io")
