"""Codegen guard for the kernels that must agree bit for bit with a CPU oracle (CPU only, needs nvcc).

nvcc contracts ``a * b + c`` into one fused multiply-add by default (--fmad=true), which rounds once where the oracles
(numpy, or C built with -ffp-contract=off) round twice.  A kernel whose result is compared bit for bit therefore writes
its floating-point arithmetic with round-to-nearest intrinsics (__dmul_rn, __dadd_rn, ...), which nvcc never fuses.
This test compiles cg_occupancy.cu and cg_cloud.cu to PTX with the flags of build.py and fails when any listed
kernel contains an ``fma.rn.f64`` or ``fma.rn.f32``.

normals_kernel is exempt: its Jacobi solver and norm are checked against an eigengap error bound, not bit for bit
(tests/test_cloud_kernels.py), and may contract.

Seeded mutation aimed at: re-enabling contraction in a bit-exact kernel, e.g. occ_cast_kernel's centre distance
written as ``sqrt(cx * cx + cy * cy + cz * cz)`` (two fma.rn.f64; the parent of this test's commit had exactly that).
"""
import os
import re
import shutil
import subprocess

import pytest

from catgrasp_b200 import build

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
pytestmark = pytest.mark.skipif(shutil.which(NVCC) is None, reason="nvcc not available")

# (kernel, template arguments as mangled): float and double depth2xyz are separate entries
BIT_EXACT = {
    "cg_occupancy.cu": [("occ_mark_kernel", ""), ("occ_cast_kernel", "")],
    "cg_cloud.cu": [("bounds_kernel", ""), ("key_kernel", ""), ("voxel_kernel", ""), ("nearest_kernel", ""),
                    ("radius_mask_kernel", ""), ("depth2xyz_kernel", "IfE"), ("depth2xyz_kernel", "IdE")],
}
EXEMPT = {"cg_cloud.cu": [("normals_kernel", "")]}


def _entries(ptx):
    """{mangled entry name: body} for every .entry of a PTX module."""
    out = {}
    starts = list(re.finditer(r"^(?:\.visible\s+|\.weak\s+)*\.entry\s+(\S+?)\s*\(", ptx, re.M))
    for m, nxt in zip(starts, starts[1:] + [None]):
        out[m.group(1)] = ptx[m.start():nxt.start() if nxt else len(ptx)]
    return out


@pytest.fixture(scope="module", params=sorted(BIT_EXACT))
def ptx(request, tmp_path_factory):
    src = os.path.join(build.CSRC, request.param)
    out = tmp_path_factory.mktemp("ptx") / (request.param + ".ptx")
    flags = [f for f in build.NVCC_FLAGS if f != "-DCG_EXPERIMENTS"]
    p = subprocess.run([NVCC] + flags + ["-ptx", src, "-o", str(out)], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    return request.param, _entries(out.read_text())


def _find(entries, name, targs):
    """The entries whose mangled name holds ``<len(name)><name><targs>`` (Itanium: an identifier follows its length,
    so bounds_kernel does not match bounds_final_kernel)."""
    key = f"{len(name)}{name}{targs}"
    return [e for e in entries if key in e]


def test_every_listed_kernel_found(ptx):
    src, entries = ptx
    for name, targs in BIT_EXACT[src] + EXEMPT.get(src, []):
        assert len(_find(entries, name, targs)) == 1, (name + targs, sorted(entries))


def test_no_fused_multiply_add(ptx):
    src, entries = ptx
    bad = {}
    for name, targs in BIT_EXACT[src]:
        (e,) = _find(entries, name, targs)
        n = len(re.findall(r"\bfma\.rn\.f(?:32|64)\b", entries[e]))
        if n:
            bad[name + targs] = n
    assert not bad, f"{src}: fused multiply-adds in bit-exact kernels: {bad}"
