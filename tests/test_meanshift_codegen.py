"""Codegen guard for cg_meanshift.cu (CPU only, needs nvcc): its kernels are compared bit for bit with
oracle/meanshift_ref.py, so none may contain a fused multiply-add (nvcc contracts a * b + c by default; the oracle
rounds twice).  Same method as test_bitexact_codegen.py.

Seeded mutation aimed at: the ascent's distance or mean written with plain operators, e.g. ``dx * dx + dy * dy``."""
import os
import re
import shutil
import subprocess

import pytest

from catgrasp_b200 import build

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
pytestmark = pytest.mark.skipif(shutil.which(NVCC) is None, reason="nvcc not available")

# (kernel, mangled template arguments)
KERNELS = [("quantise_kernel", ""), ("ascent_kernel", "IfE"), ("ascent_kernel", "IdE"), ("rank_kernel", "IfE"),
           ("rank_kernel", "IdE"), ("suppress_kernel", "")]


@pytest.fixture(scope="module")
def entries(tmp_path_factory):
    out = tmp_path_factory.mktemp("ptx") / "cg_meanshift.ptx"
    flags = [f for f in build.NVCC_FLAGS if f != "-DCG_EXPERIMENTS"]
    p = subprocess.run([NVCC] + flags + ["-ptx", os.path.join(build.CSRC, "cg_meanshift.cu"), "-o", str(out)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    ptx = out.read_text()
    starts = list(re.finditer(r"^(?:\.visible\s+|\.weak\s+)*\.entry\s+(\S+?)\s*\(", ptx, re.M))
    return {m.group(1): ptx[m.start():n.start() if n else len(ptx)] for m, n in zip(starts, starts[1:] + [None])}


@pytest.mark.parametrize("name, targs", KERNELS)
def test_no_fused_multiply_add(entries, name, targs):
    found = [e for e in entries if f"{len(name)}{name}{targs}" in e]
    assert len(found) == 1, (name + targs, sorted(entries))
    assert not re.findall(r"\bfma\.rn\.f(?:32|64)\b", entries[found[0]])
