"""Codegen guard for cg_spconv.cu (CPU only, needs nvcc): ptxas reports no spill and a 0-byte stack frame for every
kernel of the file, so the conv tile's accumulators and its gathers stay in registers."""
import os
import re
import shutil
import subprocess

import pytest

from catgrasp_b200 import build

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
pytestmark = pytest.mark.skipif(shutil.which(NVCC) is None, reason="nvcc not available")

OWN = ["point_key_kernel", "parent_key_kernel", "head_kernel", "emit_level_kernel", "nbr_kernel", "pairs_kernel",
       "spconv_kernel"]


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    out = tmp_path_factory.mktemp("obj") / "cg_spconv.o"
    flags = [f for f in build.NVCC_FLAGS if f != "-DCG_EXPERIMENTS"]
    p = subprocess.run([NVCC] + flags + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "cg_spconv.cu"), "-o",
                        str(out)], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    props = re.findall(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", p.stderr)
    return {name: tuple(int(v) for v in vals) for name, *vals in props}


@pytest.mark.parametrize("kernel", OWN)
def test_no_spills_and_no_stack(report, kernel):
    found = [n for n in report if f"{len(kernel)}{kernel}" in n]
    assert len(found) == (3 if kernel == "spconv_kernel" else 1), (kernel, sorted(report))   # 16, 32, 64 channels
    for name in found:
        assert report[name] == (0, 0, 0), name
