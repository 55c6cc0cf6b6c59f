"""Codegen guard for the per-pick kernels in cg_pick.cu (CPU only, needs nvcc): ptxas reports no spill and a 0-byte
stack frame for the segment table's and the ranking's kernels, both variants of the statistics kernel included."""
import os
import re
import shutil
import subprocess

import pytest

from catgrasp_b200 import build

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
pytestmark = pytest.mark.skipif(shutil.which(NVCC) is None, reason="nvcc not available")

OWN = ["seg_init_kernel", "seg_stats_kernelILb0", "seg_stats_kernelILb1", "seg_decide_kernel", "seg_order_kernel",
       "seg_points_kernel", "rank_score_kernel"]


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    out = tmp_path_factory.mktemp("obj") / "cg_pick.o"
    flags = [f for f in build.NVCC_FLAGS if f != "-DCG_EXPERIMENTS"]
    p = subprocess.run([NVCC] + flags + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "cg_pick.cu"), "-o",
                        str(out)], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    props = re.findall(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", p.stderr)
    return {name: tuple(int(v) for v in vals) for name, *vals in props}


@pytest.mark.parametrize("kernel", OWN)
def test_no_spills_and_no_stack(report, kernel):
    base = kernel.split("ILb")[0]
    found = [n for n in report if f"{len(base)}{kernel}" in n]
    assert len(found) == 1, (kernel, sorted(report))
    assert report[found[0]] == (0, 0, 0), found[0]
