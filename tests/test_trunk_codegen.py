"""Codegen guard for the tensor-core trunk kernel (CPU only, needs nvcc).

ptxas silently repairs a wgmma pipeline whose registers the compiler has moved across a fence or wait by injecting a
full warpgroup.wait / warpgroup.arrive (C7517 / C7519); the kernel stays correct but its L3 stream is serialised.
Local-memory traffic on the hot path (a stack frame or spills) is as invisible to the correctness tests.  This test
compiles cg_trunk_tc.cu with the flags of build.py and fails on either, for every trunk_tc_kernel instantiation.
"""
import os
import re
import shutil
import subprocess

import pytest

from catgrasp_b200 import build

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
pytestmark = pytest.mark.skipif(shutil.which(NVCC) is None, reason="nvcc not available")


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    out = tmp_path_factory.mktemp("codegen") / "cg_trunk_tc.o"
    src = os.path.join(build.CSRC, "cg_trunk_tc.cu")
    flags = [f for f in build.NVCC_FLAGS if f != "-DCG_EXPERIMENTS"]
    p = subprocess.run([NVCC] + flags + ["-Xptxas", "-v", "-c", src, "-o", str(out)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    return p.stdout + p.stderr


def _per_kernel(log):
    """{instantiation: [ptxas lines]} for every trunk_tc_kernel<PASSES>."""
    kernels = {}
    for line in log.splitlines():
        m = re.search(r"trunk_tc_kernelILi(\d)E", line)
        if m:
            kernels.setdefault(int(m.group(1)), []).append(line)
        elif line.strip().endswith("bytes spill loads") and kernels:
            # the "Function properties" line carries no name: it belongs to the entry compiled last
            last = [k for k in kernels if any("Compiling entry" in x for x in kernels[k])][-1]
            kernels[last].append(line)
    return kernels


def test_every_instantiation_compiled(ptxas_log):
    assert sorted(_per_kernel(ptxas_log)) == [1, 2, 3]


@pytest.mark.parametrize("passes", [1, 2, 3])
def test_no_injected_wgmma_waits(ptxas_log, passes):
    injected = [x for x in _per_kernel(ptxas_log)[passes] if "C7517" in x or "C7519" in x]
    assert not injected, "\n".join(injected)


@pytest.mark.parametrize("passes", [1, 2, 3])
def test_no_stack_frame_or_spills(ptxas_log, passes):
    props = [x for x in _per_kernel(ptxas_log)[passes] if "stack frame" in x]
    assert props, _per_kernel(ptxas_log)[passes]
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", props[-1])
    assert m and m.groups() == ("0", "0", "0"), props[-1]
