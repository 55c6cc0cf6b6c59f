"""The measurement scripts measure through scripts/_harness.py: one card query for the torch device, three timers,
the reference camera.  Checked without a GPU: the CUDA calls the timers make are replaced by recording stubs."""
import ast
import glob
import importlib.util
import os
import subprocess
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = os.path.join(ROOT, "scripts")
CONVERTED = ["bench_primitives", "fps_probe", "l2_stream_probe", "time_cloud_prep", "time_filter", "time_ik",
             "time_meanshift", "time_nunocs", "time_pick", "time_pointgroup", "time_sdf_build", "time_spconv"]


@pytest.fixture
def harness(monkeypatch):
    monkeypatch.setattr(sys, "path", list(sys.path))      # the harness puts the repository root on it
    spec = importlib.util.spec_from_file_location("_harness", os.path.join(SCRIPTS, "_harness.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture
def log(monkeypatch):
    """Replaces the CUDA events, the device synchronise and the host clock with stubs that append to one log."""
    log = []

    class Event:
        def __init__(self, enable_timing=False):
            assert enable_timing

        def record(self, stream=None):
            log.append("record")

        def synchronize(self):
            log.append("wait")

        def elapsed_time(self, end):
            return 1.0

    monkeypatch.setattr(torch.cuda, "Event", Event)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda device=None: log.append("wait"))
    import time
    monkeypatch.setattr(time, "perf_counter", lambda: log.append("clock") or float(len(log)))
    return log


def _timed(log, warmup):
    """The log from the first timed call on (the warm-up calls and their synchronise removed)."""
    return log[[i for i, e in enumerate(log) if e == "call"][warmup]:]


def test_only_the_harness_queries_the_card_times_with_events_or_holds_the_camera():
    for path in sorted(glob.glob(os.path.join(SCRIPTS, "*.py"))):
        if os.path.basename(path) == "_harness.py":
            continue
        with open(path) as f:
            src = f.read()
        if os.path.basename(path) == "time_pointgroup.py":
            # stages() brackets the forward and the head inside one predict with events of its own: stage logic that
            # no harness timer can take over
            stages = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "stages")
            src = src.replace(ast.get_source_segment(src, stages), "")
        for needle in ("nvidia-smi", "torch.cuda.Event", "2257.75"):
            assert needle not in src, (os.path.basename(path), needle)


def test_scripts_import_without_running_main_or_initialising_cuda():
    code = f"""
import importlib.util, os, sys
import torch
sys.path.insert(0, {SCRIPTS!r})
import _harness
def ran(*a, **k):
    raise AssertionError("main() ran on import")
_harness.card = _harness.smi = ran
for name in {CONVERTED!r}:
    spec = importlib.util.spec_from_file_location(name, os.path.join({SCRIPTS!r}, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert callable(mod.main), name
    assert not torch.cuda.is_initialized(), name
"""
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-3000:]


def test_card_needs_cuda(harness, monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError):
        harness.card()


@pytest.mark.parametrize("reps,warmup", [(4, 2), (1, 0)])
def test_synced_ms_waits_after_every_timed_call(harness, log, reps, warmup):
    ts = harness.synced_ms(lambda: log.append("call"), reps, warmup)
    assert len(ts) == reps and log.count("call") == warmup + reps
    timed = _timed(log, warmup)
    for i, e in enumerate(timed):
        if e == "call":
            assert "wait" in timed[i + 1:(timed + ["call"]).index("call", i + 1)]


@pytest.mark.parametrize("reps,warmup", [(4, 2), (1, 0)])
def test_queued_ms_waits_once_after_the_last_call(harness, log, reps, warmup):
    ts = harness.queued_ms(lambda: log.append("call"), reps, warmup)
    assert len(ts) == reps and log.count("call") == warmup + reps
    timed = _timed(log, warmup)
    assert timed.count("wait") == 1
    assert timed.index("wait") > len(timed) - 1 - timed[::-1].index("call")
    assert "wait" in log[:log.index("record")]          # the warm-up has finished before the first event


@pytest.mark.parametrize("reps,warmup", [(4, 2), (1, 0)])
def test_wall_ms_reads_the_clock_on_a_synchronised_device(harness, log, reps, warmup):
    ts = harness.wall_ms(lambda: log.append("call"), reps, warmup)
    assert len(ts) == reps and log.count("call") == warmup + reps
    clocks = [i for i, e in enumerate(log) if e == "clock"]
    assert len(clocks) == 2 * reps
    for i in clocks:
        assert log[i - 1] == "wait"
    for start, end in zip(clocks[::2], clocks[1::2]):
        assert log[start + 1:end].count("call") == 1


@pytest.fixture
def device(monkeypatch):
    props = types.SimpleNamespace(name="NVIDIA H100 80GB HBM3", uuid="0b5a1c52-7f3e-4c1d-9a66-3e2f8d1b4c07")
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "get_device_properties", lambda device=None: props)
    return props


def test_smi_selects_the_torch_device_by_uuid(harness, device, monkeypatch):
    calls = []

    def run(argv, **kw):
        calls.append(argv)
        return subprocess.CompletedProcess(argv, 0, "NVIDIA H100 80GB HBM3, 400.00 W, 1980 MHz\n", "")

    monkeypatch.setattr(subprocess, "run", run)
    assert harness.card() == "NVIDIA H100 80GB HBM3, 400.00 W, 1980 MHz"
    argv = calls[0]
    assert argv[0] == "nvidia-smi" and "--query-gpu=name,power.limit,clocks.max.sm" in argv
    assert argv[argv.index("-i") + 1] == f"GPU-{device.uuid}"


def test_card_names_the_device_and_the_reason_when_nvidia_smi_fails(harness, device, monkeypatch):
    def run(argv, **kw):
        raise FileNotFoundError(2, "No such file or directory", "nvidia-smi")

    monkeypatch.setattr(subprocess, "run", run)
    line = harness.card()
    assert line.startswith(device.name) and "power limit not read" in line and "No such file or directory" in line
