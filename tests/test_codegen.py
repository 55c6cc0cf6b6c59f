"""Code-generation contracts of every kernel the library defines (CPU only, needs nvcc).

The correctness tests cannot see three properties the kernels rely on, so this file compiles every .cu of
build.sources() with the flags of build.py, once with ``-Xptxas -v -c`` for ptxas's per-entry report and once with
``-ptx``, and holds each kernel entry to the rules of its row in KERNELS:

- No local memory: ptxas reports a 0-byte stack frame and no spills.  Local-memory traffic on a hot path is invisible
  to the correctness tests.  A row with ``local`` is exempt and says why.
- ``no_fma``: no ``fma.rn.f32`` / ``fma.rn.f64`` in the entry's PTX.  nvcc contracts ``a * b + c`` into one fused
  multiply-add by default (--fmad=true), which rounds once where the oracles (numpy, or C built with
  -ffp-contract=off) round twice.  A kernel whose result is compared bit for bit with such an oracle therefore writes
  its floating-point arithmetic with round-to-nearest intrinsics (__dmul_rn, __dadd_rn, ...), which nvcc never fuses.
  Only such kernels carry the rule.
- No injected wgmma waits, for every entry whose PTX issues ``wgmma.mma_async``: ptxas silently repairs a wgmma
  pipeline whose registers the compiler has moved across a fence or wait by injecting a full warpgroup.wait /
  warpgroup.arrive (C7517 / C7519; every such notice reads "wgmma.mma_async instructions are serialized").  The
  kernel stays correct but its pipeline is serialised.

Every entry the library defines has exactly one row, and every row names exactly one entry, so a new kernel without a
contract fails here, and so does a row whose template instantiation has gone.  CUB's kernels are not ours and are not
checked.  Register counts vary with the toolchain and are not asserted.
"""
import collections
import os
import re
import shutil
import subprocess

import pytest

from catgrasp_b200 import build

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
pytestmark = pytest.mark.skipif(shutil.which(NVCC) is None, reason="nvcc not available")

SOURCES = [os.path.basename(s) for s in build.sources() if s.endswith(".cu")]

# name: the kernel's identifier; targs: its template arguments as mangled (float and double instantiations are
# separate entries); no_fma: the kernel is compared bit for bit and contains no contracted FMA; local: why the entry
# may have a stack frame or spills.  These five are left as they are: changing their code generation can change speed.
Row = collections.namedtuple("Row", "name targs no_fma local", defaults=("", False, None))

KERNELS = {
    "cg_affordance.cu": [Row("affordance_kernel")],
    # normals_kernel may contract: its Jacobi solver and norm are checked against an eigengap error bound, not bit
    # for bit (tests/test_cloud_kernels.py).
    "cg_cloud.cu": [Row("bounds_kernel", no_fma=True), Row("bounds_final_kernel"), Row("key_kernel", no_fma=True),
                    Row("head_flag_kernel"), Row("table_kernel"), Row("voxel_kernel", no_fma=True),
                    Row("nearest_kernel", no_fma=True), Row("radius_mask_kernel", no_fma=True), Row("normals_kernel"),
                    Row("depth2xyz_kernel", "IfE", no_fma=True), Row("depth2xyz_kernel", "IdE", no_fma=True)],
    "cg_collide.cu": [Row("filter_kernel"), Row("sdf_lookup_kernel")],
    "cg_cone.cu": [Row("cone_pose_kernel"), Row("center_grasp_kernel")],
    "cg_draw.cu": [Row("draw_ids_kernel")],
    "cg_ik.cu": [
        Row("ik_kernel", local="40-byte frame of the out-of-line call to __internal_trig_reduction_slowpathd, the "
                               "large-argument reduction of double sincos"),
        Row("filter_ik_kernel", local="as ik_kernel: the same solver, inlined"),
    ],
    "cg_linear.cu": [Row("linear_kernel"), Row("linear_wide_kernel"), Row("linear_rows_kernel"),
                     Row("softmax_kernel"), Row("nunocs_post_kernel")],
    "cg_linear_tc.cu": [Row("linear_tc_kernel")],
    # Seeded mutation aimed at by no_fma here: the ascent's distance or mean written with plain operators, e.g.
    # ``dx * dx + dy * dy``.
    "cg_meanshift.cu": [
        Row("quantise_kernel", no_fma=True),
        Row("ascent_kernel", "IfE", no_fma=True,
            local="spills of the float instantiation under __launch_bounds__(MS_WARPS * 32); the double one has none"),
        Row("ascent_kernel", "IdE", no_fma=True),
        Row("seed_key_kernel", "IfE"), Row("seed_key_kernel", "IdE"), Row("head_kernel", "IfE"),
        Row("head_kernel", "IdE"), Row("group_kernel", "IfE"), Row("group_kernel", "IdE"), Row("count_key_kernel"),
        Row("rank_kernel", "IfE", no_fma=True), Row("rank_kernel", "IdE", no_fma=True),
        Row("suppress_kernel", no_fma=True), Row("kept_kernel"), Row("emit_kernel", "IfE"), Row("emit_kernel", "IdE"),
    ],
    # Seeded mutation aimed at by no_fma here: occ_cast_kernel's centre distance written as
    # ``sqrt(cx * cx + cy * cy + cz * cz)`` (two fma.rn.f64; the kernel once had exactly that).
    "cg_occupancy.cu": [
        Row("occ_mark_kernel", no_fma=True),
        Row("occ_cast_kernel", no_fma=True,
            local="the ray walk's per-axis arrays, indexed by the axis it steps along (k[dim], step[dim], tmax[dim])"),
    ],
    "cg_pick.cu": [Row("seg_init_kernel"), Row("seg_stats_kernel", "ILb0E"), Row("seg_stats_kernel", "ILb1E"),
                   Row("seg_decide_kernel", no_fma=True), Row("seg_order_kernel"), Row("seg_points_kernel"),
                   Row("rank_score_kernel", no_fma=True)],
    "cg_pn2.cu": [Row("fps_kernel", "ILb0E", no_fma=True), Row("fps_kernel", "ILb1E", no_fma=True),
                  Row("fps_cluster_kernel", "ILi4EE", no_fma=True), Row("fps_cluster_kernel", "ILi8EE", no_fma=True),
                  Row("fps_cluster_kernel", "ILi16EE", no_fma=True), Row("fps_cluster_kernel", "ILi32EE", no_fma=True),
                  Row("ball_query_kernel"), Row("square_distance_kernel"), Row("index_points_kernel"),
                  Row("group_points_kernel")],
    "cg_ransac.cu": [
        Row("ransac9d_kernel", local="thread 0's 4x4 solve with row pivoting and its Jacobi sweeps index their "
                                     "matrices at run time"),
    ],
    # three_nn_kernel, offset_head_kernel and spconv_kernel use fmaf / __fmaf_rn on purpose.
    "cg_sa.cu": [Row("group_max_kernel"), Row("three_nn_kernel"), Row("three_interp_kernel")],
    "cg_sdf_build.cu": [Row("sdf_distance_kernel"), Row("sdf_crossings_kernel"), Row("sdf_parity_kernel")],
    "cg_spconv.cu": [Row("point_key_kernel"), Row("parent_key_kernel"), Row("head_kernel"), Row("emit_level_kernel"),
                     Row("nbr_kernel"), Row("pairs_kernel"),
                     Row("spconv_kernel", "ILi1EE"), Row("spconv_kernel", "ILi2EE"), Row("spconv_kernel", "ILi4EE"),
                     Row("site_key_kernel"), Row("site_run_kernel"), Row("voxel_mean_kernel", no_fma=True),
                     Row("offset_head_kernel"), Row("gather3_kernel")],
    "cg_trunk_simt.cu": [Row("trunk_simt_kernel")],
    "cg_trunk_tc.cu": [Row("trunk_tc_kernel", "ILi1EE"), Row("trunk_tc_kernel", "ILi2EE"),
                       Row("trunk_tc_kernel", "ILi3EE")],
}

Entry = collections.namedtuple("Entry", "stack spill_stores spill_loads registers notes ptx")

FMA = re.compile(r"\bfma\.rn\.f(?:32|64)\b")
SERIALISED = re.compile(r"C7517|C7519|wgmma\.mma_async instructions are serialized")


def _ptxas_records(log):
    """{entry: (stack, spill stores, spill loads, registers, notes)} of a ``ptxas -v`` log.  The numbers come from the
    entry's report, which starts at its 'Compiling entry function' line.  The notes are the other lines that name the
    entry, wherever they stand: ptxas prints its wgmma serialisation notices ahead of the report."""
    heads = list(re.finditer(r"Compiling entry function '(\S+)'", log))
    lines = log.splitlines()
    out = {}
    for m, nxt in zip(heads, heads[1:] + [None]):
        name, report = m.group(1), log[m.start():nxt.start() if nxt else len(log)]
        props = re.search(rf"Function properties for {re.escape(name)}\s*\n\s*(\d+) bytes stack frame, (\d+) bytes "
                          r"spill stores, (\d+) bytes spill loads", report)
        regs = re.search(r"Used (\d+) registers", report)
        assert props and regs, report
        notes = [x for x in lines if name in x and not re.search(r"Compiling entry function|Function properties", x)]
        out[name] = (*map(int, props.groups()), int(regs.group(1)), notes)
    return out


def _ptx_entries(ptx):
    """{entry: body} for every .entry of a PTX module."""
    starts = list(re.finditer(r"^(?:\.visible\s+|\.weak\s+)*\.entry\s+(\S+?)\s*\(", ptx, re.M))
    return {m.group(1): ptx[m.start():nxt.start() if nxt else len(ptx)] for m, nxt in zip(starts, starts[1:] + [None])}


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """{source: {mangled entry: Entry}}, every compile of every source running at once, as build.build() runs them."""
    tmp = tmp_path_factory.mktemp("codegen")
    flags = [f for f in build.NVCC_FLAGS if f != "-DCG_EXPERIMENTS"]
    def nvcc(src, mode, ext):
        return subprocess.Popen([NVCC] + flags + mode + [os.path.join(build.CSRC, src), "-o", str(tmp / (src + ext))],
                                stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    procs = {src: (nvcc(src, ["-Xptxas", "-v", "-c"], ".o"), nvcc(src, ["-ptx"], ".ptx")) for src in SOURCES}
    out = {}
    for src, (obj, ptx) in procs.items():
        log, ptx_log = obj.communicate()[0], ptx.communicate()[0]
        assert obj.returncode == 0, log
        assert ptx.returncode == 0, ptx_log
        records, bodies = _ptxas_records(log), _ptx_entries((tmp / (src + ".ptx")).read_text())
        assert set(records) == set(bodies), (src, sorted(set(records) ^ set(bodies)))
        out[src] = {e: Entry(*records[e], bodies[e]) for e in records}
    return out


def _find(entries, row):
    """The entries whose mangled name holds ``<len(name)><name><targs>`` (Itanium: an identifier follows its length,
    so bounds_kernel does not match bounds_final_kernel)."""
    key = f"{len(row.name)}{row.name}{row.targs}"
    return [e for e in entries if key in e]


def test_one_row_per_entry(compiled):
    off = []
    for src in sorted(set(compiled) | set(KERNELS)):
        own = [e for e in compiled.get(src, {}) if not e.startswith("_ZN3cub")]
        found = {row.name + row.targs: _find(own, row) for row in KERNELS.get(src, [])}
        hits = collections.Counter(e for f in found.values() for e in f)
        off += [f"{src}: row {r} names {len(f)} entries {f}" for r, f in found.items() if len(f) != 1]
        off += [f"{src}: entry {e} has {hits[e]} rows" for e in own if hits[e] != 1]
    assert not off, "\n".join(off)


@pytest.mark.parametrize("src, row", [(s, r) for s in sorted(KERNELS) for r in KERNELS[s]],
                         ids=lambda v: v if isinstance(v, str) else v.name + v.targs)
def test_entry_contract(compiled, src, row):
    found = _find(compiled[src], row)
    assert len(found) == 1, (f"{src}: {row.name}{row.targs}", found)
    e = compiled[src][found[0]]
    what = f"{src}: {row.name}{row.targs} ({found[0]})"
    if row.local is None:
        assert (e.stack, e.spill_stores, e.spill_loads) == (0, 0, 0), (
            f"{what}: {e.stack} bytes stack frame, {e.spill_stores} bytes spill stores, {e.spill_loads} bytes spill "
            f"loads at {e.registers} registers")
    if row.no_fma:
        n = len(FMA.findall(e.ptx))
        assert n == 0, f"{what}: {n} fused multiply-adds in a bit-exact kernel"
    if "wgmma.mma_async" in e.ptx:
        injected = [x for x in e.notes if SERIALISED.search(x)]
        assert not injected, f"{what}: ptxas injected wgmma waits:\n" + "\n".join(injected)
