"""GPU tests (-m gpu): the tensor-core trunk's max-pool keys do not depend on how its persistent grid cuts the batch,
at the edges of the 256-point tiles of engine 3.

Engine 3 runs 256-point tiles and engines 1 and 2 128-point tiles.  N = 255, 256, 257 put a candidate's last tile one
point short of, exactly at and one point past a 256-point edge; N = 511 makes B x ntiles odd, so that the balanced
ranges of a 133-candidate batch cut candidates at every other tile.  The comparisons are those of
test_trunk_partition.py.
"""
import pytest
import torch

from test_trunk_partition import (TC_ENGINES, assert_alone_equal, assert_rows_equal, cuda, make_inputs,  # noqa: F401
                                  nets, probe, rows, scene)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("src", ["ids", "x"])
@pytest.mark.parametrize("N", [255, 256, 257, 511])
@pytest.mark.parametrize("engine", TC_ENGINES)
def test_keys_do_not_depend_on_the_cut_at_tile_edges(nets, scene, engine, N, src):
    net = nets[src]
    net.ctx.set_engine(engine)
    B = 133
    inp = make_inputs(src, B, N, seed=N * 7 + engine)
    full = probe(net, scene, src, inp)
    for lo, hi in [(0, 64), (64, B), (5, 69), (69, B), (1, 132)]:
        sel = torch.arange(lo, hi, device="cuda")
        assert_rows_equal(full, sel, probe(net, scene, src, rows(inp, sel)), f"rows {lo}:{hi}")
    for b in (0, 1, 66, 131, 132):
        sel = torch.full((64,), b, device="cuda")
        assert_rows_equal(full, sel, probe(net, scene, src, rows(inp, sel)), f"64 x row {b}")
        one = probe(net, scene, src, rows(inp, torch.tensor([b], device="cuda")))
        assert_alone_equal(full, b, one, "alone")
    net.ctx.set_engine(3)
