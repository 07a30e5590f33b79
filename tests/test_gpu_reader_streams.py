"""GPU: the readers of device bytes wait for torch's current stream. A zeroed tensor is filled with a valid file's
bytes on a non-default torch stream, behind a sleep of about 50 ms, and the parser is called while that stream is
current, with no host synchronisation in between: the graph must be the file's, as the oracle reads it.
  parse_metis_device; parse_parhip_device in the natural and the external ordering; parse_parhip_prepared"""
import numpy as np
import pytest

from kaminpar_b200 import lp
from kaminpar_b200 import metis as ME
from kaminpar_b200 import parhip as PH
from kaminpar_b200.graph import random_weights, rmat
from tests import metis_oracle as MO
from tests import parhip_oracle as PO

pytestmark = pytest.mark.gpu
SLEEP_CYCLES = 100_000_000  # about 50 ms at the H100's clocks


@pytest.fixture(scope="module")
def handle():
    h = lp.LPHandle(lp._cluster_config(lp.LabelPropagationCoarseningContext(), lp.EngineContext()))
    yield h
    h.close()


@pytest.fixture(scope="module")
def graph():
    return random_weights(rmat(10, 8, seed=5), seed=5, max_vwgt=9, max_adjwgt=9)


def parse_late(data: bytes, parse):
    """parse(tensor) on a zeroed tensor that torch's current stream fills with `data` after the sleep."""
    import torch

    src = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    dst = torch.zeros_like(src)
    torch.cuda.synchronize()  # src and the zeros are in place; from here on nothing waits on the host
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        dst.copy_(src)
        return parse(dst)


def same(got, expect, fields):
    for f, a in zip(fields, got):
        assert (a is None) == (expect[f] is None), f
        if a is not None:
            assert np.array_equal(np.asarray(a, np.int64), np.asarray(expect[f], np.int64)), f


def test_parse_metis_device_waits(handle, graph):
    data = MO.write_metis(graph.xadj, graph.adjncy, graph.vwgt, graph.adjwgt)
    expect = MO.parse(data)
    assert expect["kind"] == 0
    g = parse_late(data, lambda t: ME.parse_metis_device(handle, t))
    assert MO.as_dict(g.report) == MO.report_of(expect)
    c = g.get()
    same((c.xadj, c.adjncy, c.vwgt, c.adjwgt), expect, ("xadj", "adjncy", "vwgt", "adjwgt"))
    g.close()


@pytest.mark.parametrize("ordering", [PO.NATURAL, PO.EXTERNAL])
def test_parse_parhip_device_waits(handle, graph, ordering):
    data = PO.write(graph.xadj, graph.adjncy, graph.vwgt, graph.adjwgt)
    expect = PO.read(data, ordering)
    assert expect["kind"] == 0
    g = parse_late(data, lambda t: PH.parse_parhip_device(handle, t, ordering))
    assert PO.as_dict(g.report) == PO.report_of(expect)
    c = g.get()
    same((c.xadj, c.adjncy, c.vwgt, c.adjwgt, g.old_to_new()), expect,
         ("xadj", "adjncy", "vwgt", "adjwgt", "old_to_new"))
    g.close()


def test_parse_parhip_prepared_waits(handle, graph):
    data = PO.write(graph.xadj, graph.adjncy, graph.vwgt, graph.adjwgt)
    expect = PO.read(data, PO.EXTERNAL)
    pg = parse_late(data, lambda t: PH.parse_parhip_prepared(handle, t))
    assert PO.as_dict(pg.report) == PO.report_of(expect)
    same(pg._download(), expect, ("xadj", "adjncy", "vwgt", "adjwgt", "old_to_new"))
    pg.close()
