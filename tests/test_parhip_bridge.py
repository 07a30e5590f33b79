"""The ParHIP oracle (tests/parhip_oracle.py) against the unmodified reference's read_graph in all four orderings
(tests/parhip_bridge.py): the arrays, sorted() and the external ordering's permutation equal the reference's bit for
bit on the 32-bit corpus, and every 64-bit file, which the oracle reads as its 32-bit twin, makes the reference's
32-bit build exit with status 1 after the log line of ParHIPHeader::validate for that width. Checked against the live reference where
oracle/_ref/parhip_read was built, and always against its verdicts pinned in tests/golden/parhip_cases.npz."""
import numpy as np
import pytest

from tests import parhip_bridge as PB
from tests import parhip_oracle as PO

CASES = PB.corpus()
FIELDS = ("xadj", "adjncy", "vwgt", "adjwgt", "old_to_new")


def same(a, b) -> bool:
    """Equal arrays; an absent array equals an empty one (the reference cannot tell them apart)."""
    a = np.zeros(0, np.int64) if a is None else np.asarray(a).astype(np.int64)
    b = np.zeros(0, np.int64) if b is None else np.asarray(b).astype(np.int64)
    return np.array_equal(a, b)


def golden(name, o):
    z = np.load(PB.GOLDEN)
    key = f"{name}__{o}"
    out = dict(exit=int(z[key + "__exit"][0]))
    if out["exit"] != 0:
        out["log"] = str(z[key + "__log"][0])
    if out["exit"] == 0:
        out["sorted"] = int(z[key + "__sorted"][0])
        for f in FIELDS:
            out[f] = z[key + "__" + f] if key + "__" + f in z.files else None
    return out


@pytest.mark.parametrize("name,data", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("ordering", [0, 1, 2, 3])
def test_oracle_equals_reference(name, data, ordering):
    ref = golden(name, ordering)
    live = PB.run(data, ordering)
    if live is not None:
        assert live["exit"] == ref["exit"] and live.get("log") == ref.get("log")
        for f in FIELDS:
            if ref["exit"] == 0:
                assert same(live[f], ref[f]), f
    ours = PO.read(data, ordering)
    assert ours["kind"] == 0
    if "_64" in name:  # std::exit(1) after validate's line for the first 64-bit width it meets
        what = {"offsets": "edge IDs", "vwgt": "node weights", "adjwgt": "edge weights"}.get(name.split("_64")[1],
                                                                                           "node IDs")
        assert ref["exit"] == 1 and ref["log"] == f"[Error] The stored graph uses 64-Bit {what} but this build uses " \
                                                  f"32-Bit {what}.", ref
        twin = PO.read(dict(CASES)[name.split("_64")[0]], ordering)
        for f in FIELDS:
            assert (ours[f] is None) == (twin[f] is None) and same(ours[f], twin[f]), f
        return
    assert ref["exit"] == 0 and ours["sorted"] == ref["sorted"]
    for f in FIELDS:
        assert same(ours[f], ref[f]), f
        if ref[f] is None:  # absent in the reference: absent in the oracle, or a section of no entries
            assert ours[f] is None or len(ours[f]) == 0, f
