"""METIS inputs for the reader's tests: what a file may hold in the parity domain, every refusal kind at the first
line, the last line and inside a hub line, and tokens, line ends and '%' on and around the tile boundaries of a
multi-tile file. Each case is (name, bytes); the expected result is tests/metis_oracle.py's."""
from __future__ import annotations

import numpy as np

from tests import metis_oracle as MO

TILE = 4096  # KMP_METIS_TILE_BYTES


def _ring(n: int):
    """A cycle on n >= 3 vertices as CSR."""
    u = np.arange(n)
    nb = np.stack([(u - 1) % n, (u + 1) % n], 1)
    nb.sort(1)
    return np.arange(0, 2 * n + 1, 2), nb.reshape(-1)


def _star(leaves: int):
    xadj = np.concatenate([[0, leaves], leaves + np.arange(1, leaves + 1)])
    adj = np.concatenate([np.arange(1, leaves + 1), np.zeros(leaves, np.int64)])
    return xadj, adj


def valid_cases():
    out = []
    xadj, adj = _ring(6)
    n, m = 6, 12
    rng = np.random.default_rng(7)
    vw = rng.integers(1, 9, n)
    ew = np.full(m, 3)
    # all four formats, with unit weights written explicitly (dropped) and with real weights
    out.append(("fmt0", MO.write_metis(xadj, adj)))
    out.append(("fmt1_unit", MO.write_metis(xadj, adj, adjwgt=np.ones(m))))
    out.append(("fmt10_unit", MO.write_metis(xadj, adj, vwgt=np.ones(n))))
    out.append(("fmt11_unit", MO.write_metis(xadj, adj, vwgt=np.ones(n), adjwgt=np.ones(m))))
    out.append(("fmt1", MO.write_metis(xadj, adj, adjwgt=ew)))
    out.append(("fmt10", MO.write_metis(xadj, adj, vwgt=vw)))
    out.append(("fmt11", MO.write_metis(xadj, adj, vwgt=vw, adjwgt=ew)))
    out.append(("fmt011_leading_zero", b"2 1 011\n5 2 7\n3 1 7\n"))
    out.append(("fmt_explicit_0", b"2 1 0\n2\n1\n"))
    out.append(("fmt_explicit_00", b"2 1 00\n2\n1\n"))
    # comments
    out.append(("comments", b"% a\n  % b\n%\n3 2\n% c\n2\n   % d\n1 3\n%e\n2\n% after\n%x\n"))
    out.append(("comment_only_after_spaces_extra", b"2 1\n2\n1\n  % not at column 0: extra lines\n"))
    out.append(("blank_after_last_extra", b"2 1\n2\n1\n\n"))
    out.append(("garbage_after_last", b"2 1\n2\n1\nxx\t\r-1 0 99999999999999999999\n"))
    # blank and space-only lines are isolated vertices
    out.append(("blank_lines", b"5 1\n\n   \n4\n3\n  \n"))
    out.append(("space_only_last_no_newline", b"3 1\n2\n1\n   "))
    out.append(("space_runs_leading_zeros", b"  3   2  \n  002   003  \n001\n0001    \n"))
    out.append(("no_final_newline", b"2 1 1\n2 4\n1 4"))
    out.append(("crlf_in_comment", b"%\r\n2 1\r\n"[:3] + b"2 1\n%\t\r\n2\n1\n"))
    out.append(("n0", b"0 0\n"))
    out.append(("n0_trailing", b"0 0\n% c\n"))
    out.append(("n0_extra", b"0 0\n\n"))
    out.append(("m0", b"3 0\n\n\n\n"))
    out.append(("m0_weights", b"3 0 10\n1\n2\n3\n"))
    # maximum weights and ids
    big = (1 << 31) - 2  # with the other weight 1, the total is 2^31 - 1
    out.append(("max_edge_weight", b"2 1 1\n2 %d\n1 1\n" % big))
    out.append(("max_node_weight", b"2 1 10\n%d 2\n0000000000000000000001 1\n" % big))
    far = 70000
    out.append(("max_id", b"%d 1\n%d\n" % (far, far) + b"\n" * (far - 2) + b"1\n"))
    # a star whose hub line spans many tiles
    xadj, adj = _star(1 << 17)
    out.append(("star_hub", MO.write_metis(xadj, adj)))
    out.append(("star_hub_w", MO.write_metis(xadj, adj, adjwgt=(np.arange(len(adj)) % 97) + 1)))
    # a multi-tile file shifted byte by byte: tokens, line ends and '%' fall on and around every tile boundary
    xadj, adj = _ring(900)
    rng = np.random.default_rng(3)
    body = MO.write_metis(xadj, adj, vwgt=rng.integers(1, 1000, 900), adjwgt=rng.integers(1, 30, 1800))
    lines = body.split(b"\n")
    mixed = b"\n".join(lines[:1] + [ln if i % 7 else b"% c " + ln + b"\n" + ln for i, ln in enumerate(lines[1:])])
    for shift in range(0, 40):
        out.append((f"tiles_shift{shift}", b"%" + b"x" * shift + b"\n" + mixed))
    return out


def _edit(data: bytes, at: int, new: bytes, old_len: int = 1) -> bytes:
    return data[:at] + new + data[at + old_len:]


def _target_at(data: bytes, line: int, near: int) -> int:
    """The first byte of the first target token at or after `near` on the line starting at `line` (node and edge
    weights on: tokens alternate node weight, target, weight, target, ...)."""
    j, i = 0, line
    while True:
        while data[i] == 32:
            i += 1
        if i >= near and j >= 1 and (j - 1) % 2 == 0:
            return i
        while data[i] != 32:
            i += 1
        j += 1


def refusal_cases():
    """(name, bytes, kind name) for every refusal kind."""
    out = []
    out.append(("empty", b"", "EMPTY"))
    out.append(("header_blank_first", b"\n2 1\n2\n1\n", "HEADER"))
    out.append(("header_fourth_token", b"2 1 0 5\n2\n1\n", "HEADER"))
    out.append(("header_no_newline", b"2 1", "HEADER"))
    out.append(("header_only_comments", b"% a\n% b\n", "HEADER"))
    out.append(("header_crlf", b"2 1\r\n2\n1\n", "HEADER"))
    out.append(("header_tab", b"2\t1\n2\n1\n", "HEADER"))
    out.append(("header_m_impossible", b"2 2\n2 2\n1 1\n", "HEADER"))
    out.append(("format_100", b"2 1 100\n2\n1\n", "FORMAT"))
    out.append(("format_111", b"2 1 111\n1 1 2 1\n1 1 1 1\n", "FORMAT"))
    out.append(("format_2", b"2 1 2\n2\n1\n", "FORMAT"))
    out.append(("format_huge", b"2 1 99999999999999999999999\n2\n1\n", "FORMAT"))
    out.append(("too_large_n", b"4294967296 0\n", "TOO_LARGE"))
    out.append(("too_large_m", b"100000 2147483648\n", "TOO_LARGE"))
    out.append(("too_large_before_fourth_token", b"4294967296 1 0 7\n", "TOO_LARGE"))
    # data-line kinds at the first line, the last line and inside a hub line
    xadj, adj = _ring(8)
    ring = MO.write_metis(xadj, adj, vwgt=np.arange(1, 9), adjwgt=np.full(16, 2))
    first = ring.index(b"\n") + 1
    last = ring.rindex(b"\n", 0, len(ring) - 1) + 1
    sx, sa = _star(1 << 15)
    star = MO.write_metis(sx, sa, vwgt=np.ones(len(sx) - 1) * 2, adjwgt=np.ones(len(sa)) * 3)
    hub = star.index(b"\n") + 1
    mid = hub + 100000  # inside the hub line, well past its first tiles
    while star[mid] != 32:
        mid += 1
    mid += 1  # the first byte of a token (a target or a weight)
    for where, data, at in (("first", ring, first), ("last", ring, last), ("hub", star, mid)):
        out.append((f"bad_byte_tab_{where}", _edit(data, at, b"\t", 0), "BAD_BYTE"))
        out.append((f"bad_byte_sign_{where}", _edit(data, at, b"-", 0), "BAD_BYTE"))
        # a target 0 and a target above n, written as a (target, weight) pair so the pairing stays intact
        line = data.rindex(b"\n", 0, at) + 1
        t = _target_at(data, line, at)
        out.append((f"neighbor_zero_pair_{where}", _edit(data, t, b"0 3 ", 0), "NEIGHBOR_OUT_OF_RANGE"))
        out.append((f"neighbor_above_n_pair_{where}", _edit(data, t, b"%d 3 " % (len(data) + 9), 0),
                    "NEIGHBOR_OUT_OF_RANGE"))
    # a CRLF file: the '\r' ending the first data line is its first bad byte
    out.append(("bad_byte_crlf", b"2 1\n2\r\n1\r\n", "BAD_BYTE"))
    ring_eol = ring.index(b"\n", first)
    out.append(("bad_byte_crlf_ring", _edit(ring, ring_eol, b"\r", 0), "BAD_BYTE"))
    # token-role kinds
    out.append(("missing_node_weight_first", b"2 1 10\n\n1 1\n", "MISSING_NODE_WEIGHT"))
    out.append(("missing_node_weight_last", b"2 1 10\n1 2\n   \n", "MISSING_NODE_WEIGHT"))
    out.append(("missing_node_weight_last_eof", b"2 1 10\n1 2\n   ", "MISSING_NODE_WEIGHT"))
    out.append(("missing_edge_weight_first", b"2 1 1\n2\n1 1\n", "MISSING_EDGE_WEIGHT"))
    out.append(("missing_edge_weight_last_eof", b"2 1 1\n2 1\n1", "MISSING_EDGE_WEIGHT"))
    hub_line_end = star.index(b"\n", hub)
    out.append(("missing_edge_weight_hub", _edit(star, hub_line_end - 2, b"", 2), "MISSING_EDGE_WEIGHT"))
    out.append(("zero_node_weight_first", b"2 1 10\n0 2\n1 1\n", "ZERO_WEIGHT"))
    out.append(("zero_edge_weight_last", b"2 1 1\n2 1\n1 0\n", "ZERO_WEIGHT"))
    out.append(("weight_too_large_first", b"2 1 10\n2147483648 2\n1 1\n", "WEIGHT_TOO_LARGE"))
    out.append(("weight_overflow_last", b"2 1 1\n2 1\n1 99999999999999999999999999\n", "WEIGHT_TOO_LARGE"))
    out.append(("neighbor_zero_first", b"2 1\n0\n1\n", "NEIGHBOR_OUT_OF_RANGE"))
    out.append(("neighbor_above_n_last", b"2 1\n2\n3\n", "NEIGHBOR_OUT_OF_RANGE"))
    out.append(("neighbor_overflow", b"2 1\n99999999999999999999\n1\n", "NEIGHBOR_OUT_OF_RANGE"))
    out.append(("self_loop_first", b"2 1\n1\n2\n", "SELF_LOOP"))
    out.append(("self_loop_last", b"2 1\n2\n2\n", "SELF_LOOP"))
    hub_tok = star.index(b" ", hub) + 1  # the hub's first target
    out.append(("self_loop_hub", _edit(star, hub_tok, b"1 ", 0), "SELF_LOOP"))
    out.append(("zero_weight_hub", _edit(star, mid, b"0 ", 0), "ZERO_WEIGHT"))
    big_pair = b"5 2147483648 "  # a (target, weight) pair whose weight is too large
    out.append(("weight_too_large_hub", _edit(star, _target_at(star, hub, mid), big_pair, 0), "WEIGHT_TOO_LARGE"))
    out.append(("weight_too_large_last", _edit(ring, _target_at(ring, last, last), big_pair, 0), "WEIGHT_TOO_LARGE"))
    out.append(("node_weight_too_large_hub", _edit(star, hub, b"2147483648", 1), "WEIGHT_TOO_LARGE"))
    out.append(("missing_node_weight_hub", _edit(star, hub, b"", star.index(b" ", hub) + 1 - hub), "MISSING_EDGE_WEIGHT"))
    out.append(("missing_node_weight_hub_line", star[:hub] + b"\n" + star[star.index(b"\n", hub) + 1:],
                "MISSING_NODE_WEIGHT"))
    out.append(("too_large_m_2^32", b"100000 4294967296\n", "TOO_LARGE"))
    out.append(("too_few_lines", b"3 1\n2\n1\n", "TOO_FEW_LINES"))
    out.append(("too_few_lines_comment", b"3 1\n2\n1\n% c\n", "TOO_FEW_LINES"))
    out.append(("edge_count_low", b"3 2\n2\n1\n\n", "EDGE_COUNT"))
    out.append(("edge_count_high", b"3 1\n2 3\n1\n1\n", "EDGE_COUNT"))
    out.append(("total_node_weight", b"2 1 10\n2147483647 2\n1 1\n", "TOTAL_WEIGHT"))
    out.append(("total_edge_weight", b"2 1 1\n2 2147483647\n1 1\n", "TOTAL_WEIGHT"))
    # two competing violations: the first byte wins, whatever its kind
    out.append(("compete_self_loop_before_bad", b"2 1\n1 x\n2\n", "SELF_LOOP"))
    out.append(("compete_bad_before_range", b"2 1\nx 9\n2\n", "BAD_BYTE"))
    out.append(("compete_line_before_eof_kinds", b"4 5\n2\n9\n", "NEIGHBOR_OUT_OF_RANGE"))
    out.append(("compete_weight_before_target", b"3 1 11\n0 5 1\n1 1 1\n", "ZERO_WEIGHT"))
    return out


def cases():
    """Every case as (name, bytes)."""
    return valid_cases() + [(name, data) for name, data, _ in refusal_cases()]
