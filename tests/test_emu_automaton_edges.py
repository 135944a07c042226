"""Edges of the automaton on the CPU emulation of the lane logic (tests/emu), against the oracle:

  * the double-array layouts of test_gpu_automaton_edges.py (num_free_blocks 1 against 16, every kernel, staged
    records or none, forced segments);
  * every (state, byte) transition of the compact image for num_free_blocks 1, 2 and 3 and hot regions of 0, 256
    and 65 536 slots;
  * one find_overlapping scan at each 2^24-edge automaton: a relaid-out image whose new ids reach 2^24 - 1, the
    largest compact image (2^24 slots, no region), the smallest automaton without one, and both sides of the charwise
    limit.  Each call rebuilds the image from the wire (about 15 s at this size), so there are only five."""
import numpy as np
import pytest

import emu_api as E
import oracle_api as O
from cases import filler_case, layout_cases, layout_params, nul_heavy_case

ORC = {0: O.FIND, 1: O.FIND_OVERLAPPING, 2: O.FIND_OVERLAPPING_NO_SUFFIX, 3: O.LEFTMOST_FIND}
LAYOUT_CASES = layout_cases()
G24 = 1 << 24


def _runs(cw, kind, mode):
    if cw or kind:
        return [dict(kernel=0), dict(kernel=1)]
    runs = [dict(kernel=k) for k in (0, 1, 2, 4)] + [dict(kernel=3, hot_n=h) for h in (0, 6144)]
    return runs + ([dict(kernel=3, hot_n=6144, seg_len=64)] if mode in (1, 2) else [])


@pytest.mark.parametrize("case,nfb", layout_params(LAYOUT_CASES),
                         ids=["%s-nfb%d" % (LAYOUT_CASES[i][0], k) for i, k in layout_params(LAYOUT_CASES)])
def test_layouts_on_the_emulated_lanes(case, nfb):
    name, pats, cw, kind, text, offs = LAYOUT_CASES[case]
    offs = offs[:121]  # the first 120 haystacks: the emulation is slow
    pma = O.OraclePma.build(pats, charwise=cw, match_kind=kind, num_free_blocks=nfb)
    if nfb == 1 and not cw:  # the charwise arrays keep their size and move states (layout_params checks they differ)
        assert pma.num_elements() > O.OraclePma.build(pats, charwise=cw, match_kind=kind).num_elements(), name
    wire = pma.serialize()
    if not cw:
        assert E.check_image_transitions(wire, 65536)[0] == 0, name
    for mode in ((3,) if kind else (0, 1, 2)):
        ref = pma.scan_batch(ORC[mode], text, offs, want_matches=True)
        for kw in _runs(cw, kind, mode):
            rc, m, oo, need = E.scan(wire, cw, mode, text, offs, **kw)
            assert rc == 0 and need == ref["total"], (name, nfb, mode, kw)
            assert m.tobytes() == ref["matches"].tobytes(), (name, nfb, mode, kw)


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("nfb", [1, 2, 3])
def test_image_transitions_for_every_layout_and_region(kind, nfb):
    pats, _, _ = nul_heavy_case(kind, n_patterns=20000, n_hay=1)
    wire = O.OraclePma.build(pats, match_kind=kind, num_free_blocks=nfb).serialize()
    n = O.OraclePma.build(pats, match_kind=kind, num_free_blocks=nfb).num_elements()
    assert n > 52000
    for hot in (0, 256, 65536):
        bad, hs, used = E.check_image_transitions(wire, hot)
        assert bad == 0, (nfb, hot, bad)
        assert hs == min(hot, (n + 255) & ~255), (nfb, hot, hs)


EDGE = [("bytewise-a", G24 - 65536, False), ("bytewise-b", G24, False), ("bytewise-c", G24 + 256, False),
        ("charwise-compact", G24 - 256, True), ("charwise-wide", G24, True)]


@pytest.mark.parametrize("name,slots,cw", EDGE, ids=[e[0] for e in EDGE])
def test_find_overlapping_at_the_2_pow_24_edge(name, slots, cw):
    pats, text, offs = filler_case(slots, cw)
    pma = O.OraclePma.build(pats, charwise=cw)
    del pats
    assert pma.num_elements() == slots
    ref = pma.scan_batch(O.FIND_OVERLAPPING, text, offs, want_matches=True)
    assert ref["total"] > 0
    kw = dict(kernel=1) if cw else dict(kernel=3, hot_n=6144)
    rc, m, oo, need = E.scan(pma.serialize(), cw, 1, text, offs, **kw)
    assert rc == 0 and need == ref["total"], name
    assert m.tobytes() == ref["matches"].tobytes(), name
