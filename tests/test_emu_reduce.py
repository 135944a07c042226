"""Counts and first matches (dach_dev_count_batch / dach_dev_first_batch) on the kernels' lane logic compiled for the
CPU (tests/emu_reduce), against the oracle.  No GPU needed; tests/test_gpu_reduce.py runs the same checks on the device."""
import json
import os

import numpy as np
import pytest

import emu_reduce_api as E
import oracle_api as O
from cases import hand_made_case, mixed_width_case

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "search_tests.json"), encoding="utf-8"))
MODE = {"find_iter": 0, "find_overlapping_iter": 1, "find_overlapping_no_suffix_iter": 2, "leftmost_find_iter": 3}
ORC_MODE = {0: O.FIND, 1: O.FIND_OVERLAPPING, 2: O.FIND_OVERLAPPING_NO_SUFFIX, 3: O.LEFTMOST_FIND}
COUNT, FIRST = 1, 2
NONE = np.array([(0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF)], dtype=E.MATCH_DTYPE)[0]


def expected(pma, mode, text, offs):
    """(counts, first tuples, found) of iterator `mode` from the oracle's full match list."""
    ref = pma.scan_batch(ORC_MODE[mode], text, offs, want_matches=True)
    counts = ref["counts"].astype(np.uint64)
    n = len(offs) - 1
    first = np.zeros(n, dtype=E.MATCH_DTYPE)
    first[:] = NONE
    starts = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    found = counts > 0
    first[found] = ref["matches"][starts[:-1][found]]
    return counts, first, found


def check(wire, cw, mode, text, offs, pma, **kw):
    counts, first, found = expected(pma, mode, text, offs)
    rc, got, total = E.reduce(wire, cw, mode, COUNT, text, offs, **kw)
    assert rc == 0
    assert np.array_equal(got, counts), (mode, kw)
    assert total == int(counts.sum())
    rc, (gf, gfound), nf = E.reduce(wire, cw, mode, FIRST, text, offs, **kw)
    assert rc == 0
    assert np.array_equal(gfound, found), (mode, kw)
    assert gf.tobytes() == first.tobytes(), (mode, kw)
    assert nf == int(found.sum())


CONFIGS = ((0, 3), (256, 3), (1 << 16, 3), (0, 1), (0, 2), (0, 4), (0, 0))


def _cases():
    for variant, iterator, coll, kind in GOLD["configs"]:
        if iterator not in MODE:
            continue
        for g in GOLD["collections"][coll]:
            for t in GOLD["groups"][g]:
                yield pytest.param(variant, iterator, kind, t, id="%s-%s-%s-%s" % (variant, iterator, kind, t["name"]))


@pytest.mark.parametrize("variant,iterator,kind,t", list(_cases()))
def test_golden_vectors(variant, iterator, kind, t):
    cw = variant == "charwise"
    pma = O.OraclePma.build(t["patterns"], charwise=cw, match_kind=O.KIND[kind])
    wire = pma.serialize()
    hay = t["haystack"].encode()
    text = np.frombuffer(hay, dtype=np.uint8)
    offs = np.array([0, len(hay)], dtype=np.uint64)
    for hot, kernel in CONFIGS:
        check(wire, cw, MODE[iterator], text, offs, pma, hot_n=hot, kernel=kernel)


def rand_patterns(rng, n, alpha, maxlen, allow_empty=False):
    return [bytes(rng.integers(97, 97 + alpha, size=int(rng.integers(0 if allow_empty else 1, maxlen + 1))).tolist())
            for _ in range(n)]


def _batch(rng, alpha, n, maxlen):
    hays = [bytes(rng.integers(97, 97 + alpha + 1, size=int(rng.integers(0, maxlen))).tolist()) for _ in range(n)]
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    return np.frombuffer(b"".join(hays), dtype=np.uint8), offs


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("kind", [0, 1, 2])
@pytest.mark.parametrize("cw", [False, True])
def test_random_batches(seed, kind, cw):
    rng = np.random.default_rng(900 + 100 * seed + 10 * kind + cw)
    alpha = int(rng.integers(2, 5))
    pats = rand_patterns(rng, int(rng.integers(1, 60)), alpha, 7, allow_empty=(seed == 0))
    if cw:
        table = ["a", "b", "é", "あ", "𝄞"]
        pats = ["".join(table[b - 97] for b in p) for p in pats]
        syms = [table[i] for i in range(alpha)] + ["z"]
        hays = ["".join(syms[int(i)] for i in rng.integers(0, len(syms), size=int(rng.integers(0, 120)))).encode() for _ in range(25)]
        offs = np.zeros(26, dtype=np.uint64)
        offs[1:] = np.cumsum([len(h) for h in hays])
        text = np.frombuffer(b"".join(hays), dtype=np.uint8)
    else:
        text, offs = _batch(rng, alpha, 25, 120)
    pma = O.OraclePma.build(pats, charwise=cw, match_kind=kind)
    wire = pma.serialize()
    for mode in ([3] if kind else [0, 1, 2]):
        for hot, kernel in CONFIGS:
            check(wire, cw, mode, text, offs, pma, hot_n=hot, kernel=kernel)


@pytest.mark.parametrize("seed", range(45))
def test_charwise_mixed_width_chars(seed):
    kind, pats, text, offs = mixed_width_case(seed)
    pma = O.OraclePma.build(pats, charwise=True, match_kind=kind)
    for mode in ([3] if kind else [0, 1, 2]):
        for kernel in (3, 0):
            check(pma.serialize(), True, mode, text, offs, pma, kernel=kernel)


@pytest.mark.parametrize("seed", range(5))
def test_segments_and_tails(seed):
    """Forced small segments: counts are summed over a haystack's segments, the first match is the one of its lowest
    segment that has one; warm-up events never count."""
    rng = np.random.default_rng(1400 + seed)
    alpha = int(rng.integers(2, 5))
    pats = rand_patterns(rng, int(rng.integers(1, 60)), alpha, 9, allow_empty=(seed == 0))
    pma = O.OraclePma.build(pats)
    wire = pma.serialize()
    lens = list(rng.integers(0, 400, size=30)) + [0, 64, 128, 1, 63, 65]
    hays = [bytes(rng.integers(97, 97 + alpha + 1, size=int(L)).tolist()) for L in lens]
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    text = np.frombuffer(b"".join(hays), dtype=np.uint8)
    for mode in (0, 1, 2):
        for seg_len in (1, 3, 16, 64, 100, 1000):
            check(wire, False, mode, text, offs, pma, seg_len=seg_len, hot_n=256)


def test_hand_made_case_is_scanned_whole():
    wire, text, offs = hand_made_case(hay_len=6000)
    pma, _ = O.OraclePma.deserialize(wire)
    assert E.image_segmentable(wire) == 0
    for mode in (1, 2):
        check(wire, False, mode, text, offs, pma)


@pytest.mark.parametrize("hot_slots", [0, 256, 4096, 65536])
def test_hot_region_sizes(hot_slots):
    rng = np.random.default_rng(77 + hot_slots)
    pats = sorted(set(rand_patterns(rng, 1500, 6, 9)))
    E.lib().emu_set_hot_slots(hot_slots)
    try:
        for kind in (0, 1):
            pma = O.OraclePma.build(pats, match_kind=kind)
            text, offs = _batch(rng, 6, 12, 700)
            for mode in ([3] if kind else [0, 1, 2]):
                for hot in (0, 256, 1 << 16):
                    check(pma.serialize(), False, mode, text, offs, pma, hot_n=hot)
    finally:
        E.lib().emu_set_hot_slots(65536)


@pytest.mark.parametrize("cw", [False, True])
@pytest.mark.parametrize("seed", range(12))
def test_standard_modes_have_one_first_match(seed, cw):
    """find_iter, find_overlapping_iter and find_overlapping_no_suffix_iter report the same first match -- which is
    why FIRST serves all three with the find_overlapping machine."""
    rng = np.random.default_rng(3100 + seed)
    alpha = int(rng.integers(1, 5))
    pats = rand_patterns(rng, int(rng.integers(1, 40)), alpha, 6, allow_empty=(seed % 4 == 0))
    if cw:
        pats = [p.decode() for p in pats]
    pma = O.OraclePma.build(pats, charwise=cw)
    text, offs = _batch(rng, alpha, 40, 60)
    firsts = [expected(pma, mode, text, offs)[1:] for mode in (0, 1, 2)]
    for f, found in firsts[1:]:
        assert f.tobytes() == firsts[0][0].tobytes() and np.array_equal(found, firsts[0][1])
    for t in GOLD["groups"].values():
        for case in t:
            p = O.OraclePma.build(case["patterns"])
            hay = np.frombuffer(case["haystack"].encode(), dtype=np.uint8)
            o = np.array([0, hay.size], dtype=np.uint64)
            got = [expected(p, mode, hay, o)[1].tobytes() for mode in (0, 1, 2)]
            assert got[0] == got[1] == got[2], case["name"]


@pytest.mark.parametrize("cw", [False, True])
def test_chain_word_is_the_list_length(cw):
    rng = np.random.default_rng(12 + cw)
    pats = sorted(set(rand_patterns(rng, 3000, 3, 12, allow_empty=True)))
    if cw:
        pats = [p.decode() for p in pats]
    out = E.image_outputs(O.OraclePma.build(pats, charwise=cw).serialize(), cw)
    assert len(out) == len(pats)
    for i in range(len(out)):
        k, j = 0, i + 1
        while j:
            k += 1
            j = int(out[j - 1, 2])
        assert out[i, 3] == k


def test_first_stops_early():
    """4 KiB haystacks that each match within their first 16 bytes: FIRST steps a small share of what COUNT steps."""
    rng = np.random.default_rng(5)
    pats = [b"needle", b"xyz"]
    pma = O.OraclePma.build(pats)
    wire = pma.serialize()
    hays = []
    for _ in range(64):
        h = bytearray(rng.integers(97, 100, size=4096).astype(np.uint8).tobytes())
        at = int(rng.integers(0, 10))
        h[at: at + 6] = b"needle"
        hays.append(bytes(h))
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    text = np.frombuffer(b"".join(hays), dtype=np.uint8)
    steps = {}
    for rk in (COUNT, FIRST):
        E.stats(reset=True)
        assert E.reduce(wire, False, 1, rk, text, offs)[0] == 0
        steps[rk] = E.stats(reset=True)["steps"]
    assert steps[COUNT] >= 64 * 4096
    assert steps[FIRST] < 0.05 * steps[COUNT], steps
    check(wire, False, 1, text, offs, pma)


def test_empty_batch_empty_haystacks_and_the_empty_pattern():
    pma = O.OraclePma.build(["", "ab", "é"], charwise=True)
    wire = pma.serialize()
    rc, c, tot = E.reduce(wire, True, 0, COUNT, np.zeros(0, np.uint8), np.zeros(1, np.uint64))
    assert rc == 0 and len(c) == 0 and tot == 0
    hays = ["", "xab", "éé", ""]
    data = [h.encode() for h in hays]
    offs = np.zeros(5, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in data])
    text = np.frombuffer(b"".join(data), dtype=np.uint8)
    rc, c, tot = E.reduce(wire, True, 0, COUNT, text, offs, kernel=0)
    assert rc == 0 and list(c) == [len(h) + 1 for h in hays]  # find with an empty pattern: chars + 1
    check(wire, True, 0, text, offs, pma)
    wire_l = O.OraclePma.build(["a"], match_kind=1).serialize()
    assert E.reduce(wire_l, False, 1, COUNT, text, offs)[0] == 5  # DACH_MATCH_KIND_MISMATCH
