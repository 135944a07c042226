"""Per-pattern histograms (dach_dev_hist_batch) on the kernels' lane logic compiled for the CPU (tests/emu_hist), against
the oracle's match lists.  No GPU needed; tests/test_gpu_hist.py runs the same checks on the device."""
import json
import os

import numpy as np
import pytest

import emu_hist_api as H
import emu_reduce_api as ER
import oracle_api as O
from cases import hand_made_case, mixed_width_case

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "search_tests.json"), encoding="utf-8"))
MODE = {"find_iter": 0, "find_overlapping_iter": 1, "find_overlapping_no_suffix_iter": 2, "leftmost_find_iter": 3}
ORC_MODE = {0: O.FIND, 1: O.FIND_OVERLAPPING, 2: O.FIND_OVERLAPPING_NO_SUFFIX, 3: O.LEFTMOST_FIND}
# (hot records, kernel option, hist_smem)
CONFIGS = ((0, 3, 1024), (256, 3, 0), (1 << 16, 3, 3), (0, 1, 1024), (0, 2, 1 << 20), (0, 4, 0), (0, 0, 1024))


def value_hist(pma, mode, text, offs, n_hist=None):
    """bincount of the values of the oracle's matches"""
    ref = pma.scan_batch(ORC_MODE[mode], text, offs, want_matches=True)
    v = ref["matches"]["value"].astype(np.int64)
    return np.bincount(v, minlength=n_hist or 0).astype(np.uint64), int(ref["counts"].sum())


def records(wire, cw):
    return ER.image_outputs(wire, cw)


def expected(patterns, cw, kind, mode, text, offs, values=None):
    """(value-keyed, output-keyed histogram, total) from the oracle.  The output key comes from a twin automaton of the
    same patterns whose value is the pattern index: its records sit where the original's do."""
    pma = O.OraclePma.build(patterns, charwise=cw, match_kind=kind, values=values)
    recs = records(pma.serialize(), cw)
    nv = int(recs[:, 0].max()) + 1 if len(recs) else 0
    vh, total = value_hist(pma, mode, text, offs, nv)
    twin = O.OraclePma.build(patterns, charwise=cw, match_kind=kind)
    trecs = records(twin.serialize(), cw)
    assert np.array_equal(trecs[:, 1:3], recs[:, 1:3])
    ph, _ = value_hist(twin, mode, text, offs, len(patterns))
    oh = ph[trecs[:, 0].astype(np.int64)] if len(trecs) else np.zeros(0, np.uint64)
    return vh, oh, total, pma


def check(patterns, cw, kind, mode, text, offs, values=None, configs=CONFIGS, **kw):
    vh, oh, total, pma = expected(patterns, cw, kind, mode, text, offs, values)
    wire = pma.serialize()
    for hot, kernel, hs in configs:
        for key, want in (("value", vh), ("output", oh)):
            rc, got, tot, which = H.hist(wire, cw, mode, key, text, offs, len(want), hot_n=hot, kernel=kernel, hist_smem=hs, **kw)
            assert rc == 0
            assert np.array_equal(got, want), (mode, key, hot, kernel, hs, kw)
            assert tot == total == int(want.sum())
            if mode != 1:
                assert not which & 8  # only find_overlapping on a lane machine expands parent chains
    return vh, oh


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
    hay = t["haystack"].encode()
    text = np.frombuffer(hay, dtype=np.uint8)
    check(t["patterns"], cw, O.KIND[kind], MODE[iterator], text, np.array([0, len(hay)], dtype=np.uint64))


def _batch(rng, alpha, n, maxlen):
    hays = [bytes(rng.integers(97, 97 + alpha + 1, size=int(rng.integers(0, maxlen))).tolist()) for _ in range(n)]
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    return np.frombuffer(b"".join(hays), dtype=np.uint8), offs


def rand_patterns(rng, n, alpha, maxlen, allow_empty=False):
    return [bytes(rng.integers(97, 97 + alpha, size=int(rng.integers(0 if allow_empty else 1, maxlen + 1))).tolist())
            for _ in range(n)]


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_duplicates_values_and_the_empty_pattern(seed, kind):
    """Duplicate patterns (equal and distinct values), an empty pattern, values shared by different patterns;
    LeftmostFirst drops patterns that extend a shorter one."""
    rng = np.random.default_rng(7100 + 10 * seed + kind)
    alpha = int(rng.integers(2, 4))
    pats = rand_patterns(rng, int(rng.integers(5, 40)), alpha, 5, allow_empty=seed < 2)
    pats = pats + pats[: len(pats) // 3]  # duplicates
    values = None if seed == 0 else rng.integers(0, 2 * len(pats) if seed == 1 else 6, size=len(pats)).tolist()
    text, offs = _batch(rng, alpha, 30, 90)
    for mode in ([3] if kind else [0, 1, 2]):
        check(pats, False, kind, mode, text, offs, values=values)


def test_leftmost_first_drops_extensions():
    pats = [b"ab", b"abc", b"abcd", b"b", b"bc"]
    pma = O.OraclePma.build(pats, match_kind=2)
    assert len(records(pma.serialize(), False)) < len(pats)
    text = np.frombuffer(b"abcdxabcbcab", dtype=np.uint8)
    vh, oh = check(pats, False, 2, 3, text, np.array([0, text.size], dtype=np.uint64))
    assert vh.sum() > 0


@pytest.mark.parametrize("seed", range(4))
def test_segments_count_a_straddling_match_once(seed):
    rng = np.random.default_rng(1500 + seed)
    alpha = int(rng.integers(2, 4))
    pats = rand_patterns(rng, int(rng.integers(1, 50)), alpha, 9, allow_empty=(seed == 0))
    lens = list(rng.integers(0, 400, size=20)) + [0, 64, 128, 1, 63, 65]
    hays = [bytes(rng.integers(97, 97 + alpha + 1, size=int(L)).tolist()) for L in lens]
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    text = np.frombuffer(b"".join(hays), dtype=np.uint8)
    for mode in (1, 2):
        for seg_len in (1, 3, 16, 100):
            check(pats, False, 0, mode, text, offs, configs=((256, 3, 1024), (0, 3, 0)), seg_len=seg_len)


@pytest.mark.parametrize("seed", range(0, 45, 4))
def test_charwise_mixed_width_chars(seed):
    kind, pats, text, offs = mixed_width_case(seed)
    for mode in ([3] if kind else [0, 1, 2]):
        check(pats, True, kind, mode, text, offs, configs=((0, 3, 1024), (0, 3, 0), (0, 0, 0)))


def test_hand_made_automaton():
    wire, text, offs = hand_made_case(hay_len=3000)
    pma, _ = O.OraclePma.deserialize(wire)
    recs = records(wire, False)
    assert len(set(recs[:, 0].tolist())) == len(recs)  # unique values: the output key is the value key re-indexed
    for mode in (0, 1, 2):
        vh, total = value_hist(pma, mode, text, offs, int(recs[:, 0].max()) + 1)
        for key, want in (("value", vh), ("output", vh[recs[:, 0].astype(np.int64)])):
            for hs in (0, 64, 1 << 20):
                rc, got, tot, _ = H.hist(wire, False, mode, key, text, offs, len(want), seg_len=256, hist_smem=hs)
                assert rc == 0 and np.array_equal(got, want) and tot == total


@pytest.mark.parametrize("hot_slots", [0, 256, 65536])
def test_hist_smem_sizes_and_hot_regions(hot_slots):
    rng = np.random.default_rng(88 + hot_slots)
    pats = sorted(set(rand_patterns(rng, 1200, 5, 8)))
    text, offs = _batch(rng, 5, 16, 600)
    H.lib().emu_hist_set_hot_slots(hot_slots)
    try:
        for mode in (0, 1, 2):
            check(pats, False, 0, mode, text, offs, configs=[(256, 3, hs) for hs in (0, 1, 7, 256, 4096, 1 << 24)])
    finally:
        H.lib().emu_hist_set_hot_slots(65536)


def test_accumulates_across_batches():
    """A then B into one histogram == A ++ B; the total equals the COUNT total."""
    rng = np.random.default_rng(4242)
    pats = rand_patterns(rng, 40, 3, 6)
    pma = O.OraclePma.build(pats)
    wire = pma.serialize()
    text, offs = _batch(rng, 3, 40, 200)
    k = 17
    a_t, a_o = text[: int(offs[k])], offs[: k + 1]
    b_t, b_o = text[int(offs[k]):], offs[k:] - offs[k]
    for mode in (0, 1, 2):
        for key in ("value", "output"):
            n_hist = len(pats)
            rc, whole, tot, _ = H.hist(wire, False, mode, key, text, offs, n_hist)
            assert rc == 0
            acc = np.zeros(n_hist, dtype=np.uint64)
            rc1, _, t1, _ = H.hist(wire, False, mode, key, a_t, a_o, n_hist, out=acc)
            rc2, _, t2, _ = H.hist(wire, False, mode, key, b_t, b_o, n_hist, out=acc)
            assert rc1 == rc2 == 0 and np.array_equal(acc, whole) and t1 + t2 == tot
            rc, counts, ctot = ER.reduce(wire, False, mode, 1, text, offs)
            assert rc == 0 and ctot == tot == int(whole.sum())


def test_errors_and_empty_batches():
    pma = O.OraclePma.build([b"a", b"ab", b"a"], values=[3, 9, 3])
    wire = pma.serialize()
    text = np.frombuffer(b"aab", dtype=np.uint8)
    offs = np.array([0, 3], dtype=np.uint64)
    assert H.hist(wire, False, 1, "value", text, offs, 10)[0] == 0
    assert H.hist(wire, False, 1, "value", text, offs, 9)[0] == 1  # n_hist must exceed the largest value
    assert H.hist(wire, False, 1, "output", text, offs, 3)[0] == 0
    assert H.hist(wire, False, 1, "output", text, offs, 2)[0] == 1  # ... or hold every output record
    assert H.hist(wire, False, 3, "value", text, offs, 10)[0] == 5  # DACH_MATCH_KIND_MISMATCH
    rc, h, tot, _ = H.hist(wire, False, 1, "value", np.zeros(0, np.uint8), np.zeros(1, np.uint64), 10)
    assert rc == 0 and tot == 0 and not h.any()
    rc, h, tot, _ = H.hist(wire, False, 1, "value", np.zeros(0, np.uint8), np.zeros(3, np.uint64), 10)
    assert rc == 0 and tot == 0 and not h.any()
