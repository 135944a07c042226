"""Per-pattern document frequencies (dach_dev_df_batch) on the kernels' lane logic compiled for the CPU (tests/emu_df),
against the oracle's per-haystack match lists: np.unique of the (haystack, key) pairs, then a bincount.  No GPU needed;
tests/test_gpu_df.py runs the same checks on the device."""
import json
import os

import numpy as np
import pytest

import emu_df_api as F
import emu_reduce_api as ER
import oracle_api as O
from cases import hand_made_case, mixed_width_case

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "search_tests.json"), encoding="utf-8"))
MODE = {"find_iter": 0, "find_overlapping_iter": 1, "find_overlapping_no_suffix_iter": 2, "leftmost_find_iter": 3}
ORC_MODE = {0: O.FIND, 1: O.FIND_OVERLAPPING, 2: O.FIND_OVERLAPPING_NO_SUFFIX, 3: O.LEFTMOST_FIND}
# (hot records, kernel option, df_pairs): 1 is raised to the smallest table one haystack always fits in
CONFIGS = ((0, 3, 1 << 16), (256, 3, 1), (0, 1, 1 << 16), (0, 2, 1), (0, 4, 1 << 16), (0, 0, 1 << 16), (0, 0, 1))
OVERFLOW = 6  # DACH_OUTPUT_OVERFLOW


def doc_freq(hay, keys, n_keys):
    """haystacks per key: np.unique of the (haystack, key) pairs, then a bincount"""
    pairs = np.unique((hay.astype(np.uint64) << np.uint64(32)) | keys.astype(np.uint64))
    return np.bincount((pairs & np.uint64(0xffffffff)).astype(np.int64), minlength=n_keys).astype(np.uint64)


def per_match(pma, mode, text, offs):
    """(haystack index, value) of every match the oracle reports"""
    ref = pma.scan_batch(ORC_MODE[mode], text, offs, want_matches=True)
    hay = np.repeat(np.arange(len(offs) - 1), ref["counts"].astype(np.int64))
    return hay, ref["matches"]["value"].astype(np.int64)


def expected(patterns, cw, kind, mode, text, offs, values=None):
    """(value-keyed DF, output-keyed DF, value-keyed histogram) from the oracle.  The output key comes from a twin
    automaton of the same patterns whose value is the pattern index: its records sit where the original's do."""
    pma = O.OraclePma.build(patterns, charwise=cw, match_kind=kind, values=values)
    recs = ER.image_outputs(pma.serialize(), cw)
    nv = int(recs[:, 0].max()) + 1 if len(recs) else 0
    hay, v = per_match(pma, mode, text, offs)
    vdf = doc_freq(hay, v, nv)
    vh = np.bincount(v, minlength=nv).astype(np.uint64)
    twin = O.OraclePma.build(patterns, charwise=cw, match_kind=kind)
    trecs = ER.image_outputs(twin.serialize(), cw)
    assert np.array_equal(trecs[:, 1:3], recs[:, 1:3])
    rec_of = np.zeros(len(patterns) + 1, dtype=np.int64)
    rec_of[trecs[:, 0].astype(np.int64)] = np.arange(len(trecs))
    thay, tv = per_match(twin, mode, text, offs)
    odf = doc_freq(thay, rec_of[tv], len(trecs))
    return vdf, odf, vh, pma


def check(patterns, cw, kind, mode, text, offs, values=None, configs=CONFIGS, **kw):
    vdf, odf, vh, pma = expected(patterns, cw, kind, mode, text, offs, values)
    wire = pma.serialize()
    n = len(offs) - 1
    assert (vdf <= n).all() and (vdf <= vh).all() and np.array_equal(vdf > 0, vh > 0)
    for hot, kernel, pairs in configs:
        for key, want in (("value", vdf), ("output", odf)):
            rc, got, tot, info = F.df(wire, cw, mode, key, text, offs, len(want), hot_n=hot, kernel=kernel, df_pairs=pairs, **kw)
            assert rc == 0
            assert np.array_equal(got, want), (mode, key, hot, kernel, pairs, kw)
            assert tot == int(want.sum())
            assert info["left"] == 0  # every window emptied both sets
            if mode != 1:
                assert not info["which"] & 8  # only find_overlapping on a lane machine expands parent chains
    return vdf, odf, vh


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
    # the haystack, an empty one, and the haystack again: DF counts each of them once
    offs = np.array([0, len(hay), len(hay), 2 * len(hay)], dtype=np.uint64)
    check(t["patterns"], cw, O.KIND[kind], MODE[iterator], np.concatenate([text, text]), offs)


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
    """Duplicate patterns (equal and distinct values), an empty pattern (it counts every haystack the iterator reports
    it in, empty ones included), values shared by different patterns; LeftmostFirst drops patterns that extend a
    shorter one."""
    rng = np.random.default_rng(7300 + 10 * seed + kind)
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
    assert len(ER.image_outputs(pma.serialize(), False)) < len(pats)
    text = np.frombuffer(b"abcdxabcbcab" + b"bcd", dtype=np.uint8)
    vdf, _, _ = check(pats, False, 2, 3, text, np.array([0, 12, 15], dtype=np.uint64))
    assert vdf.sum() > 0


@pytest.mark.parametrize("seed", range(4))
def test_segments_count_a_haystack_once(seed):
    rng = np.random.default_rng(1700 + seed)
    alpha = int(rng.integers(2, 4))
    pats = rand_patterns(rng, int(rng.integers(1, 50)), alpha, 9, allow_empty=(seed == 0))
    lens = list(rng.integers(0, 400, size=20)) + [0, 64, 128, 1, 63, 65]
    hays = [bytes(rng.integers(97, 97 + alpha + 1, size=int(L)).tolist()) for L in lens]
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    text = np.frombuffer(b"".join(hays), dtype=np.uint8)
    for mode in (1, 2):
        for seg_len in (1, 3, 16, 100):
            check(pats, False, 0, mode, text, offs, configs=((256, 3, 1 << 16), (0, 3, 1)), seg_len=seg_len)


def test_one_haystack_many_segments():
    """A pattern that occurs in every segment of one long haystack: df = 1 while the histogram counts thousands."""
    pats = [b"ab", b"b", b"xyz"]
    text = np.frombuffer(b"ab" * 3000, dtype=np.uint8)
    offs = np.array([0, text.size], dtype=np.uint64)
    for mode in (1, 2):
        vdf, odf, vh = check(pats, False, 0, mode, text, offs, configs=((0, 3, 1), (256, 3, 1 << 16)), seg_len=64)
        assert vdf.tolist() == [1, 1 if mode == 1 else 0, 0] and vh[0] == 3000


def test_overlapping_states_share_a_chain_record():
    """find_overlapping: the states of "ba" and "ca" both report record "a" through their parent chains; the key-level
    set counts the haystack once for it."""
    pats = [b"a", b"ba", b"ca"]
    text = np.frombuffer(b"xbaxcax" + b"ca", dtype=np.uint8)
    offs = np.array([0, 7, 9], dtype=np.uint64)
    vdf, _, vh = check(pats, False, 0, 1, text, offs)
    assert vdf.tolist() == [2, 1, 2] and vh[0] == 3
    wire = O.OraclePma.build(pats).serialize()
    rc, got, tot, info = F.df(wire, False, 1, "value", text, offs, 3)
    assert rc == 0 and info["which"] == 3 + 8 and info["slot_pairs"] == 3 and info["key_pairs"] == tot == 5


@pytest.mark.parametrize("seed", range(0, 45, 4))
def test_charwise_mixed_width_chars(seed):
    kind, pats, text, offs = mixed_width_case(seed)
    for mode in ([3] if kind else [0, 1, 2]):
        check(pats, True, kind, mode, text, offs, configs=((0, 3, 1 << 16), (0, 3, 1), (0, 0, 1)))


def test_hand_made_automaton():
    wire, text, offs = hand_made_case(hay_len=3000)
    pma, _ = O.OraclePma.deserialize(wire)
    recs = ER.image_outputs(wire, False)
    assert len(set(recs[:, 0].tolist())) == len(recs)  # unique values: the output key is the value key re-indexed
    nv = int(recs[:, 0].max()) + 1
    for mode in (0, 1, 2):
        hay, v = per_match(pma, mode, text, offs)
        vdf = doc_freq(hay, v, nv)
        for key, want in (("value", vdf), ("output", vdf[recs[:, 0].astype(np.int64)])):
            for pairs in (1, 1 << 16):
                rc, got, tot, _ = F.df(wire, False, mode, key, text, offs, len(want), seg_len=256, df_pairs=pairs)
                assert rc == 0 and np.array_equal(got, want) and tot == int(want.sum())


def test_an_overflowing_window_adds_nothing():
    """A window whose pairs exceed df_pairs adds nothing and leaves both sets empty; split into halves, the batch gives
    what one large window gives."""
    rng = np.random.default_rng(99)
    pats = sorted(set(rand_patterns(rng, 60, 3, 4)))
    wire = O.OraclePma.build(pats).serialize()
    text, offs = _batch(rng, 3, 200, 120)
    for kernel in (3, 0):
        for mode in (0, 1, 2):
            rc, want, tot, info = F.df(wire, False, mode, "output", text, offs, len(pats), kernel=kernel, df_pairs=1 << 20)
            assert rc == 0 and info["windows"] == 1 and info["rescans"] == 0
            prior = np.arange(len(pats), dtype=np.uint64) * 7
            rc, got, _, info = F.df(wire, False, mode, "output", text, offs, len(pats), kernel=kernel, df_pairs=1, split=False,
                                    out=prior.copy())
            assert rc == OVERFLOW and np.array_equal(got, prior) and info["left"] == 0
            rc, got, t2, info = F.df(wire, False, mode, "output", text, offs, len(pats), kernel=kernel, df_pairs=1)
            assert rc == 0 and np.array_equal(got, want) and t2 == tot
            assert info["rescans"] > 0 and info["windows"] > 1 and info["left"] == 0


def test_accumulates_across_batches():
    """A then B into one array == A ++ B."""
    rng = np.random.default_rng(4243)
    pats = rand_patterns(rng, 40, 3, 6)
    wire = O.OraclePma.build(pats).serialize()
    text, offs = _batch(rng, 3, 40, 200)
    k = 17
    a_t, a_o = text[: int(offs[k])], offs[: k + 1]
    b_t, b_o = text[int(offs[k]):], offs[k:] - offs[k]
    for mode in (0, 1, 2):
        for key in ("value", "output"):
            n_df = len(pats)
            rc, whole, tot, _ = F.df(wire, False, mode, key, text, offs, n_df)
            assert rc == 0
            acc = np.zeros(n_df, dtype=np.uint64)
            rc1, _, t1, _ = F.df(wire, False, mode, key, a_t, a_o, n_df, out=acc)
            rc2, _, t2, _ = F.df(wire, False, mode, key, b_t, b_o, n_df, out=acc)
            assert rc1 == rc2 == 0 and np.array_equal(acc, whole) and t1 + t2 == tot


def test_errors_and_empty_batches():
    pma = O.OraclePma.build([b"a", b"ab", b"a"], values=[3, 9, 3])
    wire = pma.serialize()
    text = np.frombuffer(b"aab", dtype=np.uint8)
    offs = np.array([0, 3], dtype=np.uint64)
    rc, got, tot, _ = F.df(wire, False, 1, "value", text, offs, 10)
    assert rc == 0 and got.tolist() == [0, 0, 0, 1, 0, 0, 0, 0, 0, 1] and tot == 2  # values 3 and 9, one haystack
    assert F.df(wire, False, 1, "value", text, offs, 9)[0] == 1  # n_df must exceed the largest value
    assert F.df(wire, False, 1, "output", text, offs, 3)[0] == 0
    assert F.df(wire, False, 1, "output", text, offs, 2)[0] == 1  # ... or hold every output record
    assert F.df(wire, False, 3, "value", text, offs, 10)[0] == 5  # DACH_MATCH_KIND_MISMATCH
    for n in (0, 2):
        rc, h, tot, _ = F.df(wire, False, 1, "value", np.zeros(0, np.uint8), np.zeros(n + 1, np.uint64), 10)
        assert rc == 0 and tot == 0 and not h.any()
