"""Masked text (dach_dev_mask_batch) on the kernels' lane logic compiled for the CPU (tests/emu_mask), against the
oracle's match lists turned into spans.  No GPU needed; tests/test_gpu_mask.py runs the same checks on the device."""
import json
import os

import numpy as np
import pytest

import emu_mask_api as M
import oracle_api as O
from cases import mixed_width_case

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "search_tests.json"), encoding="utf-8"))
MODE = {"find_iter": 0, "find_overlapping_iter": 1, "find_overlapping_no_suffix_iter": 2, "leftmost_find_iter": 3}
ORC_MODE = {0: O.FIND, 1: O.FIND_OVERLAPPING, 2: O.FIND_OVERLAPPING_NO_SUFFIX, 3: O.LEFTMOST_FIND}
# (hot records, kernel option, segment length)
CONFIGS = ((0, 3, 0), (256, 3, 0), (1 << 16, 3, 0), (0, 3, 64), (256, 3, 16), (0, 1, 0), (0, 4, 0), (0, 0, 0), (64, 0, 0))
FILL = 0x2A


def oracle_mask(pma, mode, text, offs, fill=FILL):
    ref = pma.scan_batch(ORC_MODE[mode], text, offs, want_matches=True)
    return M.expected_from_matches(text, offs, ref["matches"], ref["counts"], fill)


def check(pma, cw, mode, text, offs, configs=CONFIGS, fill=FILL, want=None):
    want = oracle_mask(pma, mode, text, offs, fill) if want is None else want
    wire = pma.serialize()
    seen = set()
    for hot, kernel, seg in configs:
        rc, got, which = M.mask(wire, cw, mode, text, offs, fill, hot_n=hot, kernel=kernel, seg_len=seg)
        assert rc == 0
        assert np.array_equal(got, want), (mode, hot, kernel, seg, np.flatnonzero(got != want)[:10])
        seen.add(which)
    return seen


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
    pma = O.OraclePma.build(t["patterns"], charwise=cw, match_kind=O.KIND[kind])
    check(pma, cw, MODE[iterator], text, np.array([0, len(hay)], dtype=np.uint64))


def _batch(rng, alpha, n, maxlen):
    hays = [bytes(rng.integers(97, 97 + alpha + 1, size=int(rng.integers(0, maxlen))).tolist()) for _ in range(n)]
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    return np.frombuffer(b"".join(hays), dtype=np.uint8), offs


def rand_patterns(rng, n, alpha, maxlen, allow_empty=False):
    return [bytes(rng.integers(97, 97 + alpha, size=int(rng.integers(0 if allow_empty else 1, maxlen + 1))).tolist())
            for _ in range(n)]


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_random_batches_every_machine(seed, kind):
    """Random patterns (the empty one in some seeds) on random batches: StdMachine3 under the three Standard
    iterators, LmMachine, and the lane-per-haystack loops."""
    rng = np.random.default_rng(9100 + 10 * seed + kind)
    alpha = int(rng.integers(2, 4))
    pats = rand_patterns(rng, int(rng.integers(3, 40)), alpha, 7, allow_empty=seed % 3 == 0)
    text, offs = _batch(rng, alpha, 40, 300)
    pma = O.OraclePma.build(pats, match_kind=kind)
    seen = set()
    for mode in ([3] if kind else [0, 1, 2]):
        seen |= check(pma, False, mode, text, offs)
    assert seen & {0, 1, 3, 11}


@pytest.mark.parametrize("seed", range(4))
def test_spans_straddle_segments(seed):
    """Long haystacks cut into short segments: spans that end in one segment start in the one before it (or several
    before), and a match that ends exactly on a segment boundary is reported once."""
    rng = np.random.default_rng(9300 + seed)
    pats = rand_patterns(rng, 30, 2, 40) + [b"ab" * 20, b"a" * 33]
    lens = [1000, 0, 64, 65, 17, 2000]
    offs = np.zeros(len(lens) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    text = rng.integers(97, 99, size=int(offs[-1])).astype(np.uint8)
    pma = O.OraclePma.build(pats)
    for mode in (1, 2):
        seen = check(pma, False, mode, text, offs, configs=((0, 3, 16), (256, 3, 32), (0, 3, 256), (0, 3, 0)))
        assert any(w & 8 for w in seen)


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_heavily_overlapping_spans(kind):
    """'a' x k under the patterns 'a' .. 'a' x 64: every byte is covered by up to 64 spans, lists grow to 64 entries."""
    pats = [b"a" * k for k in range(1, 65)]
    lens = [0, 1, 5, 63, 64, 65, 300]
    offs = np.zeros(len(lens) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    text = np.full(int(offs[-1]), 97, dtype=np.uint8)
    text[::97] = 98  # a few breaks
    pma = O.OraclePma.build(pats, match_kind=kind)
    for mode in ([3] if kind else [0, 1, 2]):
        check(pma, False, mode, text, offs)


def test_lists_of_255_and_more():
    """Output lists of 255 and more entries (the saturated list length of StdMachine3's queue entries)."""
    pats = [b"x" * k for k in range(1, 301)]
    lens = [300, 254, 255, 256, 600]
    offs = np.zeros(len(lens) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    text = np.full(int(offs[-1]), ord("x"), dtype=np.uint8)
    text[700] = ord("y")
    pma = O.OraclePma.build(pats)
    for mode in (0, 1, 2):
        check(pma, False, mode, text, offs, configs=((0, 3, 0), (0, 3, 128), (0, 0, 0)))


@pytest.mark.parametrize("kind", [0, 1, 2])
@pytest.mark.parametrize("cw", [False, True])
def test_empty_pattern_masks_nothing(kind, cw):
    pats = ["", "ab", "b"] if cw else [b"", b"ab", b"b"]
    hays = [b"", b"ab", b"xxabx", b"bbb"]
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    text = np.frombuffer(b"".join(hays), dtype=np.uint8)
    pma = O.OraclePma.build(pats, charwise=cw, match_kind=kind)
    for mode in ([3] if kind else [0, 1, 2]):
        check(pma, cw, mode, text, offs)


@pytest.mark.parametrize("seed", range(6))
def test_charwise_multibyte_chars(seed):
    """Chars of 1-4 bytes (and unmapped ones): spans start and end on char boundaries, an ASCII fill keeps UTF-8."""
    kind, pats, text, offs = mixed_width_case(seed)
    pma = O.OraclePma.build(pats, charwise=True, match_kind=kind)
    for mode in ([3] if kind else [0, 1, 2]):
        want = oracle_mask(pma, mode, text, offs)
        check(pma, True, mode, text, offs, configs=((0, 3, 0), (0, 0, 0)), want=want)
        want.tobytes().decode("utf-8")


def test_bytes_outside_the_haystacks_are_copied():
    """offs[0] > 0 and offs[n] < text_bytes: the bytes before and after the batch are copied unchanged."""
    pats = [b"ab", b"b", b"zz"]
    inner = b"abzzab" * 40
    text = np.frombuffer(b"zzab" + inner + b"abzz", dtype=np.uint8)
    offs = np.array([4, 4 + 100, 4 + 100, 4 + len(inner)], dtype=np.uint64)
    pma = O.OraclePma.build(pats)
    for mode in (0, 1, 2):
        want = oracle_mask(pma, mode, text, offs)
        assert np.array_equal(want[:4], text[:4]) and np.array_equal(want[-4:], text[-4:])
        check(pma, False, mode, text, offs, want=want)


def test_bad_offsets_write_nothing():
    pma = O.OraclePma.build([b"a"])
    text = np.frombuffer(b"aaaa", dtype=np.uint8)
    out = np.full(4, 7, dtype=np.uint8)
    rc, got, _ = M.mask(pma.serialize(), False, 1, text, np.array([0, 3, 2], dtype=np.uint64), FILL, out=out)
    assert rc == 1 and (got == 7).all()


def _damaged_wire(pats, record, length):
    """The serialized automaton of `pats` with the length of output record `record` overwritten (the records are the
    wire's last 12 x n_out bytes before the match kind and the state count)."""
    pma = O.OraclePma.build(pats)
    w = bytearray(pma.serialize())
    n_out = pma.num_outputs()
    at = len(w) - 5 - 12 * n_out + 12 * record + 4
    old = int(np.frombuffer(bytes(w[at:at + 4]), dtype="<u4")[0])
    w[at:at + 4] = np.array([length], dtype="<u4").tobytes()
    return pma, bytes(w), old


def test_damaged_length_is_clamped_at_the_haystack():
    """A deserialized automaton whose output length exceeds the match end: the span starts at the haystack's first
    byte, and nothing before the haystack changes."""
    pats = [b"ab", b"cd"]
    pma, wire, _ = _damaged_wire(pats, 0, 40)
    recs = np.frombuffer(wire[len(wire) - 5 - 12 * pma.num_outputs():len(wire) - 5], dtype="<u4").reshape(-1, 3)
    assert 40 in recs[:, 1]
    hays = [b"xxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxxx", b"abxxxxcd", b"xcdxxxxxxab", b"ab"]
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    text = np.frombuffer(b"".join(hays), dtype=np.uint8)
    long_value = int(recs[recs[:, 1] == 40][0, 0])
    for mode in (0, 2):
        ref = pma.scan_batch(ORC_MODE[mode], text, offs, want_matches=True)
        m = ref["matches"]
        starts = np.where(m["value"] == long_value, np.maximum(m["end"].astype(np.int64) - 40, 0), m["start"])
        hay = np.repeat(np.arange(len(hays)), ref["counts"].astype(np.int64))
        want = M.expected_mask(text, offs, starts, m["end"], hay, FILL)
        assert np.array_equal(want[:int(offs[1])], text[:int(offs[1])])
        for hot, kernel, seg in ((0, 3, 0), (0, 0, 0)):
            rc, got, _ = M.mask(wire, False, mode, text, offs, FILL, hot_n=hot, kernel=kernel, seg_len=seg)
            assert rc == 0
            assert np.array_equal(got, want), (mode, kernel)
