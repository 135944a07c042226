"""Counts and first matches on the GPU (dach_dev_count_batch / dach_first_batch_host / ...): against the full match
list of the same scan path and against the oracle, device and host entry points, every kernel option that changes
which kernel runs."""
import json
import os

import numpy as np
import pytest

import daachorse_b200 as D
import oracle_api as O
from cases import mixed_width_case
from daachorse_b200 import synth as S

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "search_tests.json"), encoding="utf-8"))
MODE = {"find_iter": D.FIND, "find_overlapping_iter": D.FIND_OVERLAPPING,
        "find_overlapping_no_suffix_iter": D.FIND_OVERLAPPING_NO_SUFFIX, "leftmost_find_iter": D.LEFTMOST_FIND}
ORC = {D.FIND: O.FIND, D.FIND_OVERLAPPING: O.FIND_OVERLAPPING,
       D.FIND_OVERLAPPING_NO_SUFFIX: O.FIND_OVERLAPPING_NO_SUFFIX, D.LEFTMOST_FIND: O.LEFTMOST_FIND}
KIND = {"Standard": 0, "LeftmostLongest": 1, "LeftmostFirst": 2}
NONE = np.array([(0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF)], dtype=D.MATCH_DTYPE)[0]


def builder(cw):
    return D.CharwiseDoubleArrayAhoCorasickBuilder if cw else D.DoubleArrayAhoCorasickBuilder


def from_matches(r, n):
    counts = np.diff(r.offsets.astype(np.int64)).astype(np.uint64)
    first = np.zeros(n, dtype=D.MATCH_DTYPE)
    first[:] = NONE
    found = counts > 0
    first[found] = r.matches[r.offsets[:-1][found].astype(np.int64)]
    return counts, first, found


def check(pma, mode, text, offs, opma=None):
    """host and device COUNT / FIRST == the full scan's per-haystack runs (== the oracle, if given)"""
    import torch

    n = len(offs) - 1
    r = pma.scan_batch_host(mode, text, offs)
    counts, first, found = from_matches(r, n)
    if opma is not None:
        ref = opma.scan_batch(ORC[mode], text, offs, want_matches=True)
        assert np.array_equal(counts, ref["counts"].astype(np.uint64))
    c, total = pma.count_batch_host(mode, text, offs)
    assert np.array_equal(c, counts) and total == int(counts.sum())
    f, fd = pma.first_batch_host(mode, text, offs)
    assert np.array_equal(fd, found) and f.tobytes() == first.tobytes()
    t = torch.from_numpy(np.ascontiguousarray(text)).cuda() if len(text) else torch.zeros(0, dtype=torch.uint8, device="cuda")
    o = torch.from_numpy(offs.astype(np.int64)).cuda()
    cd = pma.count_batch_device(mode, t, o)
    assert np.array_equal(cd.cpu().numpy().astype(np.uint64), counts)
    fdv, fdd = pma.first_batch_device(mode, t, o)
    assert np.array_equal(fdd.cpu().numpy(), found)
    assert fdv.cpu().numpy().view(np.uint32).tobytes() == first.tobytes()
    return counts


@pytest.mark.parametrize("variant,iterator,coll,kind", [tuple(c) for c in GOLD["configs"] if c[1] in MODE])
def test_golden_vectors(variant, iterator, coll, kind):
    cw = variant == "charwise"
    for g in GOLD["collections"][coll]:
        for t in GOLD["groups"][g]:
            pma = builder(cw).new().match_kind(KIND[kind]).build(t["patterns"])
            hay = t["haystack"].encode()
            text = np.frombuffer(hay, dtype=np.uint8)
            check(pma, MODE[iterator], text, np.array([0, len(hay)], dtype=np.uint64))


@pytest.mark.parametrize("cw", [False, True])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_seeded_batches_and_options(cw, kind):
    rng = np.random.default_rng(60 + 3 * kind + cw)
    if cw:
        kind_, pats, text, offs = mixed_width_case(9 + kind)
        assert kind_ == kind
    else:
        pats = [bytes(rng.integers(97, 101, size=int(rng.integers(1, 7))).tolist()) for _ in range(300)]
        lens = rng.integers(0, 3000, size=700)
        offs = np.zeros(len(lens) + 1, dtype=np.uint64)
        offs[1:] = np.cumsum(lens)
        text = rng.integers(97, 102, size=int(offs[-1])).astype(np.uint8)
    pma = builder(cw).new().match_kind(kind).build(pats)
    opma = O.OraclePma.build(pats, charwise=cw, match_kind=kind)
    for mode in ([D.LEFTMOST_FIND] if kind else [D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX]):
        base = check(pma, mode, text, offs, opma)
        for name, values in (("kernel", (0, 1, 2, 4, 3)), ("hot_entries", (0, 6144)), ("seg_len", (64, 256, 0))):
            for v in values:
                pma.set_option(name, v)
                assert np.array_equal(check(pma, mode, text, offs), base), (name, v)


def test_c3_64mib_against_the_full_scan():
    import torch

    cfg = S.config("C3", 1.0 / 64)
    ps = S.make_patterns(cfg)
    pma = D.DoubleArrayAhoCorasick.new(ps.as_list())
    pool, bounds = S.make_pool(cfg, ps, 64 << 20, seed=2)
    n = (64 << 20) // cfg["hay_len"]
    starts = S.window_starts(bounds, len(pool), n, cfg["hay_len"], seed=3)
    t, o = S.materialise_on_device(torch.from_numpy(pool).cuda(), torch.from_numpy(starts).cuda(), cfg["hay_len"])
    for mode in (D.FIND_OVERLAPPING, D.FIND):
        r = pma.scan_batch_device(mode, t, o)
        counts = torch.diff(r.offsets)
        c = pma.count_batch_device(mode, t, o)
        assert torch.equal(c, counts)
        f, fd = pma.first_batch_device(mode, t, o)
        assert torch.equal(fd, counts > 0)
        idx = r.offsets[:-1][fd]
        assert torch.equal(f[fd], r.matches[idx])


def test_empty_batch_empty_haystacks_and_the_empty_pattern():
    for cw in (False, True):
        pma = builder(cw).new().build(["", "ab", "é"])
        c, tot = pma.count_batch_host(D.FIND, np.zeros(0, np.uint8), np.zeros(1, np.uint64))
        assert len(c) == 0 and tot == 0
        hays = ["", "xab", "éé", ""]
        data = [h.encode() for h in hays]
        offs = np.zeros(5, dtype=np.uint64)
        offs[1:] = np.cumsum([len(h) for h in data])
        text = np.frombuffer(b"".join(data), dtype=np.uint8)
        c, tot = pma.count_batch_host(D.FIND, text, offs)
        assert list(c) == [(len(h) if cw else len(d)) + 1 for h, d in zip(hays, data)]
        for mode in (D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX):
            check(pma, mode, text, offs)
        assert list(pma.is_match_batch(hays)) == [True] * 4


def test_errors():
    import torch

    pma = D.DoubleArrayAhoCorasick.new(["a"])
    bad = np.array([0, 5, 3], dtype=np.uint64)
    text = np.frombuffer(b"aaaaa", dtype=np.uint8)
    for f in (pma.count_batch_host, pma.first_batch_host):
        with pytest.raises(D.DaachorseError) as e:
            f(D.FIND, text, bad)
        assert e.value.code == 1
    t = torch.from_numpy(text.copy()).cuda()
    o = torch.tensor([0, 5, 3], dtype=torch.int64, device="cuda")
    for f in (pma.count_batch_device, pma.first_batch_device):
        with pytest.raises(D.DaachorseError) as e:
            f(D.FIND, t, o)
        assert e.value.code == 1
    with pytest.raises(AssertionError):
        pma.count_batch_host(D.LEFTMOST_FIND, text, np.array([0, 5], dtype=np.uint64))
    with pytest.raises(D.DaachorseError):
        pma.count_batch_device(D.FIND, t, torch.tensor([0, 5], dtype=torch.int64, device="cuda"),
                               out=torch.zeros(2, dtype=torch.int64, device="cuda"))


def test_u64_count():
    """Patterns a .. a x 64 on one haystack of N = 128 MiB of 'a': find_overlapping = 64 N - 2016 (> 2^32)."""
    import torch

    N = 128 << 20
    pats = [b"a" * k for k in range(1, 65)]
    t = torch.full((N,), 97, dtype=torch.uint8, device="cuda")
    o = torch.tensor([0, N], dtype=torch.int64, device="cuda")
    std = D.DoubleArrayAhoCorasick.new(pats)
    assert int(std.count_batch_device(D.FIND_OVERLAPPING, t, o)[0]) == 64 * N - 2016
    assert int(std.count_batch_device(D.FIND, t, o)[0]) == N
    lm = D.DoubleArrayAhoCorasickBuilder.new().match_kind(D.MatchKind.LeftmostLongest).build(pats)
    assert int(lm.count_batch_device(D.LEFTMOST_FIND, t, o)[0]) == N // 64


def test_convenience_calls():
    pma = D.DoubleArrayAhoCorasick.new(["bcd", "ab", "a"])
    assert list(pma.count_batch(["abcd", "xyz", ""])) == [3, 0, 0]
    assert pma.first_match_batch(["abcd", "xyz"]) == [D.Match(0, 1, 2), None]
    assert pma.is_match("zzab") and not pma.is_match("zzz")
    lm = D.DoubleArrayAhoCorasickBuilder.new().match_kind(D.MatchKind.LeftmostLongest).build(["ab", "a", "abcd"])
    assert lm.first_match_batch(["xabcd"]) == [D.Match(1, 5, 2)]
    assert list(lm.count_batch(["abcdab"])) == [2]
