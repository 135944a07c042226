"""Per-pattern document frequencies on the GPU (dach_dev_df_batch / dach_df_batch_host): against np.unique of the
(haystack, key) pairs of the matches path and of the oracle, both keys, device and host entry points, every kernel
option that changes which kernel runs, and a pair table so small that most windows are scanned again as halves."""
import ctypes as C

import numpy as np
import pytest

import daachorse_b200 as D
import oracle_api as O
from cases import seeded_reduce_case
from daachorse_b200 import _lib
from daachorse_b200 import synth as S

pytestmark = pytest.mark.gpu

ORC = {D.FIND: O.FIND, D.FIND_OVERLAPPING: O.FIND_OVERLAPPING,
       D.FIND_OVERLAPPING_NO_SUFFIX: O.FIND_OVERLAPPING_NO_SUFFIX, D.LEFTMOST_FIND: O.LEFTMOST_FIND}


def builder(cw):
    return D.CharwiseDoubleArrayAhoCorasickBuilder if cw else D.DoubleArrayAhoCorasickBuilder


def dev(text, offs):
    import torch

    t = torch.from_numpy(np.ascontiguousarray(text)).cuda() if len(text) else torch.zeros(0, dtype=torch.uint8, device="cuda")
    return t, torch.from_numpy(offs.astype(np.int64)).cuda()


def doc_freq(counts, values, n_keys):
    """haystacks per key from a match list: np.unique of the (haystack, key) pairs, then a bincount"""
    hay = np.repeat(np.arange(len(counts), dtype=np.uint64), np.asarray(counts, dtype=np.int64))
    pairs = np.unique((hay << np.uint64(32)) | np.asarray(values, dtype=np.uint64))
    return np.bincount((pairs & np.uint64(0xffffffff)).astype(np.int64), minlength=n_keys).astype(np.uint64)


def check(pma, mode, text, offs, opma=None):
    """value key == the DF of the full scan's matches (== the oracle's, if given); host == device; the invariants
    against pattern_counts on the same bytes; output key re-indexed through outputs() when values are unique"""
    vals = pma.outputs()[0]
    nv = int(vals.max()) + 1 if len(vals) else 0
    n = len(offs) - 1
    r = pma.scan_batch_host(mode, text, offs)
    want = doc_freq(np.diff(r.offsets.astype(np.int64)), r.matches["value"], nv)
    if opma is not None:
        ref = opma.scan_batch(ORC[mode], text, offs, want_matches=True)
        assert np.array_equal(doc_freq(ref["counts"], ref["matches"]["value"], nv), want)
    got = pma.doc_counts_host(mode, text, offs)
    assert np.array_equal(got, want)
    t, o = dev(text, offs)
    gd = pma.doc_counts_device(mode, t, o)
    assert np.array_equal(gd.cpu().numpy().astype(np.uint64), want)
    hist = pma.pattern_counts_host(mode, text, offs)
    assert (want <= n).all() and (want <= hist).all() and np.array_equal(want > 0, hist > 0)
    out_h = pma.doc_counts_host(mode, text, offs, key="output")
    out_d = pma.doc_counts_device(mode, t, o, key="output")
    assert len(out_h) == len(vals) and np.array_equal(out_d.cpu().numpy().astype(np.uint64), out_h)
    if len(set(vals.tolist())) == len(vals):
        assert np.array_equal(out_h, want[vals.astype(np.int64)])
    return want, out_h


@pytest.mark.parametrize("cw", [False, True])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_seeded_batches_and_options(cw, kind):
    pats, text, offs = seeded_reduce_case(cw, kind)
    pma = builder(cw).new().match_kind(kind).build(pats)
    opma = O.OraclePma.build(pats, charwise=cw, match_kind=kind)
    for mode in ([D.LEFTMOST_FIND] if kind else [D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX]):
        base = check(pma, mode, text, offs, opma)
        assert pma.last_doc_windows() == (1, 0)
        for name, values in (("kernel", (0, 1, 2, 4, 3)), ("hot_entries", (0, 6144)), ("seg_len", (64, 256, 0))):
            for v in values:
                pma.set_option(name, v)
                got = check(pma, mode, text, offs)
                assert all(np.array_equal(a, b) for a, b in zip(got, base)), (name, v)
        # the smallest table (df_pairs is raised to max(states, output records)): many windows, each re-scan exact
        pma.set_option("df_pairs", 1)
        for kernel in (3, 0):
            pma.set_option("kernel", kernel)
            got = check(pma, mode, text, offs)
            assert all(np.array_equal(a, b) for a, b in zip(got, base)), ("df_pairs", kernel)
            windows, rescans = pma.last_doc_windows()
            assert rescans > 0 and windows > 1
        pma.set_option("kernel", 3)
        pma.set_option("df_pairs", 1 << 24)


def test_duplicates_and_empty_pattern():
    pats = ["", "ab", "ab", "b", "abc", "é"]
    for cw in (False, True):
        for vals in (None, [5, 1, 1, 2, 3, 0], [0, 1, 2, 3, 4, 5]):
            pma = builder(cw).new().build_with_values(list(zip(pats, vals))) if vals else builder(cw).new().build(pats)
            hays = ["", "xabc", "éab", "bbb", ""]
            data = [h.encode() for h in hays]
            offs = np.zeros(len(data) + 1, dtype=np.uint64)
            offs[1:] = np.cumsum([len(h) for h in data])
            text = np.frombuffer(b"".join(data), dtype=np.uint8)
            for mode in (D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX):
                check(pma, mode, text, offs)
    lf = D.DoubleArrayAhoCorasickBuilder.new().match_kind(D.MatchKind.LeftmostFirst).build(["ab", "abc", "b", "bc"])
    text = np.frombuffer(b"abcbcab", dtype=np.uint8)
    check(lf, D.LEFTMOST_FIND, text, np.array([0, 3, text.size], dtype=np.uint64))


def test_c3_64mib_and_accumulation():
    import torch

    cfg = S.config("C3", 1.0 / 64)
    ps = S.make_patterns(cfg)
    pma = D.DoubleArrayAhoCorasick.new(ps.as_list())
    pool, bounds = S.make_pool(cfg, ps, 64 << 20, seed=2)
    n = (64 << 20) // cfg["hay_len"]
    starts = S.window_starts(bounds, len(pool), n, cfg["hay_len"], seed=3)
    t, o = S.materialise_on_device(torch.from_numpy(pool).cuda(), torch.from_numpy(starts).cuda(), cfg["hay_len"])
    nv = len(ps.as_list())
    for mode in (D.FIND_OVERLAPPING, D.FIND):
        r = pma.scan_batch_device(mode, t, o)
        hay = torch.repeat_interleave(torch.arange(n, device="cuda"), torch.diff(r.offsets.long()))
        pairs = torch.unique(hay * nv + r.matches[:, 2].long())
        want = torch.bincount(pairs % nv, minlength=nv)
        del r, hay, pairs
        got = pma.doc_counts_device(mode, t, o)
        assert torch.equal(got, want)
        assert pma.last_doc_windows()[1] == 0  # a 64 MiB C3 batch fits the default table
        hist = pma.pattern_counts_device(mode, t, o)
        assert bool((got <= hist).all()) and torch.equal(got > 0, hist > 0) and int(got.max()) <= n
        k = n // 3
        acc = torch.zeros(nv, dtype=torch.int64, device="cuda")
        pma.doc_counts_device(mode, t[: k * cfg["hay_len"]], o[: k + 1], out=acc)
        pma.doc_counts_device(mode, t[k * cfg["hay_len"]:], o[k:] - o[k], out=acc)
        assert torch.equal(acc, want)
        h = np.zeros(nv, dtype=np.uint64)
        pma.doc_counts_host(mode, t[: k * cfg["hay_len"]].cpu().numpy(), o[: k + 1].cpu().numpy().astype(np.uint64), out=h)
        pma.doc_counts_host(mode, t[k * cfg["hay_len"]:].cpu().numpy(), (o[k:] - o[k]).cpu().numpy().astype(np.uint64), out=h)
        assert np.array_equal(h, want.cpu().numpy().astype(np.uint64))


def test_one_byte_run_across_segments():
    """Patterns a .. a x 64 on one haystack of N = 128 MiB of 'a' under find_overlapping, cut into many segments: each
    pattern occurs about 2^27 times and every segment reports it, yet the haystack counts once."""
    import torch

    N = 128 << 20
    pats = [b"a" * k for k in range(1, 65)]
    t = torch.full((N,), 97, dtype=torch.uint8, device="cuda")
    o = torch.tensor([0, N], dtype=torch.int64, device="cuda")
    std = D.DoubleArrayAhoCorasick.new(pats)
    for mode in (D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX):
        df = std.doc_counts_device(mode, t, o)
        hist = std.pattern_counts_device(mode, t, o)
        assert torch.equal(df, (hist > 0).long())
        if mode == D.FIND_OVERLAPPING:
            assert bool((df == 1).all()) and int(hist[0]) == N


def test_empty_batches_and_errors_leave_df_unchanged():
    import torch

    pma = D.DoubleArrayAhoCorasick.with_values([("a", 3), ("ab", 9)])
    prior = np.arange(10, dtype=np.uint64)
    h = pma.doc_counts_host(D.FIND, np.zeros(0, np.uint8), np.zeros(1, np.uint64), out=prior.copy())
    assert np.array_equal(h, prior)
    e = torch.zeros(0, dtype=torch.uint8, device="cuda")
    assert not pma.doc_counts_device(D.FIND, e, torch.zeros(3, dtype=torch.int64, device="cuda")).any()
    text = np.frombuffer(b"aaaaa", dtype=np.uint8)
    h = prior.copy()
    with pytest.raises(D.DaachorseError) as ex:
        pma.doc_counts_host(D.FIND, text, np.array([0, 5, 3], dtype=np.uint64), out=h)
    assert ex.value.code == 1 and np.array_equal(h, prior)
    t = torch.from_numpy(text.copy()).cuda()
    dprior = torch.arange(10, dtype=torch.int64, device="cuda")
    for bad in ([0, 5, 3], [0, 3, 6]):  # descending; past text_bytes
        d = dprior.clone()
        with pytest.raises(D.DaachorseError) as ex:
            pma.doc_counts_device(D.FIND, t, torch.tensor(bad, dtype=torch.int64, device="cuda"), out=d)
        assert ex.value.code == 1 and torch.equal(d, dprior)
    o = torch.tensor([0, 5], dtype=torch.int64, device="cuda")
    L = _lib.load()
    d = pma.device_handle()
    tot = C.c_uint64()
    out = dprior.clone()
    args = (C.c_void_p(t.data_ptr()), C.c_void_p(o.data_ptr()), 1, 5, C.c_void_p(out.data_ptr()))
    assert L.dach_dev_df_batch(d, D.FIND, 1, *args, 9, C.byref(tot), None) == _lib.INVALID_ARGUMENT  # short n_df
    assert L.dach_dev_df_batch(d, D.FIND, 0, *args, 1, C.byref(tot), None) == _lib.INVALID_ARGUMENT
    assert L.dach_dev_df_batch(d, D.FIND, 2, *args, 10, C.byref(tot), None) == _lib.INVALID_ARGUMENT  # unknown key
    assert L.dach_dev_df_batch(d, D.LEFTMOST_FIND, 1, *args, 10, C.byref(tot), None) == _lib.MATCH_KIND_MISMATCH
    assert torch.equal(out, dprior)
    assert L.dach_dev_df_batch(d, D.FIND, 1, *args, 10, C.byref(tot), None) == 0
    assert (out - dprior).tolist() == [0, 0, 0, 1, 0, 0, 0, 0, 0, 0] and tot.value == 1


def test_convenience_calls():
    pma = D.DoubleArrayAhoCorasick.new(["bcd", "ab", "a"])
    assert pma.value_doc_counts_batch(["abcd", "xyz", "aab", "a"]).tolist() == [1, 2, 3]
    assert pma.value_counts_batch(["abcd", "xyz", "aab", "a"]).tolist() == [1, 2, 4]
    lm = D.DoubleArrayAhoCorasickBuilder.new().match_kind(D.MatchKind.LeftmostLongest).build(["ab", "a", "abcd"])
    assert lm.value_doc_counts_batch(["abcdab", "a", "ab"]).tolist() == [2, 1, 1]
