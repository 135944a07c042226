"""Per-pattern histograms on the GPU (dach_dev_hist_batch / dach_hist_batch_host): against torch.bincount of the
matches path's values and against the oracle, both keys, device and host entry points, every kernel option that
changes which kernel runs."""
import numpy as np
import pytest

import daachorse_b200 as D
import oracle_api as O
from cases import seeded_reduce_case
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


def check(pma, mode, text, offs, opma=None):
    """value key == bincount of the full scan's values (== the oracle's, if given); output key re-indexed through
    outputs() when values are unique; host == device; sum == the COUNT total"""
    import torch

    vals = pma.outputs()[0]
    nv = int(vals.max()) + 1 if len(vals) else 0
    r = pma.scan_batch_host(mode, text, offs)
    want = np.bincount(r.matches["value"].astype(np.int64), minlength=nv).astype(np.uint64)
    if opma is not None:
        ref = opma.scan_batch(ORC[mode], text, offs, want_matches=True)
        assert np.array_equal(np.bincount(ref["matches"]["value"].astype(np.int64), minlength=nv).astype(np.uint64), want)
    got = pma.pattern_counts_host(mode, text, offs)
    assert np.array_equal(got, want)
    t, o = dev(text, offs)
    gd = pma.pattern_counts_device(mode, t, o)
    assert np.array_equal(gd.cpu().numpy().astype(np.uint64), want)
    rd = pma.scan_batch_device(mode, t, o)
    assert torch.equal(torch.bincount(rd.matches[:, 2].long(), minlength=nv), gd)
    out_h = pma.pattern_counts_host(mode, text, offs, key="output")
    out_d = pma.pattern_counts_device(mode, t, o, key="output")
    assert len(out_h) == len(vals) and np.array_equal(out_d.cpu().numpy().astype(np.uint64), out_h)
    assert int(out_h.sum()) == int(want.sum()) == int(pma.count_batch_host(mode, text, offs)[1])
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
        for name, values in (("kernel", (0, 1, 2, 4, 3)), ("hot_entries", (0, 6144)), ("seg_len", (64, 256, 0)),
                             ("hist_smem", (0, 1, 4096, 1 << 20, 1024))):
            for v in values:
                pma.set_option(name, v)
                got = check(pma, mode, text, offs)
                assert all(np.array_equal(a, b) for a, b in zip(got, base)), (name, v)


def test_duplicates_and_empty_pattern():
    pats = ["", "ab", "ab", "b", "abc", "é"]
    for cw in (False, True):
        for vals in (None, [5, 1, 1, 2, 3, 0], [0, 1, 2, 3, 4, 5]):
            pma = builder(cw).new().build_with_values(list(zip(pats, vals))) if vals else builder(cw).new().build(pats)
            hays = ["", "xabc", "éab", "bbb"]
            data = [h.encode() for h in hays]
            offs = np.zeros(5, dtype=np.uint64)
            offs[1:] = np.cumsum([len(h) for h in data])
            text = np.frombuffer(b"".join(data), dtype=np.uint8)
            for mode in (D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX):
                check(pma, mode, text, offs)
    lf = D.DoubleArrayAhoCorasickBuilder.new().match_kind(D.MatchKind.LeftmostFirst).build(["ab", "abc", "b", "bc"])
    assert len(lf.outputs()[0]) < 4
    text = np.frombuffer(b"abcbcab", dtype=np.uint8)
    check(lf, D.LEFTMOST_FIND, text, np.array([0, text.size], dtype=np.uint64))


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
        want = torch.bincount(r.matches[:, 2].long(), minlength=nv)
        del r
        for hs in (1024, 0):
            pma.set_option("hist_smem", hs)
            assert torch.equal(pma.pattern_counts_device(mode, t, o), want)
        pma.set_option("hist_smem", 1024)
        k = n // 3
        acc = torch.zeros(nv, dtype=torch.int64, device="cuda")
        pma.pattern_counts_device(mode, t[: k * cfg["hay_len"]], o[: k + 1], out=acc)
        pma.pattern_counts_device(mode, t[k * cfg["hay_len"]:], o[k:] - o[k], out=acc)
        assert torch.equal(acc, want)
        oh = pma.pattern_counts_device(mode, t, o, key="output")
        assert torch.equal(oh, want[torch.from_numpy(pma.outputs()[0].astype(np.int64)).cuda()])
        h = pma.pattern_counts_host(mode, t.cpu().numpy(), o.cpu().numpy().astype(np.uint64))
        assert np.array_equal(h, want.cpu().numpy().astype(np.uint64))
        assert pma.stats()["d2h_bytes"] == nv * 8


def test_one_byte_run_u64_counts():
    """Patterns a .. a x 64 on one haystack of N = 128 MiB of 'a' under find_overlapping: pattern k occurs N - k + 1
    times; every event lands on a handful of states and the sum passes 2^32."""
    import torch

    N = 128 << 20
    pats = [b"a" * k for k in range(1, 65)]
    t = torch.full((N,), 97, dtype=torch.uint8, device="cuda")
    o = torch.tensor([0, N], dtype=torch.int64, device="cuda")
    std = D.DoubleArrayAhoCorasick.new(pats)
    want = torch.tensor([N - k + 1 for k in range(1, 65)], dtype=torch.int64, device="cuda")
    for hs in (1024, 0):
        std.set_option("hist_smem", hs)
        h = std.pattern_counts_device(D.FIND_OVERLAPPING, t, o)
        assert torch.equal(h, want) and int(h.sum()) == 64 * N - 2016
    h = std.pattern_counts_device(D.FIND, t, o)
    assert int(h[0]) == N and int(h.sum()) == N


def test_empty_batches_and_errors():
    import torch

    pma = D.DoubleArrayAhoCorasick.with_values([("a", 3), ("ab", 9)])
    h = pma.pattern_counts_host(D.FIND, np.zeros(0, np.uint8), np.zeros(1, np.uint64))
    assert len(h) == 10 and not h.any()
    e = torch.zeros(0, dtype=torch.uint8, device="cuda")
    assert not pma.pattern_counts_device(D.FIND, e, torch.zeros(3, dtype=torch.int64, device="cuda")).any()
    text = np.frombuffer(b"aaaaa", dtype=np.uint8)
    bad = np.array([0, 5, 3], dtype=np.uint64)
    with pytest.raises(D.DaachorseError) as ex:
        pma.pattern_counts_host(D.FIND, text, bad)
    assert ex.value.code == 1
    t = torch.from_numpy(text.copy()).cuda()
    with pytest.raises(D.DaachorseError) as ex:
        pma.pattern_counts_device(D.FIND, t, torch.tensor([0, 5, 3], dtype=torch.int64, device="cuda"))
    assert ex.value.code == 1
    o = torch.tensor([0, 5], dtype=torch.int64, device="cuda")
    with pytest.raises(AssertionError):
        pma.pattern_counts_device(D.LEFTMOST_FIND, t, o)
    for out in (torch.zeros(9, dtype=torch.int64, device="cuda"), torch.zeros(10, dtype=torch.int32, device="cuda"),
                torch.zeros(10, dtype=torch.int64)):
        with pytest.raises(D.DaachorseError):
            pma.pattern_counts_device(D.FIND, t, o, out=out)
    with pytest.raises(D.DaachorseError):
        pma.pattern_counts_host(D.FIND, text, np.array([0, 5], dtype=np.uint64), out=np.zeros(9, np.uint64))
    import ctypes as C

    from daachorse_b200 import _lib

    L = _lib.load()
    d = pma.device_handle()
    tot = C.c_uint64()
    hist = torch.zeros(10, dtype=torch.int64, device="cuda")
    args = (C.c_void_p(t.data_ptr()), C.c_void_p(o.data_ptr()), 1, 5, C.c_void_p(hist.data_ptr()))
    assert L.dach_dev_hist_batch(d, D.FIND, 1, *args, 9, C.byref(tot), None) == _lib.INVALID_ARGUMENT
    assert L.dach_dev_hist_batch(d, D.FIND, 0, *args, 1, C.byref(tot), None) == _lib.INVALID_ARGUMENT
    assert L.dach_dev_hist_batch(d, D.FIND, 2, *args, 10, C.byref(tot), None) == _lib.INVALID_ARGUMENT
    assert L.dach_dev_hist_batch(d, D.LEFTMOST_FIND, 1, *args, 10, C.byref(tot), None) == _lib.MATCH_KIND_MISMATCH
    assert not hist.any()
    assert L.dach_dev_hist_batch(d, D.FIND, 1, *args, 10, C.byref(tot), None) == 0
    assert hist.tolist() == [0, 0, 0, 5, 0, 0, 0, 0, 0, 0] and tot.value == 5


def test_convenience_calls():
    pma = D.DoubleArrayAhoCorasick.new(["bcd", "ab", "a"])
    assert pma.value_counts_batch(["abcd", "xyz", "aab"]).tolist() == [1, 2, 3]
    v, ln, par = pma.outputs()
    assert sorted(v.tolist()) == [0, 1, 2] and sorted(ln.tolist()) == [1, 2, 3] and len(par) == 3
    lm = D.DoubleArrayAhoCorasickBuilder.new().match_kind(D.MatchKind.LeftmostLongest).build(["ab", "a", "abcd"])
    assert lm.value_counts_batch(["abcdab", "a"]).tolist() == [1, 1, 1]
