"""GPU parity: the CUDA path, called through the C ABI, against the oracle and the
reference's golden vectors.  Bit-exact: identical (start, end, value) tuples in identical
per-haystack order."""
import json
import os

import numpy as np
import pytest

import daachorse_b200 as D
import oracle_api as O
from cases import hand_made_case, mixed_width_case, nul_heavy_case
from daachorse_b200 import synth as S

pytestmark = pytest.mark.gpu
DEFAULT_KERNEL = 3

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "search_tests.json"), encoding="utf-8"))
MODE = {"find_iter": D.FIND, "find_overlapping_iter": D.FIND_OVERLAPPING,
        "find_overlapping_no_suffix_iter": D.FIND_OVERLAPPING_NO_SUFFIX, "leftmost_find_iter": D.LEFTMOST_FIND}
ORC = {D.FIND: O.FIND, D.FIND_OVERLAPPING: O.FIND_OVERLAPPING,
       D.FIND_OVERLAPPING_NO_SUFFIX: O.FIND_OVERLAPPING_NO_SUFFIX, D.LEFTMOST_FIND: O.LEFTMOST_FIND}
KIND = {"Standard": 0, "LeftmostLongest": 1, "LeftmostFirst": 2}


def builder(cw):
    return D.CharwiseDoubleArrayAhoCorasickBuilder if cw else D.DoubleArrayAhoCorasickBuilder


def check_batch(pma, opma, mode, text, offs, nthreads=8):
    r = pma.scan_batch_host(mode, text, offs)
    ref = opma.scan_batch(ORC[mode], text, offs, nthreads=nthreads, want_matches=True)
    assert len(r.matches) == ref["total"]
    assert np.array_equal(np.diff(r.offsets.astype(np.int64)), ref["counts"].astype(np.int64))
    assert r.matches.tobytes() == ref["matches"].tobytes()
    return r


@pytest.mark.parametrize("variant,iterator,coll,kind", [tuple(c) for c in GOLD["configs"] if c[1] in MODE])
def test_golden_vectors(variant, iterator, coll, kind):
    """tests/aho_corasick_crate_test.rs:63-382 through the iterator surface of the package."""
    cw = variant == "charwise"
    for g in GOLD["collections"][coll]:
        for t in GOLD["groups"][g]:
            pma = builder(cw).new().match_kind(KIND[kind]).build(t["patterns"])
            it = getattr(pma, iterator)(t["haystack"])
            got = [(m.value(), m.start(), m.end()) for m in it]
            assert got == [tuple(x) for x in t["matches"]], (t["name"], t["patterns"], t["haystack"])


def test_config_c1():
    """BASELINE.json configs[0]: ['bcd','ab','a'] over 'abcd' x 10k (README.md:57-71)."""
    pma = D.DoubleArrayAhoCorasick.new(["bcd", "ab", "a"])
    r = pma.find_overlapping_batch(["abcd"] * 10000)
    assert len(r.matches) == 30000
    m = r.matches.reshape(10000, 3)
    assert (m["start"] == [0, 0, 1]).all() and (m["end"] == [1, 2, 4]).all() and (m["value"] == [2, 1, 0]).all()
    assert np.array_equal(r.offsets, np.arange(10001, dtype=np.uint64) * 3)


def test_charwise_zero_length_multibyte():
    """src/charwise.rs:1373-1456."""
    pats = ["a", "æ", "あ", ""]
    hay = "いあabcÆæう"
    pma = D.CharwiseDoubleArrayAhoCorasick.new(pats)
    assert [(m.start(), m.end(), m.value()) for m in pma.find_overlapping_iter(hay)] == [
        (0, 0, 3), (3, 3, 3), (3, 6, 2), (6, 6, 3), (6, 7, 0), (7, 7, 3), (8, 8, 3), (9, 9, 3),
        (11, 11, 3), (11, 13, 1), (13, 13, 3), (16, 16, 3)]
    assert [(m.start(), m.end(), m.value()) for m in pma.find_iter(hay)] == [
        (0, 0, 3), (3, 3, 3), (6, 6, 3), (7, 7, 3), (8, 8, 3), (9, 9, 3), (11, 11, 3), (13, 13, 3), (16, 16, 3)]
    pml = D.CharwiseDoubleArrayAhoCorasickBuilder.new().match_kind(D.MatchKind.LeftmostLongest).build(pats)
    assert [(m.start(), m.end(), m.value()) for m in pml.leftmost_find_iter(hay)] == [
        (0, 0, 3), (3, 6, 2), (6, 7, 0), (8, 8, 3), (9, 9, 3), (11, 13, 1), (16, 16, 3)]


def test_no_suffix_iter():
    """src/bytewise/iter.rs:484-509."""
    for cls in (D.DoubleArrayAhoCorasick, D.CharwiseDoubleArrayAhoCorasick):
        pma = cls.new(["a", "ab", ""])
        assert [(m.end() - m.start(), m.end(), m.value()) for m in pma.find_overlapping_no_suffix_iter("ab")] == [
            (0, 0, 2), (1, 1, 0), (2, 2, 1)]


def test_empty_pattern_set_all_short_haystacks():
    """test_empty_pattern_set, src/bytewise.rs:1418-1431."""
    pma = D.DoubleArrayAhoCorasick.new([])
    hays = [bytes([a]) for a in range(256)] + [bytes([a, b]) for a in range(256) for b in range(256)]
    r = pma.find_overlapping_batch(hays)
    assert len(r.matches) == 0 and int(r.offsets[-1]) == 0


def test_empty_batch_and_empty_haystacks():
    pma = D.DoubleArrayAhoCorasick.new(["a", ""])
    r = pma.scan_batch_host(D.FIND_OVERLAPPING, np.zeros(0, np.uint8), np.zeros(1, np.uint64))
    assert len(r.matches) == 0 and list(r.offsets) == [0]
    r = pma.find_overlapping_batch(["", "", "a", ""])
    assert [r.triples(i) for i in range(4)] == [[(0, 0, 1)], [(0, 0, 1)], [(0, 0, 1), (0, 1, 0), (1, 1, 1)], [(0, 0, 1)]]


def _random_case(rng, cw, allow_empty):
    alpha = int(rng.integers(2, 6))
    pats = [bytes(rng.integers(97, 97 + alpha, size=int(rng.integers(0 if allow_empty else 1, 8))).tolist())
            for _ in range(int(rng.integers(1, 300)))]
    table = ["a", "b", "é", "あ", "𝄞", "c"]
    if cw:
        pats = ["".join(table[b - 97] for b in p) for p in pats]
    n = int(rng.integers(1, 2000))
    hays = []
    for _ in range(n):
        L = int(rng.integers(0, 200))
        sym = rng.integers(0, alpha + 1, size=L)
        hays.append("".join(table[int(i)] for i in sym).encode() if cw else bytes((97 + sym).astype(np.uint8).tolist()))
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    return pats, np.frombuffer(b"".join(hays), dtype=np.uint8), offs


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("cw", [False, True])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_random_batches(seed, cw, kind):
    rng = np.random.default_rng(1000 + 100 * seed + 10 * kind + cw)
    pats, text, offs = _random_case(rng, cw, allow_empty=(seed == 0))
    pma = builder(cw).new().match_kind(kind).build(pats)
    opma = O.OraclePma.build(pats, charwise=cw, match_kind=kind)
    for mode in ([D.LEFTMOST_FIND] if kind else [D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX]):
        check_batch(pma, opma, mode, text, offs)


@pytest.mark.parametrize("seed", range(12))
def test_charwise_mixed_width_chars(seed):
    """Chars of 1-4 bytes, unmapped chars, empty patterns: lane machine and lane-per-haystack kernel."""
    kind, pats, text, offs = mixed_width_case(seed)
    pma = D.CharwiseDoubleArrayAhoCorasickBuilder.new().match_kind(kind).build(pats)
    opma = O.OraclePma.build(pats, charwise=True, match_kind=kind)
    for mode in ([D.LEFTMOST_FIND] if kind else [D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX]):
        r1 = check_batch(pma, opma, mode, text, offs)
        pma.set_option("kernel", 0)
        r0 = pma.scan_batch_host(mode, text, offs)
        pma.set_option("kernel", 1)
        assert r0.matches.tobytes() == r1.matches.tobytes() and np.array_equal(r0.offsets, r1.offsets)


def test_charwise_leftmost_empty_pattern_never_stops_inside_a_char():
    pma = D.CharwiseDoubleArrayAhoCorasickBuilder.new().match_kind(D.MatchKind.LeftmostFirst).build(["ca", "", "𝄞𝄞c"])
    r = pma.leftmost_find_batch(["bc𝄞", "𝄞", ""])
    assert r.triples(0) == [(0, 0, 1), (1, 1, 1), (6, 6, 1)]
    assert r.triples(1) == [(0, 0, 1), (4, 4, 1)]
    assert r.triples(2) == [(0, 0, 1)]


def test_kernel_options_do_not_change_results():
    rng = np.random.default_rng(77)
    pats, text, offs = _random_case(rng, False, False)
    pma = D.DoubleArrayAhoCorasick.new(pats)
    base = pma.scan_batch_host(D.FIND_OVERLAPPING, text, offs)
    for opts in ({"hot_records": -1}, {"hot_records": 17}, {"threads": 128}, {"threads": 512, "ctas_per_sm": 2},
                 {"kernel": 0}, {"kernel": 1}, {"kernel": 2}, {"kernel": 2, "threads": 256}, {"kernel": 3, "threads": 256},
                 {"kernel": 3, "threads": 768, "ctas_per_sm": 2}, {"kernel": 4}, {"kernel": 4, "threads": 768}, {"kernel": 4, "threads": 256}, {"kernel": 0, "hot_records": 100}, {"l2_hints": 0}, {"l2_hints": 1}, {"hot_entries": 4096},
                 {"hot_entries": 256}, {"hot_entries": 8192}, {"hot_entries": 1 << 20}, {"gather_ordered": 0}, {"gather_ordered": 2}, {"tail_seg": 1}):
        for k, v in opts.items():
            pma.set_option(k, v)
        r = pma.scan_batch_host(D.FIND_OVERLAPPING, text, offs)
        assert r.matches.tobytes() == base.matches.tobytes() and np.array_equal(r.offsets, base.offsets)
        pma.set_option("hot_records", 0)
        pma.set_option("threads", 1024)
        pma.set_option("ctas_per_sm", 1)
        pma.set_option("kernel", DEFAULT_KERNEL)
        pma.set_option("l2_hints", 2)
        pma.set_option("hot_entries", 0)
        pma.set_option("gather_ordered", 1)
        pma.set_option("tail_seg", 0)


def test_overflow_protocol_through_the_c_abi():
    import ctypes as C

    from daachorse_b200 import _lib

    pma = D.DoubleArrayAhoCorasick.new(["a", "aa"])
    L = _lib.load()
    d = pma.device_handle()
    text = np.frombuffer(b"a" * 1000, dtype=np.uint8)
    offs = np.array([0, 1000], dtype=np.uint64)
    out = np.zeros(1999, dtype=D.MATCH_DTYPE)
    oo = np.zeros(2, dtype=np.uint64)
    need = C.c_uint64()
    rc = L.dach_scan_batch_host(d, D.FIND_OVERLAPPING, text.ctypes.data, offs.ctypes.data, 1, out.ctypes.data, 10,
                                oo.ctypes.data, C.byref(need))
    assert rc == _lib.OUTPUT_OVERFLOW and need.value == 1999
    rc = L.dach_scan_batch_host(d, D.FIND_OVERLAPPING, text.ctypes.data, offs.ctypes.data, 1, out.ctypes.data, 1999,
                                oo.ctypes.data, C.byref(need))
    assert rc == 0 and need.value == 1999 and list(oo) == [0, 1999]
    rc = L.dach_scan_batch_host(d, D.LEFTMOST_FIND, text.ctypes.data, offs.ctypes.data, 1, out.ctypes.data, 1999,
                                oo.ctypes.data, C.byref(need))
    assert rc == _lib.MATCH_KIND_MISMATCH


def test_device_resident_api_equals_host_api():
    import torch

    rng = np.random.default_rng(5)
    pats, text, offs = _random_case(rng, False, False)
    pma = D.DoubleArrayAhoCorasick.new(pats)
    host = pma.scan_batch_host(D.FIND_OVERLAPPING, text, offs)
    t = torch.from_numpy(text.copy()).cuda()
    o = torch.from_numpy(offs.astype(np.int64)).cuda()
    dev = pma.scan_batch_device(D.FIND_OVERLAPPING, t, o)
    got = dev.matches.cpu().numpy().view(np.uint32).reshape(-1, 3)
    want = np.stack([host.matches["start"], host.matches["end"], host.matches["value"]], axis=1)
    assert np.array_equal(got, want)
    assert np.array_equal(dev.offsets.cpu().numpy().astype(np.uint64), host.offsets)


def _synth_case(name, n_patterns, n_hay, pool_bytes):
    cfg = S.config(name)
    ps = S.make_patterns(cfg, n_patterns)
    pool, b = S.make_pool(cfg, ps, pool_bytes)
    starts = S.window_starts(b, len(pool), n_hay, cfg["hay_len"])
    text, offs = S.materialise_host(pool, starts, cfg["hay_len"])
    return cfg, ps, text, offs


def test_config_c2_full_compare():
    """BASELINE.json configs[1]: 10k ASCII patterns, find_overlapping_iter, 256K x 256 B."""
    cfg, ps, text, offs = _synth_case("C2", None, 262144, 32 << 20)
    pats = ps.as_list()
    pma = D.DoubleArrayAhoCorasick.new(pats)
    opma = O.OraclePma.build_packed(ps.blob, ps.offs)
    r = check_batch(pma, opma, D.FIND_OVERLAPPING, text, offs)
    assert 0.01 < len(r.matches) / text.size < 0.5


def test_config_c3_reduced_batch_all_standard_modes():
    """BASELINE.json configs[2] automaton (675k patterns) on a 64 MiB slice of the batch, full
    tuple compare in find_overlapping_iter and find_iter."""
    cfg, ps, text, offs = _synth_case("C3", None, 16384, 32 << 20)
    pma = D.DoubleArrayAhoCorasick.new(ps.as_list())
    opma = O.OraclePma.build_packed(ps.blob, ps.offs)
    assert pma.serialize() == opma.serialize()
    check_batch(pma, opma, D.FIND_OVERLAPPING, text, offs)
    check_batch(pma, opma, D.FIND, text, offs)
    check_batch(pma, opma, D.FIND_OVERLAPPING_NO_SUFFIX, text[: 4096 * 2048], offs[:2049])
    # the three bytewise Standard lane machines (kernel 1: StdMachine, 2: StdMachine2, 3: StdMachine3 with and
    # without its shared-memory records) agree
    for mode in (D.FIND_OVERLAPPING, D.FIND, D.FIND_OVERLAPPING_NO_SUFFIX):
        res = []
        for k, hot in ((1, -1), (2, -1), (3, -1), (3, 0), (3, 4096), (4, 0)):
            pma.set_option("kernel", k)
            pma.set_option("hot_entries", hot)
            res.append(pma.scan_batch_host(mode, text, offs))
        for r in res[1:]:
            assert r.matches.tobytes() == res[0].matches.tobytes() and np.array_equal(r.offsets, res[0].offsets)


def test_config_c4_reduced_charwise_leftmost_longest():
    """BASELINE.json configs[3]: charwise 100k CJK patterns, leftmost_find_iter LeftmostLongest.
    Haystacks are cut at char boundaries and padded with ASCII spaces."""
    cfg = S.config("C4")
    ps = S.make_patterns(cfg)
    pool, b = S.make_pool(cfg, ps, 16 << 20)
    hay_len, n = cfg["hay_len"], 16384
    starts = S.window_starts(b, len(pool), n, hay_len)
    text, offs = S.materialise_host(pool, starts, hay_len)
    text = S.pad_to_char_boundary(text.reshape(n, hay_len)).reshape(-1)
    text.tobytes().decode("utf-8")  # must be valid UTF-8 now
    pma = D.CharwiseDoubleArrayAhoCorasickBuilder.new().match_kind(D.MatchKind.LeftmostLongest).build(
        [p.decode() for p in ps.as_list()])
    opma = O.OraclePma.build_packed(ps.blob, ps.offs, charwise=True, match_kind=1)
    assert pma.serialize() == opma.serialize()
    check_batch(pma, opma, D.LEFTMOST_FIND, text, offs)
    # bytewise leftmost on the same data
    pmb = D.DoubleArrayAhoCorasickBuilder.new().match_kind(D.MatchKind.LeftmostLongest).build(ps.as_list())
    opmb = O.OraclePma.build_packed(ps.blob, ps.offs, match_kind=1)
    check_batch(pmb, opmb, D.LEFTMOST_FIND, text, offs)


@pytest.mark.parametrize("kind", [1, 2])
def test_bytewise_leftmost_lane_machine(kind):
    """The leftmost lane machine (LmMachine) against the oracle and against the lane-per-haystack
    kernel it replaces, on dictionary-like data with an empty pattern in the set (init / skip_empty
    rules) and haystacks that end inside partial matches."""
    cfg = S.config("C3")
    ps = S.make_patterns(cfg, n=60000)
    pats = ps.as_list() + ([b""] if kind == 1 else [])
    pool, b = S.make_pool(cfg, ps, 8 << 20)
    rng = np.random.default_rng(5 + kind)
    n = 6000
    lens = rng.integers(0, 700, size=n)
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    text = np.ascontiguousarray(pool[: int(offs[-1])])
    pma = D.DoubleArrayAhoCorasickBuilder.new().match_kind(kind).build(pats)
    opma = O.OraclePma.build(pats, match_kind=kind)
    r1 = check_batch(pma, opma, D.LEFTMOST_FIND, text, offs)
    pma.set_option("kernel", 0)
    r0 = pma.scan_batch_host(D.LEFTMOST_FIND, text, offs)
    pma.set_option("kernel", 1)
    pma.set_option("threads", 256)
    r2 = pma.scan_batch_host(D.LEFTMOST_FIND, text, offs)
    assert r0.matches.tobytes() == r1.matches.tobytes() == r2.matches.tobytes()
    assert np.array_equal(r0.offsets, r1.offsets) and np.array_equal(r2.offsets, r1.offsets)


@pytest.mark.parametrize("kind", [0, 1])
def test_binary_text_full_of_nul_bytes_on_a_relaid_out_automaton(kind):
    """Binary patterns and haystacks made mostly of 0x00, an automaton several times the hot region (the
    shifted part keeps the holes re-placed families leave behind): label 0 must never be taken for a child
    in such a hole (dev_image.cpp); every lane-machine kernel against the oracle.  The emulated lane logic
    runs the same case on the CPU (tests/test_emu_lane.py)."""
    pats, text, offs = nul_heavy_case(kind)
    pma = D.DoubleArrayAhoCorasickBuilder.new().match_kind(kind).build(pats)
    opma = O.OraclePma.build(pats, match_kind=kind)
    for mode in ([D.LEFTMOST_FIND] if kind else [D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX]):
        for kernel in ((DEFAULT_KERNEL, 1) if kind else (DEFAULT_KERNEL, 2, 1)):
            pma.set_option("kernel", kernel)
            check_batch(pma, opma, mode, text, offs)


def test_hand_made_automaton_with_long_haystacks_is_scanned_whole():
    """A blob that passes the crate's validation but is not Aho-Corasick's automaton (failure links rewired by
    hand): the state after a text is not a function of its last bytes, so the device path must not cut the long
    haystacks into segments (HostImage::segmentable) -- results as the crate's loops give them.  The emulated
    lanes run the same case, and show that forcing segments would be wrong (tests/test_emu_lane.py)."""
    wire, text, offs = hand_made_case()
    pma, rest = D.DoubleArrayAhoCorasick.deserialize(wire)
    assert len(rest) == 0
    opma, _ = O.OraclePma.deserialize(wire)
    for mode in (D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX, D.FIND):
        check_batch(pma, opma, mode, text, offs)


def test_full_size_properties_c3():
    """Size-independent properties at a larger batch (1 GiB of the C3 workload, device resident):
    (1) find_iter output == greedy filter of the find_overlapping_iter output (SURVEY C.2);
    (2) per-haystack order-sensitive hashes of a 1 % sample == oracle;
    (3) total == sum of the per-haystack ranges, offsets ascending."""
    import torch

    cfg = S.config("C3")
    ps = S.make_patterns(cfg)
    pool, b = S.make_pool(cfg, ps, 64 << 20)
    n, hay_len = 262144, cfg["hay_len"]
    starts = S.window_starts(b, len(pool), n, hay_len)
    pool_t = torch.from_numpy(pool).cuda()
    text_t, offs_t = S.materialise_on_device(pool_t, torch.from_numpy(starts).cuda(), hay_len)
    pma = D.DoubleArrayAhoCorasick.new(ps.as_list())
    ov = pma.scan_batch_device(D.FIND_OVERLAPPING, text_t, offs_t)
    fi = pma.scan_batch_device(D.FIND, text_t, offs_t)
    oo = ov.offsets.cpu().numpy()
    assert oo[0] == 0 and (np.diff(oo) >= 0).all() and oo[-1] == ov.matches.shape[0]
    # (2) oracle on a 1 % sample
    opma = O.OraclePma.build_packed(ps.blob, ps.offs)
    rng = np.random.default_rng(9)
    sample = np.sort(rng.choice(n, size=n // 100, replace=False))
    stext, soffs = S.materialise_host(pool, starts[sample], hay_len)
    ref = opma.scan_batch(O.FIND_OVERLAPPING, stext, soffs, nthreads=8, want_matches=True)
    om = ov.matches.cpu().numpy().view(np.uint32)
    pos = 0
    for k, h in enumerate(sample):
        got = om[oo[h]:oo[h + 1]]
        cnt = int(ref["counts"][k])
        want = ref["matches"][pos:pos + cnt]
        pos += cnt
        assert got.shape[0] == cnt
        assert np.array_equal(got, np.stack([want["start"], want["end"], want["value"]], axis=1))
    # (1) greedy filter identity on the first 4096 haystacks
    fo = fi.offsets.cpu().numpy()
    fm = fi.matches.cpu().numpy().view(np.uint32)
    for h in range(4096):
        r = 0
        exp = []
        for s, e, v in om[oo[h]:oo[h + 1]]:
            if s >= r:
                exp.append((s, e, v))
                r = e
        assert [tuple(x) for x in fm[fo[h]:fo[h + 1]]] == exp


def test_host_batch_slicing_matches_single_slice():
    """dach_scan_batch_host pipelines the batch in slices; results must not depend on the slicing
    (slice boundaries at every haystack count, empty haystacks at the boundaries, non-zero offs[0])."""
    rng = np.random.default_rng(21)
    pats, text, offs = _random_case(rng, False, False)
    n = len(offs) - 1
    # make haystacks bigger so that 1 MiB slices cut the batch many times
    reps = 40
    big = np.tile(text, reps)
    boffs = np.concatenate([offs[:-1] + np.uint64(k * int(offs[-1])) for k in range(reps)] + [np.array([reps * int(offs[-1])], dtype=np.uint64)])
    pma = D.DoubleArrayAhoCorasick.new(pats)
    opma = O.OraclePma.build(pats)
    pma.set_option("slice_mib", 1 << 20)
    one = pma.scan_batch_host(D.FIND_OVERLAPPING, big, boffs)
    pma.set_option("slice_mib", 1)
    many = pma.scan_batch_host(D.FIND_OVERLAPPING, big, boffs)
    assert one.matches.tobytes() == many.matches.tobytes() and np.array_equal(one.offsets, many.offsets)
    ref = opma.scan_batch(O.FIND_OVERLAPPING, big, boffs, nthreads=8, want_matches=True)
    assert many.matches.tobytes() == ref["matches"].tobytes()
    # a view that does not start at offset 0, with preallocated outputs and an exact capacity
    sub = boffs[5:300]
    out = np.empty(int(ref["counts"][5:299].sum()), dtype=D.MATCH_DTYPE)
    r = pma.scan_batch_host(D.FIND_OVERLAPPING, big, sub, out=out)
    lo = int(ref["counts"][:5].sum())
    assert r.matches.tobytes() == ref["matches"][lo:lo + len(out)].tobytes()
    pma.set_option("slice_mib", 64)


def test_segmented_scan_equals_sequential():
    """Intra-haystack segments (SURVEY.md App. C.1) on the device: forced tiny segments, automatic
    segments on a few long haystacks (the C5 shape), and an empty pattern."""
    rng = np.random.default_rng(33)
    pats = [bytes(rng.integers(97, 101, size=int(rng.integers(1, 9))).tolist()) for _ in range(200)] + [b""]
    pma = D.DoubleArrayAhoCorasick.new(pats)
    opma = O.OraclePma.build(pats)
    lens = [0, 1, 255, 256, 257, 100000, 3, 70000, 0, 512]
    offs = np.zeros(len(lens) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    text = rng.integers(97, 102, size=int(offs[-1])).astype(np.uint8)
    for mode in (D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX):
        ref = opma.scan_batch(ORC[mode], text, offs, nthreads=8, want_matches=True)
        for seg in (0, 16, 256, 4096, -1):
            pma.set_option("seg_len", seg)
            r = pma.scan_batch_host(mode, text, offs)
            assert r.matches.tobytes() == ref["matches"].tobytes(), (mode, seg)
            assert np.array_equal(np.diff(r.offsets.astype(np.int64)), ref["counts"].astype(np.int64))
    pma.set_option("seg_len", 0)


def test_tail_segmentation_many_small_haystacks():
    """More than 4 haystacks per lane: only the last 2 x lanes haystacks are cut into segments
    (dev_scan.cu, scan_locked); ragged lengths, the longest haystacks sit in the tail."""
    import torch

    cfg = S.config("C2")
    ps = S.make_patterns(cfg, n=3000)
    pool, b = S.make_pool(cfg, ps, 8 << 20)
    rng = np.random.default_rng(11)
    n = 4 * torch.cuda.get_device_properties(0).multi_processor_count * 1024 + 5000  # lanes = SMs x 1024 threads
    lens = rng.integers(0, 96, size=n)
    lens[-3000:] = rng.integers(2000, 9000, size=3000)
    lens[-1] = 0
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    reps = int(offs[-1]) // len(pool) + 1
    text = np.ascontiguousarray(np.tile(pool, reps)[: int(offs[-1])])
    pma = D.DoubleArrayAhoCorasick.new(ps.as_list())
    opma = O.OraclePma.build_packed(ps.blob, ps.offs)
    pma.set_option("tail_seg", 1)
    for mode in (D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX):
        check_batch(pma, opma, mode, text, offs, nthreads=32)  # 46 MB: one host slice, i.e. one launch over all haystacks


def test_config_c5_shape_long_records_reduced():
    """BASELINE.json configs[4] shape: a large automaton (here 200k patterns of the C5 generator) over
    a few long records; the scan cuts them into segments automatically.  Full tuple compare."""
    cfg = S.config("C5")
    ps = S.make_patterns(cfg, 200000)
    pool, b = S.make_pool(cfg, ps, 16 << 20)
    n, hay_len = 24, 1 << 19
    starts = S.window_starts(b, len(pool), n, hay_len)
    text, offs = S.materialise_host(pool, starts, hay_len)
    pma = D.DoubleArrayAhoCorasick.new(ps.as_list())
    opma = O.OraclePma.build_packed(ps.blob, ps.offs)
    assert pma.serialize() == opma.serialize()
    check_batch(pma, opma, D.FIND_OVERLAPPING, text, offs)
    check_batch(pma, opma, D.FIND_OVERLAPPING_NO_SUFFIX, text, offs)


@pytest.mark.parametrize("mode", [D.FIND, D.FIND_OVERLAPPING])
def test_stream_chunks_equal_the_stepper_over_the_whole_stream(mode):
    """dach_dev_scan_stream: 3000 streams cut into ragged chunks, state and position carried from round
    to round, against the crate's stepper driven over each whole stream (oracle), and the carried state
    ids against a CPU walk of the reference transition function."""
    import torch

    cfg = S.config("C2")
    ps = S.make_patterns(cfg, n=4000)
    pool, b = S.make_pool(cfg, ps, 4 << 20)
    rng = np.random.default_rng(21)
    n = 3000
    lens = rng.integers(0, 1200, size=n)
    starts = rng.integers(0, len(pool) - 1300, size=n)
    streams = [pool[int(s): int(s) + int(l)] for s, l in zip(starts, lens)]
    pma = D.DoubleArrayAhoCorasick.new(ps.as_list())
    opma = O.OraclePma.build_packed(ps.blob, ps.offs)
    offs_all = np.zeros(n + 1, dtype=np.uint64)
    offs_all[1:] = np.cumsum(lens)
    whole = np.concatenate(streams) if n else np.zeros(0, np.uint8)
    ref = opma.scan_batch(O.FIND_STEPPER if mode == D.FIND else O.FIND_OVERLAPPING_STEPPER, whole, offs_all, nthreads=16,
                          want_matches=True)
    state = torch.zeros(n, dtype=torch.int32, device="cuda")
    pos = np.zeros(n, dtype=np.int64)
    got = [[] for _ in range(n)]
    while (pos < lens).any():
        k = rng.integers(0, 400, size=n)
        chunks = [st[int(p): int(p) + int(kk)] for st, p, kk in zip(streams, pos, k)]
        offs = np.zeros(n + 1, dtype=np.int64)
        offs[1:] = np.cumsum([len(c) for c in chunks])
        text = np.concatenate(chunks) if offs[-1] else np.zeros(0, np.uint8)
        t = torch.from_numpy(np.ascontiguousarray(text)).cuda() if len(text) else torch.zeros(16, dtype=torch.uint8, device="cuda")[:0]
        r = pma.scan_stream_device(mode, t, torch.from_numpy(offs).cuda(), state, torch.from_numpy(pos.astype(np.int32)).cuda())
        m = r.matches.cpu().numpy().view(np.uint32).reshape(-1, 3)
        oo = r.offsets.cpu().numpy()
        for i in range(n):
            if oo[i + 1] > oo[i]:
                got[i].append(m[oo[i]: oo[i + 1]])
        pos += np.array([len(c) for c in chunks])
    rm = ref["matches"]
    ro = np.concatenate([[0], np.cumsum(ref["counts"])]).astype(np.int64)
    for i in range(n):
        want = np.stack([rm["start"][ro[i]: ro[i + 1]], rm["end"][ro[i]: ro[i + 1]], rm["value"][ro[i]: ro[i + 1]]], axis=1)
        want = want[want[:, 1] != 0]  # matches() of the initial state, which no consume() produced
        have = np.concatenate(got[i]) if got[i] else np.zeros((0, 3), np.uint32)
        assert np.array_equal(have, want), i
    st = state.cpu().numpy().view(np.uint32)
    for i in range(0, n, 97):
        assert int(st[i]) == opma.state_after(bytes(streams[i]), find_mode=(mode == D.FIND))


def _c3_small(n=2048, hay_len=4096, seed=5):
    cfg = S.config("C3")
    ps = S.make_patterns(cfg, n=20000)
    pool, b = S.make_pool(cfg, ps, 8 << 20, seed=seed)
    starts = S.window_starts(b, len(pool), n, hay_len, seed=seed + 1)
    text, offs = S.materialise_host(pool, starts, hay_len)
    return ps, text, offs


def test_jobs_on_two_streams_equal_the_blocking_call():
    """dach_job_*: scan and place only enqueue; two jobs of one automaton run on two streams at once and each
    reproduces dach_dev_scan_batch on its batch (also with the placement on a third stream and a device-side base)."""
    import torch

    ps, text, offs = _c3_small()
    pma = D.DoubleArrayAhoCorasick.new(ps.as_list())
    dev = torch.device("cuda", 0)
    half = (len(offs) - 1) // 2
    t = torch.from_numpy(text).to(dev)
    o = torch.from_numpy(offs.astype(np.int64)).to(dev)
    parts = [(t, o[: half + 1]), (t, o[half:])]
    want = [pma.scan_batch_device(D.FIND_OVERLAPPING, tt, oo) for tt, oo in parts]
    streams = [torch.cuda.Stream(dev) for _ in range(3)]
    jobs = [pma.job(0), pma.job(0)]
    outs = [torch.zeros((w.matches.shape[0] + 7, 3), dtype=torch.int32, device=dev) for w in want]
    oofs = [torch.zeros(p[1].numel(), dtype=torch.int64, device=dev) for p in parts]
    torch.cuda.synchronize()
    for rep in range(3):  # jobs are reused: scan -> place -> wait -> scan ...
        for k in range(2):
            jobs[k].scan(D.FIND_OVERLAPPING, parts[k][0], parts[k][1], outs[k].shape[0], stream=streams[k])
        jobs[0].place(outs[0], oofs[0], stream=streams[0])
        jobs[1].place(outs[1], oofs[1], stream=streams[2])  # another stream than the scan's
        for k in range(2):
            assert jobs[k].wait() == want[k].matches.shape[0]
            assert torch.equal(outs[k][: want[k].matches.shape[0]], want[k].matches)
            assert torch.equal(oofs[k], want[k].offsets)
    # a device-side base shifts the placement and the offsets
    base = torch.tensor([5], dtype=torch.int64, device=dev)
    big = torch.zeros((outs[0].shape[0] + 5, 3), dtype=torch.int32, device=dev)
    jobs[0].scan(D.FIND_OVERLAPPING, parts[0][0], parts[0][1], big.shape[0], stream=streams[0])
    jobs[0].place(big, oofs[0], base=base, stream=streams[0])
    k = jobs[0].wait()
    assert torch.equal(big[5: 5 + k], want[0].matches) and torch.equal(oofs[0], want[0].offsets + 5)


def _group_case(world, devices):
    """One process drives `world` ranks (rank r on devices[r]): every rank scans its shard with a job and places
    it through the group; rank 0's buffers must equal the single-device result of the whole batch."""
    import torch

    from daachorse_b200 import shard

    ps, text, offs = _c3_small(n=1536)
    pma = D.DoubleArrayAhoCorasick.new(ps.as_list())
    n = len(offs) - 1
    d0 = torch.device("cuda", devices[0])
    whole = pma.scan_batch_device(D.FIND_OVERLAPPING, torch.from_numpy(text).to(d0), torch.from_numpy(offs.astype(np.int64)).to(d0))
    bounds = shard.byte_balanced_ranges(offs, world)
    cap = int(whole.matches.shape[0]) + 64
    groups = [shard.PeerGroup(r, world, devices[r], cap, n, exchange=None) for r in range(world)]
    blobs = [g.handle for g in groups]
    for g in groups:
        g.connect(blobs)
    sent32, sent64 = 0x5A5A5A5A, 0x5A5A5A5A5A5A5A5A
    with torch.cuda.device(devices[0]):
        m_all, o_all = groups[0].result(cap)  # rank 0's whole result buffers: nothing past `total` may be written
        m_all.fill_(sent32)
        o_all.fill_(sent64)
        torch.cuda.synchronize()
    jobs, inputs, streams = [], [], []
    for r in range(world):
        dev = torch.device("cuda", devices[r])
        lo, hi = bounds[r], bounds[r + 1]
        tt = torch.from_numpy(text[int(offs[lo]): int(offs[hi])]).to(dev)
        oo = torch.from_numpy((offs[lo: hi + 1] - offs[lo]).astype(np.int64)).to(dev)
        inputs.append((tt, oo))
        with torch.cuda.device(dev):
            jobs.append(pma.job(devices[r]))
            streams.append(torch.cuda.Stream(dev))
    for step in range(3):  # the buffers are reused step after step
        order = list(range(world)) if step % 2 == 0 else list(reversed(range(world)))  # scans may be issued in any order
        for r in order:
            with torch.cuda.device(devices[r]):
                jobs[r].scan(D.FIND_OVERLAPPING, inputs[r][0], inputs[r][1], cap, stream=streams[r])
        # place() blocks until the rank's host knows its base (the lower ranks' counts): one thread driving all ranks
        # has to place them in rank order (one process or thread per rank has no such constraint)
        for r in range(world):
            with torch.cuda.device(devices[r]):
                groups[r].place(jobs[r], bounds[r], r == world - 1, stream=streams[r])
        for r in reversed(range(1, world)):
            with torch.cuda.device(devices[r]):
                groups[r].finish(stream=streams[r])
        with torch.cuda.device(devices[0]):
            total = groups[0].finish(stream=streams[0])
            m, o = groups[0].result(total)
            assert total == whole.matches.shape[0]
            assert torch.equal(m, whole.matches) and torch.equal(o, whole.offsets)
            assert bool((m_all[total:] == sent32).all())
            m_all.fill_(sent32)
            o_all.fill_(sent64)
            torch.cuda.synchronize()
    for g in groups:
        g.close()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_shard_group_ranks_on_one_device(world):
    """The exchange protocol of dach_group_* (counts published, base waited for, matches stored into rank 0's
    buffer, done signalled) with all ranks on cuda:0 -- what needs two GPUs is only the NVLink under it."""
    _group_case(world, [0] * world)


def test_shard_group_across_devices():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    _group_case(2, [0, 1])
    if torch.cuda.device_count() >= 4:
        _group_case(4, [0, 1, 2, 3])


def test_bad_offsets_are_refused_on_both_paths():
    """ADVICE r1: a haystack of 4 GiB or more would be truncated silently (positions are u32); descending offsets
    or offsets past text_bytes would index outside the text.  Host path: checked before anything is copied.
    Device path: checked by a kernel before anything indexes with them; nothing is scanned."""
    import torch

    pma = D.DoubleArrayAhoCorasick.new(["ab", "b"])
    text = np.frombuffer(b"abab" * 64, dtype=np.uint8)
    for bad in ([0, 5 << 30], [0, 8, 4], [4, 0]):
        with pytest.raises(D.DaachorseError) as e:
            pma.scan_batch_host(D.FIND_OVERLAPPING, text, np.array(bad, dtype=np.uint64))
        assert e.value.code == 1
    dev = torch.device("cuda", 0)
    t = torch.from_numpy(text).to(dev)
    for bad in ([0, 8, 4, 16], [0, 1 << 33], [0, 100, 300]):
        with pytest.raises(D.DaachorseError) as e:
            pma.scan_batch_device(D.FIND_OVERLAPPING, t, torch.tensor(bad, dtype=torch.int64, device=dev))
        assert e.value.code == 1
    good = pma.scan_batch_device(D.FIND_OVERLAPPING, t, torch.tensor([0, 8, 8, 256], dtype=torch.int64, device=dev))
    assert good.matches.shape[0] == 4 + 4 + 124 + 124


@pytest.mark.parametrize("mode", [D.FIND, D.FIND_OVERLAPPING])
def test_charwise_stream_chunks_equal_the_stepper_over_the_whole_stream(mode):
    """dach_dev_scan_stream on a charwise automaton (src/charwise/iter.rs:403-534): 2000 streams of CJK text cut at
    char boundaries into ragged chunks, state and position carried from round to round."""
    import torch

    cfg = S.config("C4")
    ps = S.make_patterns(cfg, n=5000)
    pool, b = S.make_pool(cfg, ps, 4 << 20)
    rng = np.random.default_rng(33)
    n = 2000
    bi = np.sort(rng.integers(0, len(b) - 400, size=n))
    nt = rng.integers(0, 300, size=n)                      # tokens per stream
    streams, cuts = [], []
    for i in range(n):
        lo = int(b[bi[i]]); hi = int(b[bi[i] + int(nt[i])])
        streams.append(pool[lo:hi])
        cuts.append((b[bi[i]: bi[i] + int(nt[i]) + 1] - lo).astype(np.int64))   # token starts: char boundaries
    pma = D.CharwiseDoubleArrayAhoCorasick.new([p.decode() for p in ps.as_list()])
    opma = O.OraclePma.build([p.decode() for p in ps.as_list()], charwise=True)
    lens = np.array([len(x) for x in streams])
    offs_all = np.zeros(n + 1, dtype=np.uint64)
    offs_all[1:] = np.cumsum(lens)
    whole = np.concatenate(streams)
    ref = opma.scan_batch(O.FIND_STEPPER if mode == D.FIND else O.FIND_OVERLAPPING_STEPPER, whole, offs_all, nthreads=16, want_matches=True)
    state = torch.zeros(n, dtype=torch.int32, device="cuda")
    pos = np.zeros(n, dtype=np.int64)
    tok = np.zeros(n, dtype=np.int64)
    got = [[] for _ in range(n)]
    while (pos < lens).any():
        k = rng.integers(0, 60, size=n)
        chunks = []
        for i in range(n):
            t1 = min(int(tok[i] + k[i]), len(cuts[i]) - 1)
            chunks.append(streams[i][int(cuts[i][tok[i]]): int(cuts[i][t1])])
            tok[i] = t1
        offs = np.zeros(n + 1, dtype=np.int64)
        offs[1:] = np.cumsum([len(c) for c in chunks])
        text = np.concatenate(chunks) if offs[-1] else np.zeros(0, np.uint8)
        t = torch.from_numpy(np.ascontiguousarray(text)).cuda() if len(text) else torch.zeros(16, dtype=torch.uint8, device="cuda")[:0]
        r = pma.scan_stream_device(mode, t, torch.from_numpy(offs).cuda(), state, torch.from_numpy(pos.astype(np.int32)).cuda())
        m = r.matches.cpu().numpy().view(np.uint32).reshape(-1, 3)
        oo = r.offsets.cpu().numpy()
        for i in range(n):
            if oo[i + 1] > oo[i]:
                got[i].append(m[oo[i]: oo[i + 1]])
        pos += np.array([len(c) for c in chunks])
    rm = ref["matches"]
    ro = np.concatenate([[0], np.cumsum(ref["counts"])]).astype(np.int64)
    for i in range(n):
        want = np.stack([rm["start"][ro[i]: ro[i + 1]], rm["end"][ro[i]: ro[i + 1]], rm["value"][ro[i]: ro[i + 1]]], axis=1)
        want = want[want[:, 1] != 0]
        have = np.concatenate(got[i]) if got[i] else np.zeros((0, 3), np.uint32)
        assert np.array_equal(have, want), i


def test_python_daachorse_style_surface():
    """daachorse_b200.pycompat.Automaton: the surface of the crate's Python wrapper (README.md:19) -- str patterns,
    pattern indices as values, positions in characters."""
    from daachorse_b200 import pycompat as P

    pma = P.Automaton(["bcd", "ab", "a"])
    assert pma.find_overlapping("abcd") == [(0, 1, 2), (0, 2, 1), (1, 4, 0)]           # README.md:57-71
    ref = O.OraclePma.build(["bcd", "ab", "a"], charwise=True).scan_batch(
        O.FIND_OVERLAPPING_NO_SUFFIX, np.frombuffer(b"abcd", dtype=np.uint8), np.array([0, 4], dtype=np.uint64), want_matches=True)["matches"]
    assert pma.find_overlapping_no_suffix("abcd") == [(int(a), int(b), int(c)) for a, b, c in zip(ref["start"], ref["end"], ref["value"])]
    assert pma.find("abcd") == [(0, 1, 2), (1, 4, 0)]                                  # README.md:82-94
    pma = P.Automaton(["ab", "a", "abcd"], P.MATCH_KIND_LEFTMOST_LONGEST)
    assert pma.leftmost_find("abcd") == [(0, 4, 2)]                                    # README.md:102-116
    pma = P.Automaton(["ab", "a", "abcd"], P.MATCH_KIND_LEFTMOST_FIRST)
    assert pma.leftmost_find("abcd") == [(0, 2, 0)]                                    # README.md:128-142
    # positions are characters, not bytes
    pats = ["全世界", "世界", "に"]
    pma = P.Automaton(pats)
    hay = "全世界中に"
    got = pma.find_overlapping(hay)
    want = sorted((i, i + len(p), k) for k, p in enumerate(pats) for i in range(len(hay)) if hay.startswith(p, i))
    assert sorted(got) == want and pma.find_overlapping_as_strings(hay) == [hay[s:e] for s, e, _ in got]
    rng = np.random.default_rng(3)
    hays = ["".join(rng.choice(list("全世界中にab"), size=int(rng.integers(0, 40)))) for _ in range(50)]
    for h, r in zip(hays, pma.find_overlapping_batch(hays)):
        assert sorted(r) == sorted((i, i + len(p), k) for k, p in enumerate(pats) for i in range(len(h)) if h.startswith(p, i))
