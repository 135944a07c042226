"""Masked text on the GPU (dach_dev_mask_batch / dach_mask_batch_host): byte for byte against the matches path of the
same batch turned into spans (tests/emu_mask_api.py's expected_mask), and against the oracle where the batch is small.
Every kernel option that changes which kernel runs, guarded and shifted buffers, the 2^32 address line, refusals."""
import json
import os

import numpy as np
import pytest

import daachorse_b200 as D
import emu_mask_api as M
import oracle_api as O
from cases import mixed_width_case, seeded_reduce_case
from daachorse_b200 import _lib
from daachorse_b200 import synth as S

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "search_tests.json"), encoding="utf-8"))
ORC = {D.FIND: O.FIND, D.FIND_OVERLAPPING: O.FIND_OVERLAPPING,
       D.FIND_OVERLAPPING_NO_SUFFIX: O.FIND_OVERLAPPING_NO_SUFFIX, D.LEFTMOST_FIND: O.LEFTMOST_FIND}
GMODE = {"find_iter": D.FIND, "find_overlapping_iter": D.FIND_OVERLAPPING,
         "find_overlapping_no_suffix_iter": D.FIND_OVERLAPPING_NO_SUFFIX, "leftmost_find_iter": D.LEFTMOST_FIND}
FILL = 0x23
POISON = 0xA5


def builder(cw):
    return D.CharwiseDoubleArrayAhoCorasickBuilder if cw else D.DoubleArrayAhoCorasickBuilder


def modes(kind):
    return [D.LEFTMOST_FIND] if kind else [D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX]


def dev(text, offs):
    import torch

    t = torch.from_numpy(np.ascontiguousarray(text)).cuda() if len(text) else torch.zeros(0, dtype=torch.uint8, device="cuda")
    return t, torch.from_numpy(offs.astype(np.int64)).cuda()


def from_matches(pma, mode, text, offs, fill=FILL):
    """expected_mask of dach_scan_batch_host's match list"""
    r = pma.scan_batch_host(mode, text, offs)
    return M.expected_from_matches(text, offs, r.matches, np.diff(r.offsets.astype(np.int64)), fill)


def from_oracle(opma, mode, text, offs, fill=FILL):
    ref = opma.scan_batch(ORC[mode], text, offs, want_matches=True)
    return M.expected_from_matches(text, offs, ref["matches"], ref["counts"], fill)


def check(pma, mode, text, offs, want, fill=FILL, tag=None):
    """device form (fresh and preallocated out) and host form == want"""
    import torch

    t, o = dev(text, offs)
    got = pma.mask_batch_device(mode, t, o, fill=fill)
    assert np.array_equal(got.cpu().numpy(), want), (tag, mode, np.flatnonzero(got.cpu().numpy() != want)[:8])
    out = torch.full_like(t, POISON)
    assert pma.mask_batch_device(mode, t, o, fill=fill, out=out) is out
    assert torch.equal(out, got)
    assert np.array_equal(pma.mask_batch_host(mode, text, offs, fill=fill), want), (tag, mode, "host")


OPTIONS = (("kernel", (0, 1, 2, 4, 3)), ("hot_entries", (0, -2)), ("seg_len", (64, 256, -1, 0)))


@pytest.mark.parametrize("cw", [False, True])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_seeded_batches_and_options(cw, kind):
    pats, text, offs = seeded_reduce_case(cw, kind)
    pma = builder(cw).new().match_kind(kind).build(pats)
    opma = O.OraclePma.build(pats, charwise=cw, match_kind=kind)
    for mode in modes(kind):
        want = from_oracle(opma, mode, text, offs)
        assert np.array_equal(from_matches(pma, mode, text, offs), want)
        check(pma, mode, text, offs, want)
        for name, values in OPTIONS:
            for v in values:
                pma.set_option(name, v)
                check(pma, mode, text, offs, want, tag=(name, v))


def test_golden_vectors():
    for variant, iterator, coll, kind in GOLD["configs"]:
        if iterator not in GMODE:
            continue
        cw = variant == "charwise"
        for g in GOLD["collections"][coll]:
            for t in GOLD["groups"][g]:
                pma = builder(cw).new().match_kind(O.KIND[kind]).build(t["patterns"])
                opma = O.OraclePma.build(t["patterns"], charwise=cw, match_kind=O.KIND[kind])
                hay = t["haystack"].encode()
                text = np.frombuffer(hay, dtype=np.uint8)
                offs = np.array([0, len(hay)], dtype=np.uint64)
                mode = GMODE[iterator]
                want = from_oracle(opma, mode, text, offs)
                assert np.array_equal(from_matches(pma, mode, text, offs), want), t["name"]
                check(pma, mode, text, offs, want, tag=t["name"])


@pytest.mark.parametrize("seed", [0, 3, 4])
def test_charwise_mixed_widths_stay_utf8(seed):
    kind, pats, text, offs = mixed_width_case(seed)
    pma = D.CharwiseDoubleArrayAhoCorasickBuilder.new().match_kind(kind).build(pats)
    for mode in modes(kind):
        want = from_matches(pma, mode, text, offs, fill=ord("_"))
        check(pma, mode, text, offs, want, fill=ord("_"))
        want.tobytes().decode("utf-8")
    got = pma.mask_batch(["𝄞aé" * 3, ""], fill="_")
    assert all(isinstance(s, str) for s in got)


def test_mask_batch_convenience():
    p = D.DoubleArrayAhoCorasick.new(["ab", "bc", "x"])
    assert p.mask_batch([b"abc", b"", b"zxz", b"ab"]) == [b"***", b"", b"z*z", b"**"]
    assert p.mask_batch(["abc"], fill=b"-", mode=D.FIND) == [b"--c"]
    lm = D.DoubleArrayAhoCorasickBuilder.new().match_kind(D.MatchKind.LeftmostLongest).build(["ab", "abc"])
    assert lm.mask_batch([b"xabcd"], fill=0) == [b"x\x00\x00\x00d"]


@pytest.mark.parametrize("name", ["C2", "C3"])
def test_synthetic_workloads(name):
    """C2 and a 64 MiB batch of C3 (the bench workloads' automata and text), compared in full."""
    import torch

    cfg = S.config(name, 1.0 / 64)
    ps = S.make_patterns(cfg)
    pma = D.DoubleArrayAhoCorasick.new(ps.as_list())
    size = (64 << 20) if name == "C3" else (16 << 20)
    pool, bounds = S.make_pool(cfg, ps, size, seed=2)
    n = size // cfg["hay_len"]
    starts = S.window_starts(bounds, len(pool), n, cfg["hay_len"], seed=3)
    t, o = S.materialise_on_device(torch.from_numpy(pool).cuda(), torch.from_numpy(starts).cuda(), cfg["hay_len"])
    text, offs = t.cpu().numpy(), o.cpu().numpy().astype(np.uint64)
    for mode in (D.FIND_OVERLAPPING, D.FIND):
        r = pma.scan_batch_device(mode, t, o)
        m = r.matches.cpu().numpy().astype(np.int64)
        hay = np.repeat(np.arange(len(offs) - 1), np.diff(r.offsets.cpu().numpy()))
        want = M.expected_mask(text, offs, m[:, 0], m[:, 1], hay, FILL)
        del r, m
        got = pma.mask_batch_device(mode, t, o, fill=FILL)
        assert np.array_equal(got.cpu().numpy(), want), (name, mode)
        del got
    if name == "C2":
        assert np.array_equal(pma.mask_batch_host(D.FIND_OVERLAPPING, text, offs, fill=FILL),
                              from_matches(pma, D.FIND_OVERLAPPING, text, offs))


def _guard_case():
    pats = [b"ab", b"b", b"abcab", b"cab", b"a" * 9]
    rng = np.random.default_rng(5)
    lens = [0, 1, 15, 16, 17, 31, 33, 100, 5]
    body = rng.integers(97, 100, size=sum(lens)).astype(np.uint8)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    return pats, body, offs


@pytest.mark.parametrize("head", [0, 5], ids=["offs0_zero", "offs0_five"])
def test_shifted_and_guarded_buffers(head):
    """text and out at every base shift 0-15 against each other, poison before and after both: the copy kernel's
    16-byte path at every relative alignment, its ragged ends, and nothing written outside out."""
    import torch

    pats, body, offs = _guard_case()
    offs = offs + np.uint64(head)
    host = np.concatenate([np.full(head, 0x7A, np.uint8), body, np.full(3, 0x61, np.uint8)])  # bytes after offs[n]
    nb = host.size
    pma = D.DoubleArrayAhoCorasick.new(pats)
    o = torch.from_numpy(offs.astype(np.int64)).cuda()
    want = {m: from_matches(pma, m, host, offs) for m in (D.FIND, D.FIND_OVERLAPPING)}
    for m in want:
        assert np.array_equal(want[m][:head], host[:head]) and np.array_equal(want[m][-3:], host[-3:])
    arena_t = torch.empty(1 << 12, dtype=torch.uint8, device="cuda")
    arena_o = torch.empty(1 << 12, dtype=torch.uint8, device="cuda")
    for opts in ({"kernel": 3}, {"kernel": 0}):
        for k, v in opts.items():
            pma.set_option(k, v)
        for st in range(16):
            arena_t.fill_(POISON)
            t = arena_t[256 + st: 256 + st + nb]
            t.copy_(torch.from_numpy(host).cuda())
            for so in range(16):
                arena_o.fill_(POISON)
                out = arena_o[512 + so: 512 + so + nb]
                for mode, w in want.items():
                    pma.mask_batch_device(mode, t, o, fill=FILL, out=out)
                    assert np.array_equal(out.cpu().numpy(), w), (opts, st, so, mode)
                    assert (arena_o[:512 + so] == POISON).all() and (arena_o[512 + so + nb:] == POISON).all()
            assert np.array_equal(t.cpu().numpy(), host)
    pma.set_option("kernel", 3)


def test_large_copy_every_relative_alignment():
    """A few MiB through the copy kernel at every relative alignment, with no haystack and with one."""
    import torch

    p = D.DoubleArrayAhoCorasick.new(["\x01\x02\x03"])
    rng = np.random.default_rng(9)
    nb = (3 << 20) + 7
    host = rng.integers(0, 256, size=nb).astype(np.uint8)
    src = torch.from_numpy(np.concatenate([host, np.zeros(32, np.uint8)])).cuda()
    dst = torch.empty(nb + 64, dtype=torch.uint8, device="cuda")
    for a in range(16):
        t = src[:nb] if a == 0 else torch.empty(nb + 16, dtype=torch.uint8, device="cuda")[a: a + nb].copy_(src[:nb])
        for offs in (np.array([7], dtype=np.uint64), np.array([11, nb - 13], dtype=np.uint64)):
            want = from_matches(p, D.FIND, host, offs) if len(offs) > 1 else host
            dst.fill_(POISON)
            out = dst[3: 3 + nb]
            p.mask_batch_device(D.FIND, t, torch.from_numpy(offs.astype(np.int64)).cuda(), fill=0, out=out)
            assert np.array_equal(out.cpu().numpy(), want), (a, len(offs))
            assert (dst[:3] == POISON).all() and (dst[3 + nb:] == POISON).all()


def test_across_the_2_pow_32_address_line():
    import torch

    big = torch.empty((4 << 30) + (8 << 20), dtype=torch.uint8, device="cuda")
    outb = None
    try:
        ptr = big.data_ptr()
        line = ((ptr + (4 << 20)) >> 32 << 32) + (1 << 32)
        L = line - ptr
        rng = np.random.default_rng(11)
        window = rng.integers(97, 100, size=4 << 20).astype(np.uint8)
        pats = [bytes(rng.integers(97, 100, size=int(rng.integers(1, 6))).tolist()) for _ in range(40)]
        pma = D.DoubleArrayAhoCorasick.new(pats)
        lens = rng.integers(0, 5000, size=300)
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
        lo = -int(offs[-1]) // 2
        big[L + lo: L + lo + int(offs[-1])] = torch.from_numpy(window[:int(offs[-1])]).cuda()
        t = big[L + lo: L + lo + int(offs[-1])]
        o = torch.from_numpy(offs.astype(np.int64)).cuda()
        h = window[:int(offs[-1])]
        for mode in (D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX):
            want = from_matches(pma, mode, h, offs)
            for opts in ({"kernel": 3, "seg_len": 0}, {"kernel": 3, "seg_len": 64}, {"kernel": 0}):
                for k, v in opts.items():
                    pma.set_option(k, v)
                got = pma.mask_batch_device(mode, t, o, fill=FILL)
                assert np.array_equal(got.cpu().numpy(), want), (mode, opts)
            pma.set_option("seg_len", 0)
        # the output across the line, the text away from it
        src = torch.from_numpy(h).cuda()
        outb = big[L - int(offs[-1]) // 3: L - int(offs[-1]) // 3 + int(offs[-1])]
        pma.mask_batch_device(D.FIND_OVERLAPPING, src, o, fill=FILL, out=outb)
        assert np.array_equal(outb.cpu().numpy(), from_matches(pma, D.FIND_OVERLAPPING, h, offs))
    finally:
        t = big = outb = None
        torch.cuda.empty_cache()


def test_refusals_leave_out_untouched():
    import torch

    p = D.DoubleArrayAhoCorasick.new(["a", "b"])
    cw = D.CharwiseDoubleArrayAhoCorasick.new(["a"])
    t = torch.from_numpy(np.frombuffer(b"abcabc", dtype=np.uint8).copy()).cuda()
    out = torch.full((6,), POISON, dtype=torch.uint8, device="cuda")
    for offs in ([0, 4, 2], [0, 7], [3, 1]):
        with pytest.raises(D.DaachorseError) as e:
            p.mask_batch_device(D.FIND, t, torch.tensor(offs, dtype=torch.int64, device="cuda"), out=out)
        assert e.value.code == _lib.INVALID_ARGUMENT
        assert (out == POISON).all()
    o = torch.tensor([0, 6], dtype=torch.int64, device="cuda")
    for bad_out in (t, t[2:], torch.empty(5, dtype=torch.uint8, device="cuda"), torch.empty(6, dtype=torch.int32, device="cuda")):
        with pytest.raises(D.DaachorseError) as e:
            p.mask_batch_device(D.FIND, t, o, out=bad_out)
        assert e.value.code == _lib.INVALID_ARGUMENT
    with pytest.raises(D.DaachorseError) as e:
        cw.mask_batch_device(D.FIND, t, o, fill=0x80)
    assert e.value.code == _lib.INVALID_ARGUMENT
    # the C ABI's own checks: overlap and a non-ASCII charwise fill, before anything runs
    import ctypes as C

    L = _lib.load()
    h = p.device_handle(0)
    assert L.dach_dev_mask_batch(h, D.FIND, C.c_void_p(t.data_ptr()), C.c_void_p(o.data_ptr()), 1, 6, 42,
                                 C.c_void_p(t.data_ptr() + 3), None) == _lib.INVALID_ARGUMENT
    assert L.dach_dev_mask_batch(cw.device_handle(0), D.FIND, C.c_void_p(t.data_ptr()), C.c_void_p(o.data_ptr()), 1, 6, 0xC3,
                                 C.c_void_p(out.data_ptr()), None) == _lib.INVALID_ARGUMENT
    assert (out == POISON).all()
    assert L.dach_dev_mask_batch(h, D.LEFTMOST_FIND, C.c_void_p(t.data_ptr()), C.c_void_p(o.data_ptr()), 1, 6, 42,
                                 C.c_void_p(out.data_ptr()), None) == _lib.MATCH_KIND_MISMATCH


def test_empty_batches():
    import torch

    p = D.DoubleArrayAhoCorasick.new(["a"])
    t = torch.from_numpy(np.frombuffer(b"aaxa", dtype=np.uint8).copy()).cuda()
    o0 = torch.tensor([2], dtype=torch.int64, device="cuda")
    assert torch.equal(p.mask_batch_device(D.FIND, t, o0), t)  # n = 0: a copy
    e = torch.zeros(0, dtype=torch.uint8, device="cuda")
    assert p.mask_batch_device(D.FIND, e, torch.zeros(1, dtype=torch.int64, device="cuda")).numel() == 0
    assert p.mask_batch_device(D.FIND, e, torch.zeros(3, dtype=torch.int64, device="cuda")).numel() == 0
    assert p.mask_batch_host(D.FIND, np.zeros(0, np.uint8), np.zeros(1, np.uint64)).size == 0
    h = np.frombuffer(b"aaxa", dtype=np.uint8)
    assert np.array_equal(p.mask_batch_host(D.FIND, h, np.array([2], dtype=np.uint64)), h)
    assert p.mask_batch([]) == []


def test_host_form_over_many_slices():
    """slice_mib = 1 cuts the batch into many slices: equal to one slice and to the device form."""
    pats, text, offs = seeded_reduce_case(False, 0)
    reps = 4
    big = np.tile(text, reps)
    boffs = np.concatenate([offs[:-1] + np.uint64(k * text.size) for k in range(reps)] + [[np.uint64(reps * text.size)]])
    boffs = boffs.astype(np.uint64)
    pma = D.DoubleArrayAhoCorasick.new(pats)
    for mode in (D.FIND_OVERLAPPING, D.FIND):
        t, o = dev(big, boffs)
        want = pma.mask_batch_device(mode, t, o).cpu().numpy()
        pma.set_option("slice_mib", 1)
        many = pma.mask_batch_host(mode, big, boffs)
        pma.set_option("slice_mib", 4096)
        one = pma.mask_batch_host(mode, big, boffs)
        pma.set_option("slice_mib", 64)
        assert np.array_equal(many, want) and np.array_equal(one, want)


def test_launch_shapes():
    pats, text, offs = seeded_reduce_case(False, 0)
    pma = D.DoubleArrayAhoCorasick.new(pats)
    want = from_matches(pma, D.FIND_OVERLAPPING, text, offs)
    for name, v in (("threads", 256), ("threads", 96), ("ctas_per_sm", 2), ("reserve_sms", 1 << 20)):
        pma.set_option(name, v)
        check(pma, D.FIND_OVERLAPPING, text, offs, want, tag=(name, v))
    for name, v in (("threads", 1024), ("ctas_per_sm", 1), ("reserve_sms", 0)):
        pma.set_option(name, v)
