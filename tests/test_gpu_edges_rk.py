"""Every result kind at the edges of the scan's contract, against the oracle on the same bytes:

  A  the largest legal haystack (2^32 - 1 bytes): the matches path on the lane machines (kernels 1-4, every segment
     length), COUNT, FIRST, HIST and DF on the default machine, the host COUNT of one haystack larger than any slice,
     and the refusal of a haystack of exactly 2^32 bytes by every entry point.  The 4 GiB haystack is zero bytes with
     short islands of pattern bytes; no pattern holds byte 0, so every Standard iterator is in ROOT after a zero byte
     and the expected matches are the oracle's on each island, shifted to its place.
     Not covered: find (not segmented), kernel 0, leftmost and charwise run one lane per haystack; one lane over
     4 GiB takes minutes.
  B  DF on the 2^32 address line and in guarded text (test_gpu_edges.py's batches), and DF's host-side check of
     device offsets;
  C  the host forms of COUNT, FIRST, HIST and DF over many slices: equal to one slice, to the device form and to the
     oracle, and nothing written beside the caller's views;
  D  launch shapes (threads, ctas_per_sm, reserve_sms, hist_smem) for COUNT, FIRST, HIST and DF;
  E  HIST's shared-memory counter passing 2^31 in one CTA: the hand-off to global memory at 2^31."""
import ctypes as C
import time

import numpy as np
import pytest

import daachorse_b200 as D
import oracle_api as O
from cases import seeded_reduce_case
from daachorse_b200 import _lib
from test_gpu_df import doc_freq
from test_gpu_edges import POISON, S32, S64, Auto, _guard_batch, _line_batches, _patterns, _u32, check_matches

pytestmark = pytest.mark.gpu
G4 = 1 << 32
HEAD, SHORT = 4096, 300  # offs[0], and the short haystacks beside the long one


def _torch():
    import torch

    return torch


def _release():
    """Hands the cached blocks of tensors the caller has dropped back to the device."""
    torch = _torch()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _sms():
    return _torch().cuda.get_device_properties(0).multi_processor_count


def _restore(pma):
    for k, v in (("kernel", 3), ("seg_len", 0), ("hot_entries", 6144), ("threads", 1024), ("ctas_per_sm", 1),
                 ("reserve_sms", 0), ("hist_smem", 1024), ("df_pairs", 1 << 24), ("slice_mib", 64), ("slice_ramp", 1)):
        pma.set_option(k, v)


def _keyed(a, want):
    """(key name, number of keys, key of every match) for both keys"""
    vals = want["value"].astype(np.int64)
    lens = want["end"].astype(np.int64) - want["start"].astype(np.int64)
    known = np.array(sorted((v << 32) | n for v, n in a.rec_of), dtype=np.int64)
    rec = np.array([a.rec_of[(int(k) >> 32, int(k) & 0xffffffff)] for k in known], dtype=np.int64)
    at = np.searchsorted(known, (vals << 32) | lens)
    assert np.array_equal(known[np.minimum(at, len(known) - 1)], (vals << 32) | lens)
    return (("value", a.n_val, vals), ("output", a.n_out, rec[at]))


# ---- A: the largest legal haystack -----------------------------------------------------------------------------------
def _qrs_patterns():
    rng = np.random.default_rng(41)
    pats = sorted({bytes(rng.integers(ord("q"), ord("s") + 1, size=int(rng.integers(1, 7))).tolist()) for _ in range(60)})
    assert pats and all(p and 0 not in p for p in pats)
    return pats


def _auto_seg_len(text_bytes, warm):
    """The segment length the scan picks itself (enqueue_scan / enqueue_rk: about two items per lane of SMs x 1024)."""
    want = max(text_bytes // (2 * _sms() * 1024) + 1, max(256, 8 * warm))
    return (want + 255) & ~255


def _islands(H, seg_lens, gap, rng):
    """[(pos, bytes)] inside [0, H): near the start, across 2^31, across the start of the last two segments of every
    length, inside the last 300 bytes and ending on the last byte; islands closer than `gap` are merged."""
    want = [(5, 11), ((1 << 31) - 4, 9), (H - 280, 13), (H - 7, 7)]
    for s in seg_lens:
        last = (H - 1) // s * s
        want += [(last - s - 3, 7), (last - 3, 7)]
    merged = []
    for p, n in sorted(w for w in want if 0 <= w[0] <= H - w[1]):
        if merged and p < merged[-1][1] + gap:
            merged[-1][1] = max(merged[-1][1], p + n)
        else:
            merged.append([p, p + n])
    return [(p, bytes(rng.integers(ord("q"), ord("s") + 1, size=min(e, H) - p).tolist())) for p, e in merged]


def _by_pieces(a, mode, hays):
    """Expected (matches, offsets) of haystacks given as [(pos, bytes)] pieces with zero bytes between them: the
    oracle on every piece, shifted by its position."""
    pieces = [p for h in hays for p in h]
    offs = np.zeros(len(pieces) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(b) for _, b in pieces])
    ref = a.opma.scan_batch({0: O.FIND, 1: O.FIND_OVERLAPPING, 2: O.FIND_OVERLAPPING_NO_SUFFIX}[mode],
                            np.frombuffer(b"".join(b for _, b in pieces), dtype=np.uint8), offs, want_matches=True)
    m, counts = ref["matches"].copy(), ref["counts"].astype(np.int64)
    m["start"] += np.repeat(np.array([p for p, _ in pieces], dtype=np.uint32), counts)
    m["end"] += np.repeat(np.array([p for p, _ in pieces], dtype=np.uint32), counts)
    per_hay = [int(counts[i: i + len(h)].sum()) for i, h in zip(np.cumsum([0] + [len(h) for h in hays[:-1]]), hays)]
    return m, np.concatenate([[0], np.cumsum(per_hay)]).astype(np.int64)


def test_a_islands_equal_a_whole_haystack_scan():
    """The construction of the expected lists, checked on a small haystack against one oracle scan of all of it."""
    a = Auto(False, 0, _qrs_patterns())
    rng = np.random.default_rng(2)
    H = 1 << 16
    isl = _islands(H, (64, 256, 4096), 6, rng)
    text = np.zeros(H, dtype=np.uint8)
    for p, b in isl:
        text[p: p + len(b)] = np.frombuffer(b, dtype=np.uint8)
    short = rng.integers(ord("q"), ord("s") + 1, size=SHORT).astype(np.uint8)
    both = np.concatenate([short, text, short])
    offs = np.array([0, SHORT, SHORT + H, 2 * SHORT + H], dtype=np.uint64)
    for mode in (1, 2):
        want, wo = a.oracle(mode, both, offs)
        got, go = _by_pieces(a, mode, [[(0, short.tobytes())], isl, [(0, short.tobytes())]])
        assert np.array_equal(go, wo) and got.tobytes() == want.tobytes(), mode
        assert int(wo[2] - wo[1]) > 0


def _reductions_default(a, mode, t, o, want, wo, tag):
    """COUNT, FIRST, HIST and DF (both keys) on the default machine; HIST and DF add into pre-filled buffers."""
    torch = _torch()
    counts = np.diff(wo)
    has = counts > 0
    if mode:  # find is one lane per haystack (FIRST runs find_overlapping's lanes for every Standard mode)
        assert np.array_equal(a.pma.count_batch_device(mode, t, o).cpu().numpy(), counts), (tag, mode)
    first, found = a.pma.first_batch_device(mode, t, o)
    assert np.array_equal(found.cpu().numpy(), has), (tag, mode)
    assert _u32(first)[has].tobytes() == want[wo[:-1][has]].view(np.uint32).tobytes(), (tag, mode)
    if not mode:
        return
    for key, k, keys in _keyed(a, want):
        for name, call, ref in (("hist", a.pma.pattern_counts_device, np.bincount(keys, minlength=k)),
                                ("df", a.pma.doc_counts_device, doc_freq(counts, keys, k).astype(np.int64))):
            pre = torch.arange(1, k + 9, dtype=torch.int64, device=t.device) * 1000
            got = (call(mode, t, o, key=key, out=pre.clone()) - pre).cpu().numpy()
            assert np.array_equal(got[:k], ref), (tag, mode, name, key)
            assert not got[k:].any(), (tag, mode, name, key, "written past the key range")


def test_a_largest_legal_haystack():
    torch = _torch()
    dev = torch.device("cuda", 0)
    a = Auto(False, 0, _qrs_patterns())
    warm = a.pma.max_pattern_len() - 1
    big = torch.zeros((4 << 30) + (8 << 20), dtype=torch.uint8, device=dev)
    try:
        rng = np.random.default_rng(43)
        nb0 = HEAD + 2 * SHORT + G4 - 1
        s_auto = _auto_seg_len(nb0, warm)
        # H = 2^32 - 1: the last segment of every power-of-two length ends at beg + seg_len == 2^32 exactly, the last
        # one of the automatic length (a multiple of 256 that does not divide 2^32) past it.  And H whose last
        # automatic segment holds one byte, so that the island on the last byte spans two segments.
        for H in (G4 - 1, (G4 - 1) // s_auto * s_auto + 1):
            nb = HEAD + 2 * SHORT + H
            assert _auto_seg_len(nb, warm) == s_auto
            big.zero_()
            shorts = [rng.integers(ord("q"), ord("s") + 1, size=SHORT).astype(np.uint8) for _ in range(2)]
            isl = _islands(H, (64, 256, 4096, s_auto), max(warm + 1, 8), rng)
            big[HEAD: HEAD + SHORT] = torch.from_numpy(shorts[0]).to(dev)
            big[HEAD + SHORT + H: nb] = torch.from_numpy(shorts[1]).to(dev)
            for p, b in isl:
                big[HEAD + SHORT + p: HEAD + SHORT + p + len(b)] = torch.from_numpy(np.frombuffer(b, dtype=np.uint8).copy()).to(dev)
            assert isl[-1][0] + len(isl[-1][1]) == H  # an island ends on the haystack's last byte
            t = big[:nb]
            o = torch.tensor([HEAD, HEAD + SHORT, HEAD + SHORT + H, nb], dtype=torch.int64, device=dev)
            hays = [[(0, shorts[0].tobytes())], isl, [(0, shorts[1].tobytes())]]
            a.machines = [{"kernel": k, "seg_len": s} for k in (1, 2, 3, 4) for s in (0, 64, 256, 4096)]
            for mode in (1, 2):
                want, wo = _by_pieces(a, mode, hays)
                assert int(wo[2] - wo[1]) > 0
                check_matches(a, mode, t, o, want, wo, ("largest", H))
            free, total = torch.cuda.mem_get_info()
            print("largest haystack %d: device memory in use after the matches path %.1f GiB" % (H, (total - free) / 2**30))
            for mode in (0, 1, 2):
                want, wo = _by_pieces(a, mode, hays)
                _reductions_default(a, mode, t, o, want, wo, ("largest", H))
            # only the island on the last byte is left: FIRST and COUNT of the long haystack depend on its last segment
            for p, b in isl[:-1]:
                big[HEAD + SHORT + p: HEAD + SHORT + p + len(b)] = 0
            for mode in (0, 1, 2):
                want, wo = _by_pieces(a, mode, [hays[0], isl[-1:], hays[2]])
                assert int(wo[2] - wo[1]) > 0
                _reductions_default(a, mode, t, o, want, wo, ("last segment only", H))
    finally:
        _restore(a.pma)
        a = None  # the device handle's workspace (segment tables and block pool of every seg_len)
        t = big = None  # the view and the 4 GiB tensor: nothing may keep the block alive
        _release()


def test_a_host_count_of_one_haystack_larger_than_any_slice():
    a = Auto(False, 0, _qrs_patterns())
    H = G4 - 1
    text = np.zeros(H, dtype=np.uint8)  # zero pages: nothing is touched but the island
    isl = _islands(H, (), 8, np.random.default_rng(44))[-1:]
    p, b = isl[0]
    text[p:] = np.frombuffer(b, dtype=np.uint8)
    want, wo = _by_pieces(a, 1, [isl])
    counts, total = a.pma.count_batch_host(1, text, np.array([0, H], dtype=np.uint64))
    assert counts.tolist() == [int(wo[1])] and total == int(wo[1]) > 0
    del a  # and with it the 4 GiB slice buffer of the device handle


def test_a_haystack_of_2_pow_32_bytes_is_refused_everywhere():
    torch = _torch()
    dev = torch.device("cuda", 0)
    L = _lib.load()
    a = Auto(False, 0, _qrs_patterns())
    d = a.pma.device_handle(0)
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    big = torch.zeros(G4 + 64, dtype=torch.uint8, device=dev)
    try:
        o = torch.tensor([8, 8 + G4], dtype=torch.int64, device=dev)
        tp, op, nb = C.c_void_p(big.data_ptr()), C.c_void_p(o.data_ptr()), big.numel()
        out = torch.full((64, 3), S32, dtype=torch.int32, device=dev)
        oo = torch.full((18,), S64, dtype=torch.int64, device=dev)
        need = C.c_uint64()
        IA = _lib.INVALID_ARGUMENT
        assert L.dach_dev_scan_batch(d, 1, tp, op, 1, nb, out.data_ptr(), 64, oo.data_ptr(), C.byref(need), st) == IA
        state = torch.zeros(1, dtype=torch.int32, device=dev)
        assert L.dach_dev_scan_stream(d, 1, tp, op, 1, nb, state.data_ptr(), None, out.data_ptr(), 64, oo.data_ptr(),
                                      C.byref(need), st) == IA
        j = C.c_void_p()
        assert L.dach_job_create(d, C.byref(j)) == 0
        try:
            assert L.dach_job_scan(j, 1, tp, op, 1, nb, 64, st) == 0
            assert L.dach_job_place(j, out.data_ptr(), 64, oo.data_ptr(), None, st) == 0
            assert L.dach_job_wait(j, C.byref(need)) == IA
        finally:
            L.dach_job_free(j)
        assert bool((out == S32).all()) and bool((oo == S64).all()), "a refused scan wrote matches or offsets"
        assert int(state[0]) == 0, "a refused stream chunk moved its state"
        cb = torch.full((1,), S64, dtype=torch.int64, device=dev)
        fb = torch.full((1, 3), S32, dtype=torch.int32, device=dev)
        gb = torch.full((1,), 0x5A, dtype=torch.uint8, device=dev)
        total = C.c_uint64()
        assert L.dach_dev_count_batch(d, 1, tp, op, 1, nb, cb.data_ptr(), C.byref(total), st) == IA
        assert L.dach_dev_first_batch(d, 1, tp, op, 1, nb, fb.data_ptr(), gb.data_ptr(), C.byref(total), st) == IA
        torch.cuda.synchronize()
        assert bool((cb == S64).all()) and bool((fb == S32).all()) and bool((gb == 0x5A).all())
        for fn in (L.dach_dev_hist_batch, L.dach_dev_df_batch):
            for key, k in ((0, a.n_out), (1, a.n_val)):
                prior = torch.arange(k, dtype=torch.int64, device=dev) + 7
                h = prior.clone()
                assert fn(d, 1, key, tp, op, 1, nb, h.data_ptr(), k, C.byref(total), st) == IA
                torch.cuda.synchronize()
                assert torch.equal(h, prior), (fn, key)
    finally:
        big = None
        _release()
    # the host forms refuse it before anything is copied (the array stays untouched zero pages)
    text = np.zeros(G4 + 8, dtype=np.uint8)
    offs = np.array([8, 8 + G4], dtype=np.uint64)
    for call in (lambda: a.pma.scan_batch_host(1, text, offs), lambda: a.pma.count_batch_host(1, text, offs),
                 lambda: a.pma.first_batch_host(1, text, offs), lambda: a.pma.pattern_counts_host(1, text, offs),
                 lambda: a.pma.doc_counts_host(1, text, offs)):
        with pytest.raises(D.DaachorseError) as e:
            call()
        assert e.value.code == _lib.INVALID_ARGUMENT


# ---- B: DF on the address line and in guarded text --------------------------------------------------------------------
DF_MACHINES = [{"kernel": 0}, {"kernel": 3}, {"hot_entries": 0}, {"seg_len": 64}, {"kernel": 3, "df_pairs": 1},
               {"kernel": 0, "df_pairs": 1}]


def check_df(a, mode, t, o, want, wo, tag):
    """DF (both keys) on the lane-per-haystack kernel, the lane machines and the smallest pair table, added into a
    longer, pre-filled buffer."""
    torch = _torch()
    counts = np.diff(wo)
    for opts in DF_MACHINES:
        if (opts.get("seg_len") and mode not in (1, 2)) or ((a.cw or a.kind) and ("seg_len" in opts or "hot_entries" in opts)):
            continue
        a.configure(opts)
        a.pma.set_option("df_pairs", opts.get("df_pairs", 1 << 24))
        for key, k, keys in _keyed(a, want):
            pre = torch.arange(1, k + 9, dtype=torch.int64, device=t.device) * 1000
            got = (a.pma.doc_counts_device(mode, t, o, key=key, out=pre.clone()) - pre).cpu().numpy()
            assert np.array_equal(got[:k], doc_freq(counts, keys, k).astype(np.int64)), (tag, mode, opts, key)
            assert not got[k:].any(), (tag, mode, opts, key, "df written past the key range")
    a.pma.set_option("df_pairs", 1 << 24)
    a.configure({})


def _autos():
    pats = _patterns()
    return [Auto(cw, kind, pats) for cw in (False, True) for kind in (0, 1, 2)]


def test_b_df_across_the_2_pow_32_address_line():
    torch = _torch()
    dev = torch.device("cuda", 0)
    big = torch.empty((4 << 30) + (8 << 20), dtype=torch.uint8, device=dev)
    try:
        ptr = big.data_ptr()
        line = ((ptr + (4 << 20)) >> 32 << 32) + (1 << 32)
        L = line - ptr
        rng = np.random.default_rng(11)
        window = rng.integers(97, 100, size=4 << 20).astype(np.uint8)
        big[L - (2 << 20): L + (2 << 20)] = torch.from_numpy(window).to(dev)
        autos = _autos()
        for lo, offs in _line_batches(rng):
            t = big[L + lo: L + lo + int(offs[-1])]
            o = torch.from_numpy(offs.astype(np.int64)).to(dev)
            h = window[(2 << 20) + lo: (2 << 20) + lo + int(offs[-1])]
            for a in autos:
                for mode in a.modes:
                    want, wo = a.oracle(mode, h, offs)
                    check_df(a, mode, t, o, want, wo, ("line", lo))
    finally:
        t = big = None
        _release()


@pytest.mark.parametrize("head", [0, 5], ids=["offs0_zero", "offs0_five"])
def test_b_df_guarded_text_every_shift(head):
    torch = _torch()
    dev = torch.device("cuda", 0)
    body, offs = _guard_batch()
    offs = offs + head
    nb = int(offs[-1])
    host = np.full(nb, POISON, dtype=np.uint8)
    host[head:] = np.frombuffer(body, dtype=np.uint8)
    o = torch.from_numpy(offs.astype(np.int64)).to(dev)
    autos = _autos()
    want = {(id(a), m): a.oracle(m, host, offs) for a in autos for m in a.modes}
    arena = torch.empty(1 << 16, dtype=torch.uint8, device=dev)
    for shift in range(16):
        arena.fill_(POISON)
        t = arena[256 + shift: 256 + shift + nb]
        t.copy_(torch.from_numpy(host).to(dev))
        for a in autos:
            for mode in a.modes:
                w, wo = want[(id(a), mode)]
                check_df(a, mode, t, o, w, wo, ("guard", shift))


def test_b_df_device_offsets_checked_on_the_host():
    """dach_dev_df_batch copies the offsets to the host and checks them there: descending ones, ones past text_bytes
    and (part A) a haystack of 2^32 bytes are refused before any window runs and leave df as it was; offs[0] > 0
    with poison below it counts only the haystacks."""
    torch = _torch()
    dev = torch.device("cuda", 0)
    a = Auto(False, 0, _patterns())
    rng = np.random.default_rng(8)
    lens = rng.integers(0, 200, size=400)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64) + 64
    host = rng.integers(97, 100, size=int(offs[-1])).astype(np.uint8)
    host[:64] = POISON
    t = torch.from_numpy(host).to(dev)
    k = a.n_val
    prior = torch.arange(k, dtype=torch.int64, device=dev) * 3
    for pairs in (1 << 24, 1):
        a.pma.set_option("df_pairs", pairs)
        desc = offs.copy()
        desc[200] = desc[199] - 1
        for bad in (desc,                                                 # descending in the middle
                    np.concatenate([offs[:-1], [offs[-1] + 1]]),          # past text_bytes
                    np.concatenate([[offs[-1] + 1], offs[1:]])):          # offs[0] past the text
            d = prior.clone()
            with pytest.raises(D.DaachorseError) as e:
                a.pma.doc_counts_device(1, t, torch.from_numpy(bad.astype(np.int64)).to(dev), out=d)
            assert e.value.code == _lib.INVALID_ARGUMENT and torch.equal(d, prior), (pairs, bad[:3])
        for mode in (0, 1, 2):
            want, wo = a.oracle(mode, host, offs)
            got = a.pma.doc_counts_device(mode, t, torch.from_numpy(offs.astype(np.int64)).to(dev), out=prior.clone()) - prior
            assert np.array_equal(got.cpu().numpy(), doc_freq(np.diff(wo), want["value"], k).astype(np.int64)), (pairs, mode)
    a.pma.set_option("df_pairs", 1 << 24)


# ---- C: host forms across slices --------------------------------------------------------------------------------------
def _cuts(offs, slice_bytes):
    """Where the host forms cut a batch for find_overlapping at 1 MiB slices (cut_slices in dev_scan.cu, whose slices
    never go below 1 MiB, ramp or not): the index of every slice's first haystack after the first."""
    n, i, cuts = len(offs) - 1, 0, []
    while i < n:
        j = i + 1
        if j < n and offs[j + 1] <= offs[i] + slice_bytes:
            j = int(np.searchsorted(offs, offs[i] + slice_bytes, side="right")) - 1
        if j < n:
            cuts.append(j)
        i = j
    return cuts


def _sliced_batch():
    """About 40 MiB over "abcd": haystacks of 0-6000 bytes, 8 % of them empty, one of 3 MiB, and two empty haystacks
    closing every 1 MiB slice."""
    rng = np.random.default_rng(31)
    lens = rng.integers(0, 6000, size=13000)
    lens[rng.random(lens.size) < 0.08] = 0
    lens[6500] = 3 << 20
    cuts = _cuts(np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64), 1 << 20)
    lens = np.insert(lens, np.repeat(cuts, 2), 0)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    cuts = _cuts(offs, 1 << 20)
    # every slice ends in two empty haystacks, but the 3 MiB one's (a slice of its own: the empties open the next)
    assert len(cuts) > 30 and all(lens[j - 1] == lens[j - 2] == 0 or (lens[j - 1] > (1 << 20) and lens[j] == 0) for j in cuts)
    text = rng.integers(97, 101, size=int(offs[-1])).astype(np.uint8)
    pats = sorted({bytes(rng.integers(97, 101, size=int(rng.integers(3, 9))).tolist()) for _ in range(200)})
    return pats, text, offs


def _host_results(pma, text, offs, modes, tables=(1 << 24,)):
    r = {}
    for mode in modes:
        r[("count", mode)] = pma.count_batch_host(mode, text, offs)[0]
        f, g = pma.first_batch_host(mode, text, offs)
        r[("first", mode)] = (f.tobytes(), g.tobytes())
        for key in ("value", "output"):
            r[("hist", mode, key)] = pma.pattern_counts_host(mode, text, offs, key=key)
            for pairs in tables:
                pma.set_option("df_pairs", pairs)
                r[("df", mode, key, pairs)] = pma.doc_counts_host(mode, text, offs, key=key)
            pma.set_option("df_pairs", 1 << 24)
    return r


def _device_results(pma, text, offs, modes):
    torch = _torch()
    t, o = torch.from_numpy(text).cuda(), torch.from_numpy(offs.astype(np.int64)).cuda()
    r = {}
    for mode in modes:
        r[("count", mode)] = pma.count_batch_device(mode, t, o).cpu().numpy().astype(np.uint64)
        f, g = pma.first_batch_device(mode, t, o)
        f = f.cpu().numpy().view(np.uint32).reshape(-1)
        r[("first", mode)] = (f.view(D.MATCH_DTYPE).tobytes(), g.cpu().numpy().astype(np.uint8).view(bool).tobytes())
        for key in ("value", "output"):
            r[("hist", mode, key)] = pma.pattern_counts_device(mode, t, o, key=key).cpu().numpy().astype(np.uint64)
            for pairs in (1 << 24, 1):
                pma.set_option("df_pairs", pairs)
                r[("df", mode, key, pairs)] = pma.doc_counts_device(mode, t, o, key=key).cpu().numpy().astype(np.uint64)
            pma.set_option("df_pairs", 1 << 24)
    return r


def _oracle_results(a, text, offs, modes):
    r = {}
    for mode in modes:
        want, wo = a.oracle(mode, text, offs)
        counts = np.diff(wo)
        r[("count", mode)] = counts.astype(np.uint64)
        has = counts > 0
        f = np.full(len(counts), 0xFF, dtype=np.uint8).repeat(12).view(D.MATCH_DTYPE)
        f[has] = want[wo[:-1][has]]
        r[("first", mode)] = (f.tobytes(), has.tobytes())
        for key, k, keys in _keyed(a, want):
            r[("hist", mode, key)] = np.bincount(keys, minlength=k).astype(np.uint64)
            for pairs in (1 << 24, 1):
                r[("df", mode, key, pairs)] = doc_freq(counts, keys, k)
    return r


def _same(x, y):
    return all(np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b for a, b in zip(x, y)) \
        if isinstance(x, tuple) else np.array_equal(x, y)


@pytest.mark.parametrize("kind", [0, 1])
def test_c_host_reductions_across_many_slices(kind):
    pats, text, offs = _sliced_batch()
    a = Auto(False, kind, pats)
    modes = (3,) if kind else (0, 1, 2)
    sub = offs[5:-5]  # a view that does not start at offset 0
    for view in (offs, sub):
        ref = _oracle_results(a, text, view, modes)
        dref = _device_results(a.pma, text, view, modes)
        a.pma.set_option("slice_mib", 1 << 20)
        one = _host_results(a.pma, text, view, modes)
        for ramp in (0, 1):
            a.pma.set_option("slice_ramp", ramp)
            a.pma.set_option("slice_mib", 1)
            # the smallest pair table too: windows of a few haystacks, most scanned again as halves
            many = _host_results(a.pma, text, view, modes, (1 << 24, 1))
            for k in many:
                assert _same(many[k], one[k[:3] + (1 << 24,) if k[0] == "df" else k]), (k, ramp, "many slices != one slice")
                assert _same(many[k], dref[k]), (k, ramp, "host != device")
                assert _same(many[k], ref[k]), (k, ramp, "host != oracle")
        _restore(a.pma)


def test_c_host_views_inside_sentinel_buffers():
    """The C ABI on views inside sentinel-filled arrays, with 1 MiB slices: COUNT, FIRST and found write nothing
    outside [0, n), HIST and DF nothing past n_hist."""
    pats, text, offs = _sliced_batch()
    a = Auto(False, 0, pats)
    L = _lib.load()
    d = a.pma.device_handle(0)
    n = len(offs) - 1
    tp, op = C.c_void_p(text.ctypes.data), C.c_void_p(offs.ctypes.data)
    a.pma.set_option("slice_mib", 1)
    for mode in (0, 1):
        want, wo = a.oracle(mode, text, offs)
        counts = np.diff(wo)
        cb = np.full(n + 8, S64, dtype=np.uint64)
        fb = np.full((n + 8) * 3, S32, dtype=np.uint32)
        gb = np.full(n + 8, 0x5A, dtype=np.uint8)
        total = C.c_uint64()
        assert L.dach_count_batch_host(d, mode, tp, op, n, C.c_void_p(cb[4:].ctypes.data), C.byref(total)) == 0
        assert L.dach_first_batch_host(d, mode, tp, op, n, C.c_void_p(fb[12:].ctypes.data), C.c_void_p(gb[4:].ctypes.data),
                                       C.byref(total)) == 0
        assert np.array_equal(cb[4: 4 + n], counts) and np.array_equal(gb[4: 4 + n], counts > 0)
        for buf, s, w in ((cb, S64, 1), (fb, S32, 3), (gb, 0x5A, 1)):
            assert (buf[: 4 * w] == s).all() and (buf[(4 + n) * w:] == s).all(), (mode, "written beside the view")
        for fn in (L.dach_hist_batch_host, L.dach_df_batch_host):
            for key, k, keys in _keyed(a, want):
                ref = np.bincount(keys, minlength=k) if fn is L.dach_hist_batch_host else doc_freq(counts, keys, k)
                h = np.full(k + 8, 5, dtype=np.uint64)
                assert fn(d, mode, 1 if key == "value" else 0, tp, op, n, C.c_void_p(h.ctypes.data), k, C.byref(total)) == 0
                assert np.array_equal(h[:k] - np.uint64(5), ref.astype(np.uint64)), (mode, key)
                assert (h[k:] == 5).all(), (mode, key, "written past n_hist")
    _restore(a.pma)


# ---- D: launch shapes ---------------------------------------------------------------------------------------------------
def _shapes():
    sms = _sms()
    return ([{"threads": t} for t in (128, 256, 512, 768)] + [{"threads": t, "ctas_per_sm": 2} for t in (512, 768)] +
            [{"reserve_sms": sms - 1}])


@pytest.mark.parametrize("cw", [False, True])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_d_reductions_under_every_launch_shape(cw, kind):
    torch = _torch()
    pats, text, offs = seeded_reduce_case(cw, kind)  # the batches of test_gpu_hist.py
    pma = (D.CharwiseDoubleArrayAhoCorasickBuilder if cw else D.DoubleArrayAhoCorasickBuilder).new().match_kind(kind).build(pats)
    t, o = torch.from_numpy(np.ascontiguousarray(text)).cuda(), torch.from_numpy(offs.astype(np.int64)).cuda()

    def results(mode):
        f, g = pma.first_batch_device(mode, t, o)
        r = {"count": pma.count_batch_device(mode, t, o), "first": f, "found": g}
        for key in ("value", "output"):
            r["df", key] = pma.doc_counts_device(mode, t, o, key=key)
        return r

    def hists(mode):
        return {key: pma.pattern_counts_device(mode, t, o, key=key) for key in ("value", "output")}

    try:
        for mode in ([D.LEFTMOST_FIND] if kind else [D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX]):
            pma.set_option("kernel", 0)
            base, hbase = results(mode), hists(mode)
            pma.set_option("kernel", 3)
            assert int(base["count"].sum()) > 0
            for shape in _shapes():
                for k, v in shape.items():
                    pma.set_option(k, v)
                got = results(mode)
                for k in base:
                    assert torch.equal(got[k], base[k]), (mode, shape, k)
                for hs in (0, 1024, 1 << 20):
                    pma.set_option("hist_smem", hs)
                    got = hists(mode)
                    for k in hbase:
                        assert torch.equal(got[k], hbase[k]), (mode, shape, hs, k)
                _restore(pma)
    finally:
        _restore(pma)


# ---- E: the 2^31 hand-off of HIST's shared-memory counter -------------------------------------------------------------
def test_e_hist_shared_counter_passes_2_pow_31_in_one_cta():
    """Patterns ["a"], find_overlapping, one CTA, 4 GiB + 16 MiB of "a" in two haystacks: every byte is one event on
    the state of "a", which counts in shared memory (hist_smem is clamped to the compact slots), so the CTA's counter
    passes 2^31 twice; each time 2^31 is handed on to global memory."""
    torch = _torch()
    dev = torch.device("cuda", 0)
    N = (4 << 30) + (16 << 20)
    pma = D.DoubleArrayAhoCorasick.new(["a"])
    big = torch.full((N,), 97, dtype=torch.uint8, device=dev)
    try:
        o = torch.tensor([0, N // 2, N], dtype=torch.int64, device=dev)
        pma.set_option("reserve_sms", _sms() - 1)
        pma.set_option("ctas_per_sm", 1)
        for hs in (1024, 1 << 20, 0):
            pma.set_option("hist_smem", hs)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            h = pma.pattern_counts_device(D.FIND_OVERLAPPING, big, o)
            torch.cuda.synchronize()
            print("hist_smem %d: one CTA over %d bytes in %.2f s" % (hs, N, time.perf_counter() - t0))
            assert h.tolist() == [N], hs
    finally:
        _restore(pma)
        big = None
        _release()
