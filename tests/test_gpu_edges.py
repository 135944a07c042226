"""The device scan at the edges of its contract, against the oracle on the same bytes copied to the host:

  A  the 2^32 address line: StdMachine3's cursor is the low word of the text address (Lane3::ap, block_of adds the
     carry back), so haystacks, segments and stream chunks are placed across a multiple of 2^32 in device memory;
  B  guarded text: the batch sits at every base shift 0-15 with poison before it, between d_text and offs[0], and
     after text_end -- bytes that would add or extend matches if a kernel read them as text;
  C  output slack: nothing outside [base, base + needed) of d_out, past n + 1 offsets, past the key range of a
     histogram, beside COUNT / FIRST views or past out_cap on overflow is written;
  D  jobs of every iterator (event expansion with and without lists, leftmost and charwise tuple gathers), with and
     without a device-side base, and a job that overflows and is reused;
  E  needed past 2^32 matches in one haystack: exact, and the scan is refused rather than reported as an overflow.

"Every machine": bytewise Standard kernels 0-4, hot_entries 0, forced segments, gather_ordered 0 / 2; LmMachine;
CwMachine.  "Every result kind": matches, COUNT, FIRST, HIST by value and by output record, stream chunks."""
import ctypes as C

import numpy as np
import pytest

import daachorse_b200 as D
import oracle_api as O
from daachorse_b200 import _lib

pytestmark = pytest.mark.gpu
ORC = {0: O.FIND, 1: O.FIND_OVERLAPPING, 2: O.FIND_OVERLAPPING_NO_SUFFIX, 3: O.LEFTMOST_FIND}
S32 = 0x5A5A5A5A            # sentinel of int32 output words
S64 = 0x5A5A5A5A5A5A5A5A    # ... of int64 offsets / counts
POISON = ord("x")
DEFAULTS = {"kernel": 3, "hot_entries": 6144, "seg_len": 0, "gather_ordered": 1}
STD_MACHINES = ([{"kernel": k} for k in (0, 1, 2, 3, 4)] + [{"hot_entries": 0}, {"seg_len": 64}, {"seg_len": 256},
                {"gather_ordered": 0}, {"gather_ordered": 2}])
LANE_MACHINES = [{"kernel": 0}, {"kernel": 3}]


def _torch():
    import torch

    return torch


def _patterns(seed=3):
    """Patterns over "abc" plus ones that only poison ("x") can complete: x, xa, xab, abx, bx, xxx."""
    rng = np.random.default_rng(seed)
    pats = sorted({bytes(rng.integers(97, 100, size=int(rng.integers(1, 7))).tolist()) for _ in range(80)})
    return pats + [b"x", b"xa", b"xab", b"abx", b"bx", b"xxx"]


class Auto:
    """One automaton on the device and in the oracle, with the machines and iterators that serve it."""

    def __init__(self, cw, kind, pats):
        self.cw, self.kind = cw, kind
        p = [x.decode() for x in pats] if cw else pats
        cls = D.CharwiseDoubleArrayAhoCorasickBuilder if cw else D.DoubleArrayAhoCorasickBuilder
        self.pma = cls.new().match_kind(kind).build(p)
        self.opma = O.OraclePma.build(p, charwise=cw, match_kind=kind)
        self.modes = (3,) if kind else (0, 1, 2)
        self.machines = STD_MACHINES if (not cw and not kind) else LANE_MACHINES
        vals, lens, _ = self.pma.outputs()
        self.rec_of = {(int(v), int(n)): i for i, (v, n) in enumerate(zip(vals, lens))}
        self.n_out, self.n_val = len(vals), int(vals.max()) + 1

    def configure(self, opts):
        for k, v in DEFAULTS.items():
            self.pma.set_option(k, opts.get(k, v))

    def oracle(self, mode, text, offs):
        ref = self.opma.scan_batch(ORC[mode], np.ascontiguousarray(text), offs, want_matches=True)
        counts = ref["counts"].astype(np.int64)
        return ref["matches"], np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)


def automata():
    pats = _patterns()
    return [Auto(False, 0, pats), Auto(False, 1, pats), Auto(False, 2, pats), Auto(True, 0, pats), Auto(True, 1, pats),
            Auto(True, 2, pats)]


def _u32(t):
    return t.cpu().numpy().view(np.uint32).reshape(-1, 3)


def check_matches(a, mode, t, o, want, wo, tag):
    """Matches path on every machine of `a`, out / out_offs filled with sentinels and 64 / 16 entries of slack."""
    torch = _torch()
    n, total = len(wo) - 1, int(wo[-1])
    for opts in a.machines:
        if opts.get("seg_len") and mode not in (1, 2):
            continue
        a.configure(opts)
        out = torch.full((total + 64, 3), S32, dtype=torch.int32, device=t.device)
        oo = torch.full((n + 17,), S64, dtype=torch.int64, device=t.device)
        r = a.pma.scan_batch_device(mode, t, o, out=out, out_offs=oo)
        assert r.matches.shape[0] == total, (tag, mode, opts)
        assert _u32(out[:total]).tobytes() == want.view(np.uint32).tobytes(), (tag, mode, opts)
        assert bool((out[total:] == S32).all()), (tag, mode, opts, "d_out written past needed")
        assert np.array_equal(oo[: n + 1].cpu().numpy(), wo), (tag, mode, opts)
        assert bool((oo[n + 1:] == S64).all()), (tag, mode, opts, "out_offs written past n + 1")
    a.configure({})


def check_reductions(a, mode, t, o, want, wo, tag):
    """COUNT, FIRST and HIST (both keys) on the lane-per-haystack kernel and the lane machines; HIST is added into a
    longer, pre-filled histogram."""
    torch = _torch()
    n = len(wo) - 1
    counts = np.diff(wo)
    has = counts > 0
    vals = want["value"].astype(np.int64)
    by_val = np.bincount(vals, minlength=a.n_val)
    lens = (want["end"].astype(np.int64) - want["start"].astype(np.int64))
    by_rec = np.bincount(np.array([a.rec_of[(int(v), int(k))] for v, k in zip(vals, lens)], dtype=np.int64),
                         minlength=a.n_out)
    machines = [{"kernel": 0}, {"kernel": 3}] + ([{"hot_entries": 0}, {"seg_len": 64}] if not a.cw and not a.kind else [])
    for opts in machines:
        if opts.get("seg_len") and mode not in (1, 2):
            continue
        a.configure(opts)
        c = a.pma.count_batch_device(mode, t, o)
        assert np.array_equal(c.cpu().numpy(), counts), (tag, mode, opts)
        first, found = a.pma.first_batch_device(mode, t, o)
        assert np.array_equal(found.cpu().numpy(), has), (tag, mode, opts)
        if has.any():
            assert _u32(first)[has].tobytes() == want[wo[:-1][has]].view(np.uint32).tobytes(), (tag, mode, opts)
        for key, ref, k in (("value", by_val, a.n_val), ("output", by_rec, a.n_out)):
            pre = torch.arange(1, k + 9, dtype=torch.int64, device=t.device) * 1000
            h = a.pma.pattern_counts_device(mode, t, o, key=key, out=pre.clone())
            got = (h - pre).cpu().numpy()
            assert np.array_equal(got[:k], ref), (tag, mode, opts, key)
            assert not got[k:].any(), (tag, mode, opts, key, "hist written past the key range")
    a.configure({})
    assert n == len(counts)


def check_batch(autos, t, o, host_text, host_offs, tag):
    for a in autos:
        for mode in a.modes:
            want, wo = a.oracle(mode, host_text, host_offs)
            check_matches(a, mode, t, o, want, wo, tag)
            check_reductions(a, mode, t, o, want, wo, tag)


def check_stream(a, mode, buf, lo, mid, hi, tag):
    """One stream [lo, hi) of `buf` in two chunks split at `mid` (state and position carried), against the stepper
    over the whole stream."""
    torch = _torch()
    whole = buf[lo:hi].cpu().numpy()
    ref = a.opma.scan_batch(O.FIND_STEPPER if mode == 0 else O.FIND_OVERLAPPING_STEPPER, whole,
                            np.array([0, hi - lo], dtype=np.uint64), want_matches=True)["matches"]
    want = ref[ref["end"] != 0]
    state = torch.zeros(1, dtype=torch.int32, device=buf.device)
    got = []
    for a0, a1 in ((lo, mid), (mid, hi)):
        o = torch.tensor([0, a1 - a0], dtype=torch.int64, device=buf.device)
        pos = torch.tensor([a0 - lo], dtype=torch.int32, device=buf.device)
        r = a.pma.scan_stream_device(mode, buf[a0:a1], o, state, pos)
        got.append(_u32(r.matches))
    assert np.concatenate(got).tobytes() == want.view(np.uint32).tobytes(), (tag, mode, lo, mid, hi)


def _line_batches(rng):
    """(lo, offs) around the line at 0 (offsets relative to lo): haystacks that start 1-17, 255 and 4096 bytes below
    the line and end above it, one ending exactly at it, one starting there, long ones whose segments' warm-up
    crosses it."""
    out = []
    for d in list(range(1, 18)) + [255, 4096]:
        out.append((-d - 64, np.array([0, 64, 64 + d + int(rng.integers(1, 400)), 64 + d + 500], dtype=np.uint64)))
    out.append((-700, np.array([0, 300, 700, 1100, 1117], dtype=np.uint64)))
    out.append((-3000, np.array([0, 2990, 4490, 4497, 5190], dtype=np.uint64)))
    out.append((-9000, np.array([0, 8963, 14000], dtype=np.uint64)))
    return out


def test_a_haystacks_across_the_2_pow_32_address_line():
    torch = _torch()
    dev = torch.device("cuda", 0)
    big = torch.empty((4 << 30) + (8 << 20), dtype=torch.uint8, device=dev)
    try:
        ptr = big.data_ptr()
        line = ((ptr + (4 << 20)) >> 32 << 32) + (1 << 32)
        assert ptr + (4 << 20) < line <= ptr + (4 << 30) + (4 << 20)
        L = line - ptr
        rng = np.random.default_rng(11)
        window = rng.integers(97, 100, size=4 << 20).astype(np.uint8)
        big[L - (2 << 20): L + (2 << 20)] = torch.from_numpy(window).to(dev)
        host = window  # host[i] is the byte at line - 2 MiB + i
        autos = automata()
        for lo, offs in _line_batches(rng):
            a0 = L + lo
            t = big[a0: a0 + int(offs[-1])]
            o = torch.from_numpy(offs.astype(np.int64)).to(dev)
            h = host[(2 << 20) + lo: (2 << 20) + lo + int(offs[-1])]
            check_batch(autos, t, o, h, offs, ("line", lo))
        for a in autos:
            if a.kind:
                continue
            for mode in (0, 1):
                # chunks that end below the line with the state carried across it, and chunks that straddle it
                for lo, mid, hi in ((-300, -5, 200), (-4096, -17, 4096), (-1000, 0, 1000), (-64, 1, 64)):
                    check_stream(a, mode, big, L + lo, L + mid, L + hi, "line")
    finally:
        del big
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def _guard_batch():
    """Haystacks over "abc" that start and end with "ab" (poison before / after would complete "xab" / "abx"), an
    empty one, one ending in "x" before one starting with "ab", and one that is poison-free but short."""
    rng = np.random.default_rng(5)
    mid = lambda k: bytes(rng.integers(97, 100, size=k).tolist())  # noqa: E731
    hays = [b"ab" + mid(40) + b"ab", b"", b"ab", mid(17) + b"x", b"ab" + mid(100), b"b", mid(33) + b"ab"]
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    return b"".join(hays), offs


@pytest.mark.parametrize("head", [0, 5], ids=["offs0_zero", "offs0_five"])
def test_b_guarded_text_every_shift_and_tail(head):
    torch = _torch()
    dev = torch.device("cuda", 0)
    body, offs = _guard_batch()
    offs = offs + head  # [d_text, d_text + head) holds poison: offs[0] > 0
    nb = int(offs[-1])
    host = np.full(nb, POISON, dtype=np.uint8)
    host[head:] = np.frombuffer(body, dtype=np.uint8)
    o = torch.from_numpy(offs.astype(np.int64)).to(dev)
    autos = automata()
    want = {(id(a), m): a.oracle(m, host, offs) for a in autos for m in a.modes}
    arena = torch.empty(1 << 16, dtype=torch.uint8, device=dev)
    assert arena.data_ptr() % 256 == 0
    for shift in range(16):
        for slack in (0, 1, 7, 8, 15):
            arena.fill_(POISON)
            t = arena[256 + shift: 256 + shift + nb]
            t.copy_(torch.from_numpy(host).to(dev))
            assert bool((arena[256 + shift + nb: 256 + shift + nb + slack + 64] == POISON).all())
            for a in autos:
                for mode in a.modes:
                    w, wo = want[(id(a), mode)]
                    check_matches(a, mode, t, o, w, wo, ("guard", shift, slack))
                    if slack == 0:
                        check_reductions(a, mode, t, o, w, wo, ("guard", shift))
            if slack == 0:
                for a in autos:
                    if not a.kind:
                        for mode in (0, 1):  # the stream's chunk ends next to poison
                            check_stream(a, mode, arena, 256 + shift + head, 256 + shift + head + 45, 256 + shift + nb, "guard")


def _c3ish():
    pats = _patterns(9)
    rng = np.random.default_rng(17)
    lens = rng.integers(0, 600, size=300)
    offs = np.zeros(len(lens) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    text = rng.integers(97, 100, size=int(offs[-1])).astype(np.uint8)
    return pats, text, offs


def test_c_overflow_writes_nothing_past_cap_and_reports_exact_needed():
    torch = _torch()
    dev = torch.device("cuda", 0)
    pats, text, offs = _c3ish()
    t = torch.from_numpy(text).to(dev)
    o = torch.from_numpy(offs.astype(np.int64)).to(dev)
    L = _lib.load()
    n = len(offs) - 1
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    for a in (Auto(False, 0, pats), Auto(False, 1, pats), Auto(True, 0, pats)):
        for mode in a.modes:
            want, wo = a.oracle(mode, text, offs)
            total = int(wo[-1])
            for opts in a.machines:
                a.configure(opts)
                for cap in (0, 1, total - 1):
                    out = torch.full((total + 64, 3), S32, dtype=torch.int32, device=dev)
                    oo = torch.full((n + 17,), S64, dtype=torch.int64, device=dev)
                    need = C.c_uint64()
                    rc = L.dach_dev_scan_batch(a.pma.device_handle(0), mode, t.data_ptr(), o.data_ptr(), n, t.numel(),
                                               out.data_ptr(), cap, oo.data_ptr(), C.byref(need), st)
                    assert rc == _lib.OUTPUT_OVERFLOW and need.value == total, (mode, opts, cap, rc, need.value)
                    assert bool((out[cap:] == S32).all()), (mode, opts, cap, "d_out written past out_cap")
                    assert bool((oo[n + 1:] == S64).all()), (mode, opts, cap)
            a.configure({})


def test_c_count_first_views_inside_sentinel_buffers():
    torch = _torch()
    dev = torch.device("cuda", 0)
    pats, text, offs = _c3ish()
    t = torch.from_numpy(text).to(dev)
    o = torch.from_numpy(offs.astype(np.int64)).to(dev)
    L = _lib.load()
    n = len(offs) - 1
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    for a in (Auto(False, 0, pats), Auto(False, 1, pats), Auto(True, 0, pats), Auto(True, 2, pats)):
        for mode in a.modes:
            want, wo = a.oracle(mode, text, offs)
            counts = np.diff(wo)
            for opts in LANE_MACHINES:
                a.configure(opts)
                cb = torch.full((n + 9,), S64, dtype=torch.int64, device=dev)
                fb = torch.full((n + 9, 3), S32, dtype=torch.int32, device=dev)
                gb = torch.full((n + 9,), 0x5A, dtype=torch.uint8, device=dev)
                total, nf = C.c_uint64(), C.c_uint64()
                assert L.dach_dev_count_batch(a.pma.device_handle(0), mode, t.data_ptr(), o.data_ptr(), n, t.numel(),
                                              cb[4:].data_ptr(), C.byref(total), st) == 0
                assert L.dach_dev_first_batch(a.pma.device_handle(0), mode, t.data_ptr(), o.data_ptr(), n, t.numel(),
                                              fb[4:].data_ptr(), gb[4:].data_ptr(), C.byref(nf), st) == 0
                torch.cuda.synchronize()
                assert total.value == int(wo[-1]) and np.array_equal(cb[4: 4 + n].cpu().numpy(), counts), (mode, opts)
                assert nf.value == int((counts > 0).sum())
                for buf, s in ((cb, S64), (fb, S32), (gb, 0x5A)):
                    assert bool((buf[:4] == s).all()) and bool((buf[4 + n:] == s).all()), (mode, opts, "written beside the view")
            a.configure({})


def _job_cases():
    pats, text, offs = _c3ish()
    return [(Auto(False, 0, pats), m) for m in (0, 1, 2)] + [(Auto(False, 1, pats), 3), (Auto(False, 2, pats), 3)] + \
        [(Auto(True, 0, pats), m) for m in (0, 1, 2)] + [(Auto(True, 1, pats), 3), (Auto(True, 2, pats), 3)], text, offs


def test_d_jobs_of_every_iterator_on_two_streams_with_and_without_base():
    torch = _torch()
    dev = torch.device("cuda", 0)
    cases, text, offs = _job_cases()
    t = torch.from_numpy(text).to(dev)
    o = torch.from_numpy(offs.astype(np.int64)).to(dev)
    half = (len(offs) - 1) // 2
    parts = [(o[: half + 1], offs[: half + 1]), (o[half:], offs[half:])]
    streams = [torch.cuda.Stream(dev) for _ in range(3)]
    for a, mode in cases:
        wants = [a.oracle(mode, text, ho) for _, ho in parts]
        jobs = [a.pma.job(0), a.pma.job(0)]
        for base in (None, 5):
            outs, oofs = [], []
            for k in range(2):
                w, wo = wants[k]
                outs.append(torch.full((int(wo[-1]) + 5 + 40, 3), S32, dtype=torch.int32, device=dev))
                oofs.append(torch.full((len(wo) + 16,), S64, dtype=torch.int64, device=dev))
            torch.cuda.synchronize()
            for k in range(2):
                jobs[k].scan(mode, t, parts[k][0], outs[k].shape[0], stream=streams[k])
            b = None if base is None else torch.tensor([base], dtype=torch.int64, device=dev)
            jobs[0].place(outs[0], oofs[0], base=b, stream=streams[0])
            jobs[1].place(outs[1], oofs[1], base=b, stream=streams[2])
            for k in range(2):
                w, wo = wants[k]
                nk = len(wo) - 1
                b0 = base or 0
                assert jobs[k].wait() == int(wo[-1]), (a.cw, a.kind, mode, base)
                got = outs[k]
                assert _u32(got[b0: b0 + int(wo[-1])]).tobytes() == w.view(np.uint32).tobytes(), (a.cw, a.kind, mode, base)
                assert bool((got[:b0] == S32).all()) and bool((got[b0 + int(wo[-1]):] == S32).all()), (mode, base)
                assert np.array_equal(oofs[k][: nk + 1].cpu().numpy(), wo + b0)
                assert bool((oofs[k][nk + 1:] == S64).all())


def test_d_job_overflow_then_reuse():
    torch = _torch()
    dev = torch.device("cuda", 0)
    cases, text, offs = _job_cases()
    t = torch.from_numpy(text).to(dev)
    o = torch.from_numpy(offs.astype(np.int64)).to(dev)
    L = _lib.load()
    small = torch.from_numpy(offs[:11].astype(np.int64)).to(dev)
    for a, mode in cases:
        w, wo = a.oracle(mode, text, offs)
        total = int(wo[-1])
        job = a.pma.job(0)
        out = torch.full((total + 8, 3), S32, dtype=torch.int32, device=dev)
        oo = torch.zeros(len(offs), dtype=torch.int64, device=dev)
        cap = total // 3
        job.scan(mode, t, o, cap)
        job.place(out[:cap], oo)
        need = C.c_uint64()
        assert L.dach_job_wait(job._h, C.byref(need)) == _lib.OUTPUT_OVERFLOW and need.value == total, (a.cw, a.kind, mode)
        assert bool((out[cap:] == S32).all())
        with pytest.raises(D.DaachorseError) as e:  # the Python form raises the overflow
            job.scan(mode, t, o, cap)
            job.place(out[:cap], oo)
            job.wait()
        assert e.value.code == _lib.OUTPUT_OVERFLOW
        ws, wso = a.oracle(mode, text, offs[:11])
        job.scan(mode, t, small, total + 8)
        job.place(out, oo[:11])
        assert job.wait() == int(wso[-1])
        assert _u32(out[: int(wso[-1])]).tobytes() == ws.view(np.uint32).tobytes()
        assert np.array_equal(oo[:11].cpu().numpy(), wso)


def test_d_device_freed_before_its_job():
    """A garbage collector finalises a cycle in any order: an automaton's device image may be freed before a job of it.
    The job keeps scanning on the image, the last dach_job_free releases it, and nothing is left behind for later
    calls (a freed image read through the job once surfaced as "invalid device ordinal" in an unrelated launch)."""
    import gc

    torch = _torch()
    dev = torch.device("cuda", 0)
    pats, text, offs = _c3ish()
    t = torch.from_numpy(text).to(dev)
    o = torch.from_numpy(offs.astype(np.int64)).to(dev)
    n = len(offs) - 1
    L = _lib.load()
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    a = Auto(False, 0, pats)
    want, wo = a.oracle(1, text, offs)
    total = int(wo[-1])
    d, j = C.c_void_p(), C.c_void_p()
    assert L.dach_dev_upload(a.pma._h, 0, C.byref(d)) == 0
    assert L.dach_job_create(d, C.byref(j)) == 0
    L.dach_dev_free(d)  # the owner lets go first
    out = torch.full((total + 8, 3), S32, dtype=torch.int32, device=dev)
    oo = torch.empty(n + 1, dtype=torch.int64, device=dev)
    assert L.dach_job_scan(j, 1, t.data_ptr(), o.data_ptr(), n, t.numel(), total + 8, st) == 0
    assert L.dach_job_place(j, out.data_ptr(), total + 8, oo.data_ptr(), None, st) == 0
    need = C.c_uint64()
    assert L.dach_job_wait(j, C.byref(need)) == 0 and need.value == total
    assert _u32(out[:total]).tobytes() == want.view(np.uint32).tobytes()
    L.dach_job_free(j)  # releases the device image
    # the Python objects in one garbage cycle, listed in both orders
    for first_job in (False, True):
        b = Auto(False, 0, pats)
        job = b.pma.job(0)
        job.scan(1, t, o, total + 8)
        job.place(out, oo)
        assert job.wait() == total
        cyc = [job, b] if first_job else [b, job]
        cyc.append(cyc)
        del b, job, cyc
        gc.collect()
    torch.cuda.synchronize()
    for kernel in (0, 3):  # later scans of a fresh automaton run
        a.configure({"kernel": kernel})
        r = a.pma.scan_batch_host(1, text, offs)
        assert r.matches.tobytes() == want.tobytes()
    a.configure({})


# ---- E: needed past 2^32 matches ------------------------------------------------------------------------------------
# One haystack of N x "a", patterns "a" .. "a" x 64, find_overlapping: 64 N - 2016 matches.
ABOVE = 67108896  # 2^32 + 32
BELOW = ABOVE - 1  # 2^32 - 32


@pytest.mark.parametrize("n", [BELOW, ABOVE], ids=["below", "above"])
def test_e_needed_past_2_pow_32_matches(n):
    torch = _torch()
    dev = torch.device("cuda", 0)
    exact = 64 * n - 2016
    t = torch.full((n,), 97, dtype=torch.uint8, device=dev)
    o = torch.tensor([0, n], dtype=torch.int64, device=dev)
    L = _lib.load()
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    out = torch.full((1024 + 16, 3), S32, dtype=torch.int32, device=dev)
    oo = torch.empty(2, dtype=torch.int64, device=dev)
    want_rc = _lib.OUTPUT_OVERFLOW if exact <= 0xffffffff else _lib.INVALID_ARGUMENT
    pats = ["a" * k for k in range(1, 65)]
    bw = D.DoubleArrayAhoCorasick.new(pats)
    cw = D.CharwiseDoubleArrayAhoCorasick.new(pats)
    assert int(bw.count_batch_device(1, t, o)[0]) == exact
    if exact > 0xffffffff:  # one CwMachine lane over the whole haystack: once is enough
        assert int(cw.count_batch_device(1, t, o)[0]) == exact
    # The tuple-block paths (kernel 0, CwMachine) emit 2^32 matches one by one from a single lane, minutes of GPU time
    # per scan; their carry (Emitter::emit, the same source) is checked on the CPU emulation (test_emu_edges.py).
    runs = [(bw, {"kernel": 3, "seg_len": -1}, "k3_whole"), (bw, {}, "default_segmented")]
    for pma, opts, tag in runs:
        for k, v in opts.items():
            pma.set_option(k, v)
        need = C.c_uint64()
        rc = L.dach_dev_scan_batch(pma.device_handle(0), 1, t.data_ptr(), o.data_ptr(), 1, n, out.data_ptr(), 1024,
                                   oo.data_ptr(), C.byref(need), st)
        for k in opts:
            pma.set_option(k, DEFAULTS[k])
        # segmented, every item stays far below 2^32: an ordinary overflow with the exact total
        assert need.value == exact, (tag, need.value)
        assert rc == (_lib.OUTPUT_OVERFLOW if tag == "default_segmented" else want_rc), (tag, rc)
        assert bool((out[1024:] == S32).all()), tag
    # one stream chunk (never segmented)
    state = torch.zeros(1, dtype=torch.int32, device=dev)
    need = C.c_uint64()
    rc = L.dach_dev_scan_stream(bw.device_handle(0), 1, t.data_ptr(), o.data_ptr(), 1, n, state.data_ptr(), None,
                                out.data_ptr(), 1024, oo.data_ptr(), C.byref(need), st)
    assert need.value == exact and rc == want_rc, ("stream", rc, need.value)
    if exact > 0xffffffff:
        # the Python forms raise the refusal at once (no retry with a larger buffer)
        bw.set_option("seg_len", -1)
        with pytest.raises(D.DaachorseError) as e:
            bw.scan_batch_device(1, t, o)
        bw.set_option("seg_len", 0)
        assert e.value.code == _lib.INVALID_ARGUMENT and "2^32" in str(e.value)
        job = bw.job(0)
        bw.set_option("seg_len", -1)
        job.scan(1, t, o, 1024)
        job.place(out[:1024], oo)
        need = C.c_uint64()
        assert L.dach_job_wait(job._h, C.byref(need)) == _lib.INVALID_ARGUMENT and need.value == exact
        bw.set_option("seg_len", 0)
    del t
    torch.cuda.empty_cache()
