"""Counts, first matches, per-pattern histograms and masked text on jobs (dach_job_count / _first / _hist / _mask):
byte for byte what the synchronous calls report, on every mode and the kernels that serve them, across streams and
host threads, in stream order without a wait, alternating with the matches form on one job, with inputs dropped right
after they are enqueued, on bad offsets and host refusals, and with the handle freed before a reduction is enqueued
or while it is in flight.

Where a race must happen, ``torch.cuda._sleep`` holds a stream busy for about 50 ms (a bounded spin) while the host
queues the work that has to wait for it."""
import ctypes as C
import functools
import json
import os
import threading

import numpy as np
import pytest

import daachorse_b200 as D
from cases import seeded_reduce_case
from daachorse_b200 import _lib
from daachorse_b200 import synth as S
from daachorse_b200.automaton import HIST_KEYS, _check

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "search_tests.json"), encoding="utf-8"))
MODE = {"find_iter": D.FIND, "find_overlapping_iter": D.FIND_OVERLAPPING,
        "find_overlapping_no_suffix_iter": D.FIND_OVERLAPPING_NO_SUFFIX, "leftmost_find_iter": D.LEFTMOST_FIND}
KIND = {"Standard": 0, "LeftmostLongest": 1, "LeftmostFirst": 2}
STD_MODES = (D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX)
SLEEP_CYCLES = 80_000_000  # ~40-55 ms at H100 clocks
FILL = 0x2A
THREAD_TIMEOUT_S = 120


def builder(cw):
    return D.CharwiseDoubleArrayAhoCorasickBuilder if cw else D.DoubleArrayAhoCorasickBuilder


def modes(kind):
    return (D.LEFTMOST_FIND,) if kind else STD_MODES


def on_device(text, offs):
    import torch

    t = torch.from_numpy(np.array(text, dtype=np.uint8)).cuda() if len(text) else torch.zeros(0, dtype=torch.uint8, device="cuda")
    return t, torch.from_numpy(offs.astype(np.int64)).cuda()


def _p(t):
    return C.c_void_p(t.data_ptr())


def _stream():
    import torch

    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def sync_results(pma, mode, t, o):
    """What the synchronous calls report, each with its *total: {name: (tensors, total)}."""
    import torch

    L = _lib.load()
    d = pma.device_handle(0)
    n = o.numel() - 1
    tot = C.c_uint64()
    res = {}
    counts = torch.empty(n, dtype=torch.int64, device="cuda")
    _check(L.dach_dev_count_batch(d, mode, _p(t), _p(o), n, t.numel(), _p(counts), C.byref(tot), _stream()))
    res["count"] = ((counts,), tot.value)
    first = torch.empty((n, 3), dtype=torch.int32, device="cuda")
    found = torch.empty(n, dtype=torch.bool, device="cuda")
    _check(L.dach_dev_first_batch(d, mode, _p(t), _p(o), n, t.numel(), _p(first), _p(found), C.byref(tot), _stream()))
    res["first"] = ((first, found), tot.value)
    for key in HIST_KEYS:
        h = torch.zeros(pma._hist_len(key), dtype=torch.int64, device="cuda")
        _check(L.dach_dev_hist_batch(d, mode, HIST_KEYS[key], _p(t), _p(o), n, t.numel(), _p(h), h.numel(), C.byref(tot), _stream()))
        res["hist-" + key] = ((h,), tot.value)
    res["mask"] = ((pma.mask_batch_device(mode, t, o, fill=FILL),), 0)
    return res


def job_results(job, mode, t, o, stream=None):
    """The same on a job, each result waited for: {name: (tensors, wait())}."""
    res = {"count": ((job.count(mode, t, o, stream=stream),), job.wait())}
    res["first"] = (job.first(mode, t, o, stream=stream), job.wait())
    for key in HIST_KEYS:
        res["hist-" + key] = ((job.pattern_counts(mode, t, o, key=key, stream=stream),), job.wait())
    res["mask"] = ((job.mask(mode, t, o, fill=FILL, stream=stream),), job.wait())
    return res


def assert_same(got, want, tag):
    import torch

    assert got.keys() == want.keys()
    for name in want:
        (gt, gtot), (wt, wtot) = got[name], want[name]
        assert gtot == wtot, (tag, name, gtot, wtot)
        for a, b in zip(gt, wt):
            assert a.dtype == b.dtype and torch.equal(a, b), (tag, name)


def check_parity(pma, job, mode, t, o, tag, stream=None):
    want = sync_results(pma, mode, t, o)
    assert_same(job_results(job, mode, t, o, stream=stream), want, tag)
    return want


# ---- parity with the synchronous calls ---------------------------------------------------------------------------

@pytest.mark.parametrize("variant,iterator,coll,kind", [tuple(c) for c in GOLD["configs"] if c[1] in MODE])
def test_golden_vectors(variant, iterator, coll, kind):
    cw = variant == "charwise"
    for g in GOLD["collections"][coll]:
        for case in GOLD["groups"][g]:
            pma = builder(cw).new().match_kind(KIND[kind]).build(case["patterns"])
            job = pma.job(0)
            hay = case["haystack"].encode()
            t, o = on_device(np.frombuffer(hay, dtype=np.uint8), np.array([0, len(hay)], dtype=np.uint64))
            check_parity(pma, job, MODE[iterator], t, o, case["name"])


@pytest.mark.parametrize("cw", [False, True])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_seeded_batches_kernels_and_segments(cw, kind):
    """Every mode, bytewise and charwise; kernel 3 (the lane machines) and 0 (lane per haystack), and forced segments."""
    pats, text, offs = seeded_reduce_case(cw, kind)
    pma = builder(cw).new().match_kind(kind).build(pats)
    job = pma.job(0)
    t, o = on_device(text, offs)
    try:
        for mode in modes(kind):
            for opts in ({"kernel": 3}, {"kernel": 0}, {"kernel": 3, "seg_len": 256}, {"kernel": 3, "seg_len": 64}):
                for k, v in opts.items():
                    pma.set_option(k, v)
                check_parity(pma, job, mode, t, o, (cw, kind, mode, opts))
                pma.set_option("seg_len", 0)
    finally:
        pma.set_option("kernel", 3)
        pma.set_option("seg_len", 0)


@functools.lru_cache(maxsize=None)
def c2_case(n=4096, hay_len=4096, seed=7):
    """A seeded C2 batch (16 MiB of text): the C2 automaton and device tensors."""
    cfg = S.config("C2")
    ps = S.make_patterns(cfg, n=4000)
    pool, b = S.make_pool(cfg, ps, 8 << 20)
    starts = S.window_starts(b, len(pool), n, hay_len, seed=seed)
    text, offs = S.materialise_host(pool, starts, hay_len)
    return D.DoubleArrayAhoCorasick.new(ps.as_list()), text, offs


def test_c2_batch_every_mode():
    pma, text, offs = c2_case()
    t, o = on_device(text, offs)
    job = pma.job(0)
    for mode in STD_MODES:
        want = check_parity(pma, job, mode, t, o, mode)
        assert want["count"][1] > 0


# ---- concurrency ------------------------------------------------------------------------------------------------

def _run_threads(n, target):
    barrier = threading.Barrier(n)
    errors = []

    def body(i):
        try:
            barrier.wait(timeout=60)
            target(i)
        except BaseException as e:  # a failure in a thread fails the test
            errors.append((i, repr(e)))

    threads = [threading.Thread(target=body, args=(i,), daemon=True) for i in range(n)]
    for th in threads:
        th.start()
    for th in threads:
        th.join(timeout=THREAD_TIMEOUT_S)
    assert not any(th.is_alive() for th in threads), "threads did not finish in %d s" % THREAD_TIMEOUT_S
    assert not errors, errors


def test_two_threads_two_jobs_each():
    """Two host threads, each with two jobs on streams of their own, run COUNT and HIST on one automaton at once (step
    s+1 enqueued before step s is waited for); every result equals the synchronous call's."""
    import torch

    pma, text, offs = c2_case()
    mode = D.FIND_OVERLAPPING
    batches = []
    for k in range(4):  # four slices of the C2 batch, of different sizes
        lo, hi = k * 512, k * 512 + 256 * (k + 1)
        o = offs[lo:hi + 1] - offs[lo]
        batches.append(on_device(text[int(offs[lo]):int(offs[hi])], o))
    refs = [sync_results(pma, mode, t, o) for t, o in batches]
    torch.cuda.synchronize()

    def worker(i):
        jobs = [pma.job(0) for _ in range(2)]
        sts = [torch.cuda.Stream() for _ in range(2)]
        for r in range(6):
            pending = []
            for k, (job, st) in enumerate(zip(jobs, sts)):
                b = (i + r + k) % len(batches)
                t, o = batches[b]
                if (r + k) % 2:
                    pending.append((job, b, "count", (job.count(mode, t, o, stream=st),)))
                else:
                    pending.append((job, b, "hist-value", (job.pattern_counts(mode, t, o, stream=st),)))
            for job, b, name, got in pending:
                total = job.wait()
                want, wtot = refs[b][name]
                assert total == wtot, (i, r, name)
                assert all(torch.equal(g, w) for g, w in zip(got, want)), (i, r, name)

    _run_threads(2, worker)


def test_four_jobs_add_into_one_histogram():
    """Four jobs on four streams add into one histogram at the same time; it ends as the sum of their batches'."""
    import torch

    pma, text, offs = c2_case()
    mode = D.FIND_OVERLAPPING
    batches, want, want_total = [], 0, 0
    for k in range(4):
        lo, hi = k * 1024, (k + 1) * 1024
        t, o = on_device(text[int(offs[lo]):int(offs[hi])], offs[lo:hi + 1] - offs[lo])
        (h,), tot = sync_results(pma, mode, t, o)["hist-value"]
        batches.append((t, o))
        want, want_total = want + h, want_total + tot
    for key in HIST_KEYS:
        jobs = [pma.job(0) for _ in range(4)]
        sts = [torch.cuda.Stream() for _ in range(4)]
        shared = torch.zeros(pma._hist_len(key), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        for job, st, (t, o) in zip(jobs, sts, batches):
            job.pattern_counts(mode, t, o, key=key, out=shared, stream=st)
        assert sum(job.wait() for job in jobs) == want_total
        if key == "value":
            assert torch.equal(shared, want)
        else:
            vals = torch.from_numpy(pma.outputs()[0].astype(np.int64)).cuda()
            assert torch.equal(torch.zeros_like(want).index_add_(0, vals, shared), want)


def test_stream_order_without_a_wait():
    """COUNT and MASK consumed by torch ops on the job's stream before wait(): the stream is held by a spin, so the
    ops are queued while the job's work is still pending, and they see its results."""
    import torch

    pma, text, offs = c2_case()
    mode = D.FIND
    t, o = on_device(text, offs)
    want = sync_results(pma, mode, t, o)
    job = pma.job(0)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        torch.cuda._sleep(SLEEP_CYCLES)
        counts = job.count(mode, t, o, stream=st)
        total = counts.sum()
        doubled = counts * 2
    n = job.wait()
    with torch.cuda.stream(st):
        torch.cuda._sleep(SLEEP_CYCLES)
        masked = job.mask(mode, t, o, fill=FILL, stream=st)
        hits = (masked == FILL).sum()
        same = (masked == want["mask"][0][0]).all()
    st.synchronize()
    assert int(total) == n == want["count"][1]
    assert torch.equal(doubled, want["count"][0][0] * 2)
    assert bool(same) and int(hits) == int((want["mask"][0][0] == FILL).sum())
    assert job.wait() == 0


# ---- one job, every kind in turn -----------------------------------------------------------------------------------

def test_one_job_alternates_scans_and_reductions():
    """scan / place / wait -> mask -> count over the masked text -> hist -> scan / place / wait on one job; each step
    equals its synchronous form.  A reduction while a scan waits for its placement, and a placement after a
    reduction, are refused and leave the job usable; the handle's timings are the synchronous calls' alone."""
    import torch

    pma, text, offs = c2_case()
    mode = D.FIND_OVERLAPPING
    t, o = on_device(text, offs)
    job = pma.job(0)
    ref = pma.scan_batch_device(mode, t, o)
    k = ref.matches.shape[0]

    def scan_place_wait():
        out = torch.zeros((k + 16, 3), dtype=torch.int32, device="cuda")
        oo = torch.zeros(o.numel(), dtype=torch.int64, device="cuda")
        job.scan(mode, t, o, k + 16)
        with pytest.raises(D.DaachorseError) as e:
            job.count(mode, t, o)  # the scan is not placed yet
        assert e.value.code == _lib.INVALID_ARGUMENT
        with pytest.raises(D.DaachorseError) as e:
            job.wait()  # nor a wait: the last placement's report would be stale
        assert e.value.code == _lib.INVALID_ARGUMENT
        job.place(out, oo)
        assert job.wait() == k
        assert torch.equal(out[:k], ref.matches) and torch.equal(oo, ref.offsets)

    scan_place_wait()
    masked = job.mask(mode, t, o, fill=FILL)
    assert job.wait() == 0
    assert torch.equal(masked, pma.mask_batch_device(mode, t, o, fill=FILL))
    with pytest.raises(D.DaachorseError) as e:  # nothing to place after a reduction
        job.place(torch.zeros((k + 16, 3), dtype=torch.int32, device="cuda"), torch.zeros(o.numel(), dtype=torch.int64, device="cuda"))
    assert e.value.code == _lib.INVALID_ARGUMENT
    counts = job.count(mode, masked, o)
    total = job.wait()
    want = sync_results(pma, mode, masked, o)["count"]
    assert total == want[1] and torch.equal(counts, want[0][0])
    stats = pma.stats()  # the last synchronous call's figures
    hist = job.pattern_counts(mode, t, o)
    htotal = job.wait()
    assert job.scan_kernel_ms() > 0
    times = job.times()
    assert 0 <= times[0] <= times[1] and times[2:] == (0.0, 0.0)
    assert pma.stats()["scan_kernel_ms"] == stats["scan_kernel_ms"] and pma.stats()["total_ms"] == stats["total_ms"]
    (want_h,), want_htotal = sync_results(pma, mode, t, o)["hist-value"]
    assert htotal == want_htotal and torch.equal(hist, want_h)
    scan_place_wait()


# ---- lifetimes ----------------------------------------------------------------------------------------------------

def test_tensors_live_in_stream_order():
    """Inputs copied just before the calls and dropped right after them, while the job's stream is held; blocks of
    their size are allocated and filled with junk on the current stream.  Caller-given outputs are freed after
    wait().  Every result equals the synchronous call's."""
    import torch

    pma, text, offs = c2_case()
    mode = D.FIND_OVERLAPPING
    t0, o0 = on_device(text, offs)
    want = sync_results(pma, mode, t0, o0)
    job = pma.job(0)
    st = torch.cuda.Stream()
    n = o0.numel() - 1

    def run(raced):
        got = {}
        for name in ("count", "first", "hist-value", "mask"):
            torch.cuda.synchronize()
            if raced:
                with torch.cuda.stream(st):
                    torch.cuda._sleep(SLEEP_CYCLES)  # the job's calls below are queued behind the spin
            t, o = t0.clone(), o0.clone()
            if name == "count":
                outs = (torch.full((n,), -1, dtype=torch.int64, device="cuda"),)
            elif name == "first":
                outs = (torch.zeros((n, 3), dtype=torch.int32, device="cuda"), torch.zeros(n, dtype=torch.bool, device="cuda"))
            st.wait_stream(torch.cuda.current_stream())  # the inputs and outputs were written here: the caller orders them
            if name == "count":
                job.count(mode, t, o, out=outs[0], stream=st)
            elif name == "first":
                job.first(mode, t, o, out=outs[0], found=outs[1], stream=st)
            elif name == "hist-value":
                outs = (job.pattern_counts(mode, t, o, stream=st),)
            else:
                outs = (job.mask(mode, t, o, fill=FILL, stream=st),)
            size = t.numel()
            del t, o  # dropped right after the enqueue
            junk = [torch.empty(size, dtype=torch.uint8, device="cuda") for _ in range(8)]
            for x in junk:
                x.fill_(0x23)
            del junk, x
            total = job.wait()
            got[name] = (tuple(x.clone() for x in outs), total)
            del outs  # freed after wait()
        return got

    run(False)  # sizes the workspaces and caches the junk blocks
    assert_same(run(True), {k: want[k] for k in ("count", "first", "hist-value", "mask")}, "raced")


# ---- errors -------------------------------------------------------------------------------------------------------

def test_bad_offsets_leave_the_outputs_alone():
    import torch

    pma, text, offs = c2_case()
    mode = D.FIND_OVERLAPPING
    t, o = on_device(text[: 4096 * 4], offs[:5])
    bad = torch.tensor([0, 9000, 4000, 16384], dtype=torch.int64, device="cuda")
    n = bad.numel() - 1
    job = pma.job(0)
    outs = {
        "count": lambda: (torch.full((n,), 0x5A5A, dtype=torch.int64, device="cuda"),),
        "first": lambda: (torch.full((n, 3), 0x5A5A, dtype=torch.int32, device="cuda"), torch.ones(n, dtype=torch.bool, device="cuda")),
        "hist": lambda: (torch.full((pma._hist_len("value"),), 7, dtype=torch.int64, device="cuda"),),
        "mask": lambda: (torch.full((t.numel(),), 0x5A, dtype=torch.uint8, device="cuda"),),
    }
    call = {
        "count": lambda b: job.count(mode, t, bad, out=b[0]),
        "first": lambda b: job.first(mode, t, bad, out=b[0], found=b[1]),
        "hist": lambda b: job.pattern_counts(mode, t, bad, out=b[0]),
        "mask": lambda b: job.mask(mode, t, bad, out=b[0]),
    }
    for name in outs:
        bufs = outs[name]()
        before = tuple(b.clone() for b in bufs)
        call[name](bufs)
        with pytest.raises(D.DaachorseError) as e:
            job.wait()
        assert e.value.code == _lib.INVALID_ARGUMENT and "ascending" in str(e.value), name
        assert all(torch.equal(a, b) for a, b in zip(bufs, before)), name
    assert_same(job_results(job, mode, t, o), sync_results(pma, mode, t, o), "after bad offsets")


def test_host_refusals_enqueue_nothing():
    """Null arguments, the match kind, the histogram's key and size, an overlapping or non-ASCII charwise mask, too many
    haystacks: each refused with its status and no launch, and the job works afterwards."""
    import torch

    L = _lib.load()
    pats, text, offs = seeded_reduce_case(False, 0)
    pma = D.DoubleArrayAhoCorasick.new(pats)
    cw = D.CharwiseDoubleArrayAhoCorasick.new([p.decode() for p in pats])
    t, o = on_device(text, offs)
    n = o.numel() - 1
    counts = torch.zeros(n, dtype=torch.int64, device="cuda")
    first = torch.zeros((n, 3), dtype=torch.int32, device="cuda")
    found = torch.zeros(n, dtype=torch.bool, device="cuda")
    hist = torch.zeros(max(pma._hist_len("output"), cw._hist_len("output")), dtype=torch.int64, device="cuda")
    masked = torch.zeros(t.numel(), dtype=torch.uint8, device="cuda")
    for p in (pma, cw):
        job = p.job(0)
        d = p.device_handle(0)
        nh = p._hist_len("output")
        h, s, tb = job._h, _stream(), t.numel()
        cases = [
            (lambda: L.dach_job_count(h, 0, _p(t), None, n, tb, _p(counts), s), _lib.INVALID_ARGUMENT),
            (lambda: L.dach_job_count(h, 0, _p(t), _p(o), n, tb, None, s), _lib.INVALID_ARGUMENT),
            (lambda: L.dach_job_first(h, 0, _p(t), _p(o), n, tb, _p(first), None, s), _lib.INVALID_ARGUMENT),
            (lambda: L.dach_job_hist(h, 0, 0, _p(t), _p(o), n, tb, None, nh, s), _lib.INVALID_ARGUMENT),
            (lambda: L.dach_job_mask(h, 0, None, _p(o), n, tb, FILL, _p(masked), s), _lib.INVALID_ARGUMENT),
            (lambda: L.dach_job_count(h, D.LEFTMOST_FIND, _p(t), _p(o), n, tb, _p(counts), s), _lib.MATCH_KIND_MISMATCH),
            (lambda: L.dach_job_first(h, 4, _p(t), _p(o), n, tb, _p(first), _p(found), s), _lib.INVALID_ARGUMENT),
            (lambda: L.dach_job_hist(h, 0, 0, _p(t), _p(o), n, tb, _p(hist), nh - 1, s), _lib.INVALID_ARGUMENT),
            (lambda: L.dach_job_hist(h, 0, 2, _p(t), _p(o), n, tb, _p(hist), nh, s), _lib.INVALID_ARGUMENT),
            (lambda: L.dach_job_mask(h, 0, _p(t), _p(o), n, tb, FILL, C.c_void_p(t.data_ptr() + 1), s), _lib.INVALID_ARGUMENT),
            (lambda: L.dach_job_count(h, 0, _p(t), _p(o), 0xFFFFFFF1, tb, _p(counts), s), _lib.INVALID_ARGUMENT),
        ]
        if p is cw:
            cases.append((lambda: L.dach_job_mask(h, 0, _p(t), _p(o), n, tb, 0x80, _p(masked), s), _lib.INVALID_ARGUMENT))
        torch.cuda.synchronize()
        launches = L.dach_dev_kernel_launches(d)
        for i, (call, want) in enumerate(cases):
            rc = call()
            assert rc == want, (i, rc, _lib.last_error())
        assert L.dach_dev_kernel_launches(d) == launches
        assert_same(job_results(job, D.FIND_OVERLAPPING, t, o), sync_results(p, D.FIND_OVERLAPPING, t, o), "after refusals")


@pytest.mark.parametrize("free_first", [True, False], ids=["freed-before-enqueue", "freed-in-flight"])
def test_handle_freed_before_its_job(free_first):
    """dach_dev_free before dach_job_free: HIST (the reduction that reads the most image tables and allocates the
    job's tables on first use) and COUNT are queued behind a spin on the job's stream, with the handle freed before
    they are enqueued or while they are still pending.  The job keeps the image alive: both equal the synchronous calls
    of an independently uploaded handle, the last dach_job_free releases the image, and a fresh automaton works
    afterwards."""
    import torch

    L = _lib.load()
    pats, text, offs = seeded_reduce_case(False, 0)
    pma = D.DoubleArrayAhoCorasick.new(pats)
    t, o = on_device(text, offs)
    n = o.numel() - 1
    want = sync_results(pma, D.FIND_OVERLAPPING, t, o)  # pma's own handle, not the one freed below
    (want_h,), want_htotal = want["hist-value"]
    (want_c,), want_ctotal = want["count"]
    d, j = C.c_void_p(), C.c_void_p()
    _check(L.dach_dev_upload(pma._h, 0, C.byref(d)))
    _check(L.dach_job_create(d, C.byref(j)))
    hist = torch.zeros(want_h.numel(), dtype=torch.int64, device="cuda")
    counts = torch.full((n,), -1, dtype=torch.int64, device="cuda")
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    if free_first:
        L.dach_dev_free(d)
    with torch.cuda.stream(st):
        torch.cuda._sleep(SLEEP_CYCLES)
    s = C.c_void_p(st.cuda_stream)
    total = C.c_uint64()
    _check(L.dach_job_hist(j, D.FIND_OVERLAPPING, HIST_KEYS["value"], _p(t), _p(o), n, t.numel(), _p(hist), hist.numel(), s))
    if not free_first:
        L.dach_dev_free(d)  # the histogram is still queued behind the spin
    _check(L.dach_job_wait(j, C.byref(total)))
    assert total.value == want_htotal and torch.equal(hist, want_h)
    with torch.cuda.stream(st):
        torch.cuda._sleep(SLEEP_CYCLES)
    _check(L.dach_job_count(j, D.FIND_OVERLAPPING, _p(t), _p(o), n, t.numel(), _p(counts), s))
    _check(L.dach_job_wait(j, C.byref(total)))
    assert total.value == want_ctotal and torch.equal(counts, want_c)
    L.dach_job_free(j)  # the last reference: the image goes now
    torch.cuda.synchronize()
    fresh = D.DoubleArrayAhoCorasick.new([b"ab", b"b"])
    job = fresh.job(0)
    ft, fo = on_device(np.frombuffer(b"abab", dtype=np.uint8), np.array([0, 2, 4], dtype=np.uint64))
    assert job.count(D.FIND_OVERLAPPING, ft, fo).tolist() == [2, 2] and job.wait() == 4
