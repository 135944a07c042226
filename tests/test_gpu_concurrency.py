"""Scans across streams and host threads, against the oracle: the device forms on a stream other than the current one
(outputs the wrapper allocates, inputs written just before the call, the overflow retry of stream chunks), tensors
handed to jobs and dropped before the job has read them, jobs and synchronous calls of one automaton in eight host
threads at once, and pipelined jobs whose batch sizes change from step to step.

The races are made to happen on every run: ``torch.cuda._sleep`` holds a stream busy for about 50 ms (a bounded spin)
while the host queues the work that must wait for it.  Junk only ever goes into text bytes, which the scan reads in
bounds; offsets and buffers the library writes only ever hold real values."""
import functools
import threading

import numpy as np
import pytest

import daachorse_b200 as D
import emu_mask_api as M
import oracle_api as O
from daachorse_b200 import _lib
from daachorse_b200 import automaton as A
from daachorse_b200 import synth as S

pytestmark = pytest.mark.gpu

SLEEP_CYCLES = 80_000_000  # ~40-55 ms at H100 clocks
JUNK = 0x23  # '#': ASCII (valid UTF-8) and in no pattern here
STEPPER = {D.FIND: O.FIND_STEPPER, D.FIND_OVERLAPPING: O.FIND_OVERLAPPING_STEPPER}
THREAD_TIMEOUT_S = 120


# ---- automata and batches ----------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def _source(cw):
    cfg = S.config("C4" if cw else "C2")
    ps = S.make_patterns(cfg, n=5000 if cw else 4000)
    pool, b = S.make_pool(cfg, ps, 4 << 20)
    return ps, pool, b


@functools.lru_cache(maxsize=None)
def automaton(kind):
    """kind: "bw" (bytewise Standard), "bw-ll" (LeftmostLongest), "bw-lf" (LeftmostFirst), "cw" (charwise Standard);
    returns (pma, oracle)."""
    cw = kind == "cw"
    ps = _source(cw)[0]
    mk = {"bw": 0, "bw-ll": 1, "bw-lf": 2, "cw": 0}[kind]
    builder = D.CharwiseDoubleArrayAhoCorasickBuilder if cw else D.DoubleArrayAhoCorasickBuilder
    pats = [p.decode() for p in ps.as_list()] if cw else ps.as_list()
    pma = builder.new().match_kind(D.MatchKind(mk)).build(pats)
    return pma, O.OraclePma.build_packed(ps.blob, ps.offs, charwise=cw, match_kind=mk)


@functools.lru_cache(maxsize=None)
def batch(cw, n, hay_len, seed):
    """n windows of hay_len bytes of the pool (charwise: cut at a char boundary), host text + uint64 offsets."""
    _, pool, b = _source(cw)
    if len(pool) < hay_len + 1:
        raise ValueError("hay_len above the pool")
    starts = S.window_starts(b, len(pool), n, hay_len, seed=seed)
    text, offs = S.materialise_host(pool, starts, hay_len)
    if cw:
        text = S.pad_to_char_boundary(text.reshape(n, hay_len)).reshape(-1)
    return text, offs


def on_device(text, offs):
    import torch

    return torch.from_numpy(np.ascontiguousarray(text)).cuda(), torch.from_numpy(offs.astype(np.int64)).cuda()


def _u32(t):
    return t.cpu().numpy().view(np.uint32)


def expected(opma, omode, text, offs, n_values):
    """Everything the forms report, from the oracle's match list: matches (k, 3) u32, offsets, counts, first / found,
    histogram and document frequencies by value, and (unless omode is a stepper) the masked text."""
    r = opma.scan_batch(omode, text, offs, nthreads=16, want_matches=True)
    m = r["matches"]
    mm = np.stack([m["start"], m["end"], m["value"]], axis=1).astype(np.uint32) if len(m) else np.zeros((0, 3), np.uint32)
    counts = r["counts"].astype(np.int64)
    n = len(counts)
    oo = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    has = counts > 0
    first = np.full((n, 3), 0xFFFFFFFF, dtype=np.uint32)
    first[has] = mm[oo[:-1][has]]
    hay = np.repeat(np.arange(n, dtype=np.int64), counts)
    pairs = np.unique(hay * n_values + mm[:, 2].astype(np.int64))
    want = dict(m=mm, offs=oo, counts=counts, first=first, found=has,
                hist=np.bincount(mm[:, 2].astype(np.int64), minlength=n_values),
                df=np.bincount(pairs % n_values, minlength=n_values))
    if omode < O.FIND_STEPPER:
        want["mask"] = M.expected_from_matches(text, offs, m, r["counts"], 0x2A)
    return want


def check_hist(pma, got, want, key, tag):
    """key "value": bin = value; key "output": bin = output record, summed over the records of each value."""
    got = got.cpu().numpy()
    if key == "value":
        assert np.array_equal(got, want), tag
    else:
        vals = pma.outputs()[0].astype(np.int64)
        assert np.array_equal(np.bincount(vals, weights=got.astype(np.float64), minlength=len(want)), want), tag


def check_df(pma, got, want, key, tag):
    got = got.cpu().numpy()
    if key == "value":
        assert np.array_equal(got, want), tag
    else:
        vals = pma.outputs()[0].astype(np.int64)
        assert len(np.unique(vals)) == len(vals)  # one record per value: DF by record = DF of its value
        assert np.array_equal(got, want[vals]), tag


def n_values(pma):
    return int(pma.outputs()[0].max()) + 1


def hold(stream=None):
    """Queue a bounded ~50 ms spin on ``stream`` (default: the current stream)."""
    import torch

    if stream is None:
        torch.cuda._sleep(SLEEP_CYCLES)
    else:
        with torch.cuda.stream(stream):
            torch.cuda._sleep(SLEEP_CYCLES)


# ---- 1. device forms on a second stream ------------------------------------------------------------------------

FORM_CASES = [("bw", D.FIND), ("bw", D.FIND_OVERLAPPING), ("bw", D.FIND_OVERLAPPING_NO_SUFFIX), ("bw-ll", D.LEFTMOST_FIND),
              ("cw", D.FIND_OVERLAPPING)]


def _stream_case(kind, mode):
    return kind in ("bw", "cw") and mode in STEPPER


class _Forms:
    """One batch, its expected results and a second stream S; every form has run once on the current stream, so the
    handle's workspaces have their size and no raced call frees one (a free would wait for the whole device)."""

    def __init__(self, kind, mode, as_int):
        import torch

        cw = kind == "cw"
        pma, opma = automaton(kind)
        nv = n_values(pma)
        text, offs = batch(cw, 1024, 4000, seed=11)
        t, o = on_device(text, offs)
        n = len(offs) - 1
        want = expected(opma, mode, text, offs, nv)
        stream_case = _stream_case(kind, mode)
        want_st = expected(opma, STEPPER[mode], text, offs, nv) if stream_case else None
        S_ = torch.cuda.Stream()
        sarg = S_.cuda_stream if as_int else S_

        def zeros_state():
            return torch.zeros(n, dtype=torch.int32, device="cuda")

        # every form once on the current stream: the handle's workspaces take their size (no free inside a raced call)
        pma.scan_batch_device(mode, t, o)
        pma.count_batch_device(mode, t, o)
        pma.first_batch_device(mode, t, o)
        pma.mask_batch_device(mode, t, o)
        for key in ("value", "output"):
            pma.pattern_counts_device(mode, t, o, key=key)
            pma.doc_counts_device(mode, t, o, key=key)
        ref_state = None
        if stream_case:
            ref_state = zeros_state()
            pma.scan_stream_device(mode, t, o, ref_state)
            pma.count_stream_device(mode, t, o, zeros_state())
            pma.first_stream_device(mode, t, o, zeros_state())
            pma.pattern_counts_stream_device(mode, t, o, zeros_state())
        torch.cuda.synchronize()
        self.__dict__.update(S=S_, cw=cw, pma=pma, t=t, o=o, n=n, want=want, want_st=want_st, sarg=sarg, stream_case=stream_case,
                             ref_state=ref_state, zeros_state=zeros_state)


FORMS = pytest.mark.parametrize("kind,mode", FORM_CASES)
AS_INT = pytest.mark.parametrize("as_int", [True, False], ids=["raw-handle", "stream-object"])


@AS_INT
@FORMS
def test_zeroed_outputs_on_a_second_stream(kind, mode, as_int):
    """a. The histograms and document frequencies the wrapper zero-fills on the current stream, held busy, while the
    call adds into them on S."""
    import torch

    F = _Forms(kind, mode, as_int)
    pma, t, o, want, want_st, sarg, ref_state = F.pma, F.t, F.o, F.want, F.want_st, F.sarg, F.ref_state
    stream_case, zeros_state = F.stream_case, F.zeros_state

    # a. zero-filled outputs: torch.zeros is queued behind the spin on the current stream
    for key in ("value", "output"):
        for name, call, check, w in (("pattern_counts_device", pma.pattern_counts_device, check_hist, want["hist"]),
                                     ("doc_counts_device", pma.doc_counts_device, check_df, want["df"])):
            hold()
            got = call(mode, t, o, key=key, stream=sarg)
            torch.cuda.synchronize()
            check(pma, got, w, key, (name, key))
        if stream_case:
            st = zeros_state()
            torch.cuda.synchronize()
            hold()
            got = pma.pattern_counts_stream_device(mode, t, o, st, key=key, stream=sarg)
            torch.cuda.synchronize()
            check_hist(pma, got, want_st["hist"], key, ("pattern_counts_stream_device", key))
            assert torch.equal(st, ref_state)


@AS_INT
@FORMS
def test_reused_blocks_on_a_second_stream(kind, mode, as_int):
    """b. Blocks shaped like the outputs the wrapper allocates are filled with junk behind the spin on the current
    stream and freed at once, so the caching allocator hands them to the wrapper while the fill is still pending."""
    import torch

    F = _Forms(kind, mode, as_int)
    pma, t, o, n, want, want_st, sarg, ref_state = F.pma, F.t, F.o, F.n, F.want, F.want_st, F.sarg, F.ref_state
    stream_case, zeros_state = F.stream_case, F.zeros_state

    def reused(specs, call):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        junk = [torch.empty(shape, dtype=dt, device="cuda") for shape, dt in specs]
        hold()
        for j in junk:
            j.fill_(1 if j.dtype == torch.bool else 0x5A)
        del junk
        got = call()
        torch.cuda.synchronize()
        return got

    cap = max(1024, t.numel() // 8)
    r = reused([((n + 1,), torch.int64), ((cap, 3), torch.int32)], lambda: pma.scan_batch_device(mode, t, o, stream=sarg))
    assert np.array_equal(r.offsets.cpu().numpy(), want["offs"]), "scan_batch_device offsets"
    assert np.array_equal(_u32(r.matches).reshape(-1, 3), want["m"]), "scan_batch_device matches"
    got = reused([((n,), torch.int64)], lambda: pma.count_batch_device(mode, t, o, stream=sarg))
    assert np.array_equal(got.cpu().numpy(), want["counts"]), "count_batch_device"
    first, found = reused([((n, 3), torch.int32), ((n,), torch.bool)], lambda: pma.first_batch_device(mode, t, o, stream=sarg))
    assert np.array_equal(found.cpu().numpy(), want["found"]) and np.array_equal(_u32(first).reshape(n, 3), want["first"]), "first"
    got = reused([((t.numel(),), torch.uint8)], lambda: pma.mask_batch_device(mode, t, o, fill=0x2A, stream=sarg))
    assert np.array_equal(got.cpu().numpy(), want["mask"]), "mask_batch_device"
    if stream_case:
        ws = want_st
        st = zeros_state()
        r = reused([((n + 1,), torch.int64), ((cap, 3), torch.int32)], lambda: pma.scan_stream_device(mode, t, o, st, stream=sarg))
        assert np.array_equal(r.offsets.cpu().numpy(), ws["offs"]) and np.array_equal(_u32(r.matches).reshape(-1, 3), ws["m"])
        assert torch.equal(st, ref_state)
        st = zeros_state()
        got = reused([((n,), torch.int64)], lambda: pma.count_stream_device(mode, t, o, st, stream=sarg))
        assert np.array_equal(got.cpu().numpy(), ws["counts"]) and torch.equal(st, ref_state), "count_stream_device"
        st = zeros_state()
        first, found = reused([((n, 3), torch.int32), ((n,), torch.bool)], lambda: pma.first_stream_device(mode, t, o, st, stream=sarg))
        assert np.array_equal(found.cpu().numpy(), ws["found"]) and np.array_equal(_u32(first).reshape(n, 3), ws["first"])
        assert torch.equal(st, ref_state), "first_stream_device"


@AS_INT
@pytest.mark.parametrize("kind,mode", [c for c in FORM_CASES if c[0] != "cw"])
def test_fresh_input_on_a_second_stream(kind, mode, as_int):
    """c. The text is copied on the current stream, held busy, just before the call reads the copy on S (the copy's
    block held junk before)."""
    import torch

    F = _Forms(kind, mode, as_int)
    pma, t, o, want, sarg = F.pma, F.t, F.o, F.want, F.sarg
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    tmp = torch.full_like(t, JUNK)
    torch.cuda.synchronize()
    del tmp
    hold()
    t2 = t.clone()
    got = pma.count_batch_device(mode, t2, o, stream=sarg)
    torch.cuda.synchronize()
    assert np.array_equal(got.cpu().numpy(), want["counts"]), "count_batch_device of a fresh copy"


def _halves(text, offs):
    """Every haystack cut in two chunks at the first char boundary at or after its middle: (round 1, round 2) as
    (text, offsets, stream positions)."""
    o = offs.astype(np.int64)
    rounds = ([], [])
    cuts = []
    for i in range(len(o) - 1):
        h = text[o[i]:o[i + 1]]
        c = len(h) // 2
        while c < len(h) and (h[c] & 0xC0) == 0x80:
            c += 1
        rounds[0].append(h[:c])
        rounds[1].append(h[c:])
        cuts.append(c)
    out = []
    for r, pos in zip(rounds, (np.zeros(len(cuts), np.uint32), np.array(cuts, dtype=np.uint32))):
        ro = np.concatenate([[0], np.cumsum([len(x) for x in r])]).astype(np.int64)
        out.append((np.concatenate(r), ro, pos))
    return out


@pytest.mark.parametrize("as_int", [True, False], ids=["raw-handle", "stream-object"])
@pytest.mark.parametrize("kind,mode", [("bw", D.FIND), ("bw", D.FIND_OVERLAPPING), ("cw", D.FIND_OVERLAPPING)])
def test_stream_overflow_retry_on_a_second_stream(kind, mode, as_int):
    """d. scan_stream_device on S with an `out` too small for the chunk while the current stream is held: the retry
    restarts from the states the call was given.  Both rounds' matches and the final states are the stepper's."""
    import torch

    cw = kind == "cw"
    pma, opma = automaton(kind)
    text, offs = batch(cw, 512, 2000, seed=13)
    want = expected(opma, STEPPER[mode], text, offs, n_values(pma))
    (t1, o1, p1), (t2, o2, p2) = _halves(text, offs)
    n = len(offs) - 1
    d1, d2 = on_device(t1, o1), on_device(t2, o2)
    pos1, pos2 = (torch.from_numpy(p.view(np.int32)).cuda() for p in (p1, p2))
    ref = torch.zeros(n, dtype=torch.int32, device="cuda")
    for (tt, oo) in (d1, d2):
        pma.count_stream_device(mode, tt, oo, ref)
    state = torch.zeros(n, dtype=torch.int32, device="cuda")
    r1 = pma.scan_stream_device(mode, d1[0], d1[1], state, pos1)
    small = torch.zeros((1, 3), dtype=torch.int32, device="cuda")
    S_ = torch.cuda.Stream()
    torch.cuda.synchronize()
    hold()
    r2 = pma.scan_stream_device(mode, d2[0], d2[1], state, pos2, out=small, stream=S_.cuda_stream if as_int else S_)
    torch.cuda.synchronize()
    assert r2.matches.shape[0] > 1  # it did overflow `small`
    m1, m2 = _u32(r1.matches).reshape(-1, 3), _u32(r2.matches).reshape(-1, 3)
    oo1, oo2 = r1.offsets.cpu().numpy(), r2.offsets.cpu().numpy()
    for i in range(n):
        got = np.concatenate([m1[oo1[i]:oo1[i + 1]], m2[oo2[i]:oo2[i + 1]]])
        assert np.array_equal(got, want["m"][want["offs"][i]:want["offs"][i + 1]]), i
    assert torch.equal(state, ref)
    if not cw:
        sv = _u32(state)
        o = offs.astype(np.int64)
        for i in range(0, n, 97):
            assert int(sv[i]) == opma.state_after(bytes(text[o[i]:o[i + 1]]), find_mode=(mode == D.FIND)), i


def test_same_stream_issues_no_wait(monkeypatch):
    """e. stream=None, the current stream's raw handle and the current stream object: the same results, the same
    library launches, and no wait; another stream: the same results and launches, one wait per library call."""
    import torch

    pma, opma = automaton("bw")
    mode = D.FIND_OVERLAPPING
    text, offs = batch(False, 256, 3000, seed=17)
    t, o = on_device(text, offs)
    want = expected(opma, mode, text, offs, n_values(pma))
    waits = []
    real = A._wait_stream
    monkeypatch.setattr(A, "_wait_stream", lambda *a: (waits.append(a[0]), real(*a)))
    cur = torch.cuda.current_stream()
    other = torch.cuda.Stream()
    pma.scan_batch_device(mode, t, o)
    launches = {}
    for name, sarg in (("none", None), ("handle", cur.cuda_stream), ("object", cur), ("other", other)):
        del waits[:]
        l0 = pma.stats()["launches"]
        r = pma.scan_batch_device(mode, t, o, stream=sarg)
        c = pma.count_batch_device(mode, t, o, stream=sarg)
        h = pma.pattern_counts_device(mode, t, o, stream=sarg)
        launches[name] = pma.stats()["launches"] - l0
        torch.cuda.synchronize()
        assert np.array_equal(r.offsets.cpu().numpy(), want["offs"]) and np.array_equal(_u32(r.matches).reshape(-1, 3), want["m"])
        assert np.array_equal(c.cpu().numpy(), want["counts"]) and np.array_equal(h.cpu().numpy(), want["hist"])
        if name == "other":
            assert waits == [other.cuda_stream] * 3, name
        else:
            assert waits == [], name
    assert len(set(launches.values())) == 1 and launches["none"] > 0, launches


# ---- 2. tensors handed to jobs ------------------------------------------------------------------------------------

@pytest.mark.parametrize("n_jobs", [1, 2])
def test_job_tensors_live_in_stream_order(n_jobs):
    """Scans held back behind a spin on the scan stream, placements on their own stream, each placement given a base
    tensor the test drops at once; the next scan is enqueued before any wait and the test drops its references to
    the text and offsets it handed over, then allocates blocks shaped like that text on the current stream and fills
    them with junk.  Every step lands at its base, equal to the oracle."""
    import torch

    pma, opma = automaton("bw")
    mode = D.FIND_OVERLAPPING
    steps = 4
    batches = [batch(False, 1024, 4096, seed=40 + s) for s in range(steps)]  # 4 MiB each: not in the small-block pool
    wants = [expected(opma, mode, tx, of, n_values(pma)) for tx, of in batches]
    cap = max(len(w["m"]) for w in wants) + 4096
    jobs = [pma.job(0) for _ in range(n_jobs)]
    st_scan, st_place = torch.cuda.Stream(), torch.cuda.Stream()
    cur = torch.cuda.current_stream()
    outs = [torch.zeros((cap + 16, 3), dtype=torch.int32, device="cuda") for _ in range(steps)]
    oofs = [torch.zeros(len(of), dtype=torch.int64, device="cuda") for _, of in batches]

    def run(raced):
        if raced:
            hold(st_scan)
        for s in range(steps):
            j = jobs[s % n_jobs]
            t, o = on_device(*batches[s])
            st_scan.wait_stream(cur)  # the inputs were written on the current stream: the caller orders them
            j.scan(mode, t, o, cap, stream=st_scan)
            size = t.numel()
            del t, o
            # as many text-sized blocks as take every free one of that size, the block of the text just dropped
            # included (a freed block merges with its free neighbours, so one allocation might land beside it); the
            # run that sizes the workspaces caches them, so that the raced run needs no cudaMalloc
            junk = [torch.empty(size, dtype=torch.uint8, device="cuda") for _ in range(8)]
            for x in junk:
                x.fill_(JUNK)
            del junk, x
            base = torch.tensor([5 + s], dtype=torch.int64, device="cuda")
            st_place.wait_stream(cur)
            j.place(outs[s], oofs[s], base=base, stream=st_place)
            del base
        for j in jobs:
            j.wait()
        torch.cuda.synchronize()

    run(False)  # sizes the jobs' workspaces and caches the junk blocks: no cudaFree or cudaMalloc inside the raced run
    for x in outs + oofs:
        x.zero_()
    torch.cuda.synchronize()
    run(True)
    for s, w in enumerate(wants):
        b, k = 5 + s, len(w["m"])
        assert np.array_equal(oofs[s].cpu().numpy(), w["offs"] + b), s
        assert np.array_equal(_u32(outs[s][b:b + k]).reshape(-1, 3), w["m"]), s


# ---- 3. host threads, one job each ---------------------------------------------------------------------------------

THREAD_SIZES = [(1, 1024), (64, 1024), (256, 4096), (2048, 4096), (16384, 4096)]  # 1 KiB .. 64 MiB
ORACLE_MAX = 1 << 20


def _references(pma, opma, mode, cw, sizes, seed):
    """Per batch: device text and offsets, and the expected matches and offsets on the device -- from the oracle up
    to 1 MiB, from the blocking call on the current stream above (checked against the oracle on a prefix)."""
    import torch

    refs = []
    for i, (n, hay_len) in enumerate(sizes):
        text, offs = batch(cw, n, hay_len, seed=seed + i)
        t, o = on_device(text, offs)
        if text.size <= ORACLE_MAX:
            w = expected(opma, mode, text, offs, n_values(pma))
            wm = torch.from_numpy(w["m"].view(np.int32)).cuda().reshape(-1, 3)
            wo = torch.from_numpy(w["offs"]).cuda()
        else:
            r = pma.scan_batch_device(mode, t, o)
            wm, wo = r.matches.clone(), r.offsets.clone()
            k = 64
            w = expected(opma, mode, text[: int(offs[k])], offs[: k + 1], n_values(pma))
            assert np.array_equal(_u32(wm[: len(w["m"])]).reshape(-1, 3), w["m"])
            assert np.array_equal(wo[: k + 1].cpu().numpy(), w["offs"])
        refs.append((t, o, wm, wo))
    torch.cuda.synchronize()
    return refs


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
    stuck = [i for i, th in enumerate(threads) if th.is_alive()]
    assert not stuck, "threads %s did not finish in %d s" % (stuck, THREAD_TIMEOUT_S)
    assert not errors, errors


@pytest.mark.parametrize("kind,mode", [("bw", D.FIND), ("bw", D.FIND_OVERLAPPING), ("bw", D.FIND_OVERLAPPING_NO_SUFFIX),
                                       ("bw-lf", D.LEFTMOST_FIND), ("cw", D.FIND_OVERLAPPING)])
def test_threads_with_a_job_each(kind, mode):
    """8 threads, each with its own job and stream, 5 rounds on one automaton; every thread takes the batches in its
    own order, so the workspaces grow and shrink between rounds."""
    import torch

    pma, opma = automaton(kind)
    refs = _references(pma, opma, mode, kind == "cw", THREAD_SIZES, seed=60)

    def worker(i):
        job = pma.job(0)
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            for r in range(len(refs)):
                t, o, wm, wo = refs[(i + r * (1 + i % 2)) % len(refs)]
                k = wm.shape[0]
                out = torch.empty((k + 16, 3), dtype=torch.int32, device="cuda")
                oo = torch.empty(o.numel(), dtype=torch.int64, device="cuda")
                job.scan(mode, t, o, k + 4096, stream=st if r % 2 else None)
                job.place(out, oo, stream=st.cuda_stream if r % 2 else None)
                assert job.wait() == k, (i, r)
                assert torch.equal(oo, wo) and torch.equal(out[:k], wm), (i, r)

    _run_threads(8, worker)


# ---- 4. host threads sharing one handle ---------------------------------------------------------------------------

def test_threads_share_a_handle():
    """Threads 0-3: every synchronous form on one automaton, each thread on its own stream (half of them through
    stream=, half as their current stream), stream chunks with a state of their own; threads 4-5: jobs of the same
    automaton; thread 6: a second automaton side by side; thread 7: keeps passing descending offsets and gets
    INVALID_ARGUMENT with its own message, which no other thread sees."""
    import torch

    mode = D.FIND_OVERLAPPING
    pma, opma = automaton("bw")
    cpma, copma = automaton("cw")
    nv, cnv = n_values(pma), n_values(cpma)
    text, offs = batch(False, 256, 1000, seed=80)
    t, o = on_device(text, offs)
    want = expected(opma, mode, text, offs, nv)
    want_st = expected(opma, STEPPER[mode], text, offs, nv)
    ctext, coffs = batch(True, 256, 1000, seed=81)
    ct, co = on_device(ctext, coffs)
    cwant = expected(copma, mode, ctext, coffs, cnv)
    n = len(offs) - 1
    ref_state = torch.zeros(n, dtype=torch.int32, device="cuda")
    pma.count_stream_device(mode, t, o, ref_state)
    bad_o = torch.tensor([0, 500, 200, 1000], dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    last_errors = [None] * 8
    rounds = 4

    def forms(i, st):
        sarg = st if i % 2 else None
        for r in range(rounds):
            res = pma.scan_batch_device(mode, t, o, stream=sarg)
            assert np.array_equal(res.offsets.cpu().numpy(), want["offs"]) and np.array_equal(_u32(res.matches).reshape(-1, 3), want["m"])
            assert np.array_equal(pma.count_batch_device(mode, t, o, stream=sarg).cpu().numpy(), want["counts"])
            first, found = pma.first_batch_device(mode, t, o, stream=sarg)
            assert np.array_equal(_u32(first).reshape(n, 3), want["first"]) and np.array_equal(found.cpu().numpy(), want["found"])
            for key in ("value", "output"):
                check_hist(pma, pma.pattern_counts_device(mode, t, o, key=key, stream=sarg), want["hist"], key, (i, r, key))
                check_df(pma, pma.doc_counts_device(mode, t, o, key=key, stream=sarg), want["df"], key, (i, r, key))
            assert np.array_equal(pma.mask_batch_device(mode, t, o, fill=0x2A, stream=sarg).cpu().numpy(), want["mask"])
            state = torch.zeros(n, dtype=torch.int32, device="cuda")
            res = pma.scan_stream_device(mode, t, o, state, stream=sarg)
            assert np.array_equal(_u32(res.matches).reshape(-1, 3), want_st["m"])
            assert torch.equal(state, ref_state)
            state.zero_()
            assert np.array_equal(pma.count_stream_device(mode, t, o, state, stream=sarg).cpu().numpy(), want_st["counts"])
            state.zero_()
            check_hist(pma, pma.pattern_counts_stream_device(mode, t, o, state, stream=sarg), want_st["hist"], "value", (i, r))
            assert torch.equal(state, ref_state)

    def jobs(i, st):
        job = pma.job(0)
        k = len(want["m"])
        for r in range(rounds * 3):
            out = torch.empty((k + 8, 3), dtype=torch.int32, device="cuda")
            oo = torch.empty(n + 1, dtype=torch.int64, device="cuda")
            job.scan(mode, t, o, k + 4096, stream=st)
            job.place(out, oo, stream=st)
            assert job.wait() == k
            assert np.array_equal(oo.cpu().numpy(), want["offs"]) and np.array_equal(_u32(out[:k]).reshape(-1, 3), want["m"])

    def second(i, st):
        for r in range(rounds):
            res = cpma.scan_batch_device(mode, ct, co)
            assert np.array_equal(res.offsets.cpu().numpy(), cwant["offs"]) and np.array_equal(_u32(res.matches).reshape(-1, 3), cwant["m"])
            assert np.array_equal(cpma.count_batch_device(mode, ct, co).cpu().numpy(), cwant["counts"])
            check_hist(cpma, cpma.pattern_counts_device(mode, ct, co), cwant["hist"], "value", (i, r))

    def refused(i, st):
        for r in range(rounds * 4):
            with pytest.raises(D.DaachorseError) as e:
                pma.count_batch_device(mode, t, bad_o)
            assert e.value.code == _lib.INVALID_ARGUMENT
            msg = _lib.last_error()
            assert "ascending" in msg and msg in str(e.value), msg

    def worker(i):
        st = torch.cuda.Stream()
        role = forms if i < 4 else jobs if i < 6 else second if i == 6 else refused
        if role is forms and i % 2:
            role(i, st)  # stream=st with the thread's default stream current
        else:
            with torch.cuda.stream(st):
                role(i, st)
        last_errors[i] = _lib.last_error()

    _run_threads(8, worker)
    assert "ascending" in last_errors[7]
    for i in range(7):
        assert "ascending" not in last_errors[i], (i, last_errors[i])


# ---- 5. pipelined jobs with changing sizes ---------------------------------------------------------------------------

PIPE_SIZES = [(1, 4096), (24576, 4096), (256, 4096), (76800, 4096)]  # 4 KiB, 96 MiB, 1 MiB, 300 MiB (past 256 MiB)
PIPE_STEPS = 12


@functools.lru_cache(maxsize=None)
def _pipe_batches():
    """The four batches on the device, made from the pool on the device (300 MiB is not built on the host)."""
    import torch

    _, pool, b = _source(False)
    pool_t = torch.from_numpy(pool).cuda()
    out = []
    for i, (n, hay_len) in enumerate(PIPE_SIZES):
        starts = torch.from_numpy(S.window_starts(b, len(pool), n, hay_len, seed=90 + i)).cuda()
        out.append(S.materialise_on_device(pool_t, starts, hay_len))
    torch.cuda.synchronize()
    return out


@functools.lru_cache(maxsize=None)
def _pipe_refs(kind, mode):
    pma, opma = automaton(kind)
    refs = []
    for t, o in _pipe_batches():
        r = pma.scan_batch_device(mode, t, o)
        if t.numel() <= ORACLE_MAX:
            w = expected(opma, mode, t.cpu().numpy(), o.cpu().numpy().astype(np.uint64), n_values(pma))
            assert np.array_equal(r.offsets.cpu().numpy(), w["offs"]) and np.array_equal(_u32(r.matches).reshape(-1, 3), w["m"])
        refs.append((r.matches.clone(), r.offsets.clone()))
    return refs


@pytest.mark.parametrize("gather_ordered", [1, 2])
@pytest.mark.parametrize("n_jobs", [1, 2])
@pytest.mark.parametrize("kind,mode", [("bw", D.FIND), ("bw", D.FIND_OVERLAPPING), ("bw-ll", D.LEFTMOST_FIND)])
def test_pipelined_jobs_with_changing_sizes(kind, mode, n_jobs, gather_ordered):
    """12 steps cycling 4 KiB -> 96 MiB -> 1 MiB -> 300 MiB, queued as bench.py's run_pipeline queues them (with two
    jobs the scan of step s+1 before step s is placed), placement on its own stream; every step equals the blocking
    call on its batch, which equals the oracle on the batches of 1 MiB and less."""
    import torch

    import bench

    pma, _ = automaton(kind)
    batches = _pipe_batches()
    refs = _pipe_refs(kind, mode)
    cap = max(int(m.shape[0]) for m, _ in refs) + 4096
    jobs = [pma.job(0) for _ in range(n_jobs)]
    st_scan = torch.cuda.Stream(priority=-1)
    st_place = torch.cuda.Stream()
    outs = [torch.empty((cap, 3), dtype=torch.int32, device="cuda") for _ in range(n_jobs)]
    oofs = [torch.empty(max(o.numel() for _, o in batches), dtype=torch.int64, device="cuda") for _ in range(n_jobs)]
    checked = []
    pma.set_option("gather_ordered", gather_ordered)
    try:
        torch.cuda.synchronize()
        st_scan.wait_stream(torch.cuda.current_stream())

        def scan(s):
            t, o = batches[s % len(batches)]
            jobs[s % n_jobs].scan(mode, t, o, cap, stream=st_scan)

        def place(s):
            o = batches[s % len(batches)][1]
            jobs[s % n_jobs].place(outs[s % n_jobs], oofs[s % n_jobs][: o.numel()], stream=st_place)

        def finish(s):
            k = jobs[s % n_jobs].wait()
            wm, wo = refs[s % len(refs)]
            assert k == wm.shape[0], s
            assert torch.equal(oofs[s % n_jobs][: wo.numel()], wo), s
            assert torch.equal(outs[s % n_jobs][:k], wm), s
            checked.append(s)
            return k

        bench.run_pipeline(PIPE_STEPS, n_jobs, scan, place, finish)
    finally:
        pma.set_option("gather_ordered", 1)
        torch.cuda.synchronize()
    assert checked == list(range(PIPE_STEPS))
