"""Counts, first matches and per-pattern histograms of stream chunks on the GPU (dach_dev_count_stream /
dach_dev_first_stream / dach_dev_hist_stream): every round against dach_dev_scan_stream on the same chunks with the
state carried side by side, calls of every kind taking turns on one stream against the oracle stepper, FIRST's stream
positions across 2^32, and the refusals, which must leave every caller buffer as it was."""
import ctypes as C

import numpy as np
import pytest

import daachorse_b200 as D
import oracle_api as O
from daachorse_b200 import _lib
from daachorse_b200 import synth as S

pytestmark = pytest.mark.gpu

STEPPER = {D.FIND: O.FIND_STEPPER, D.FIND_OVERLAPPING: O.FIND_OVERLAPPING_STEPPER}


def _cuda(a, dtype=None):
    import torch

    a = np.ascontiguousarray(a)
    if a.size == 0:
        return torch.zeros(16, dtype=dtype or torch.uint8, device="cuda")[:0]
    return torch.from_numpy(a).cuda()


def bytewise_case(n=1000, seed=21):
    cfg = S.config("C2")
    ps = S.make_patterns(cfg, n=4000)
    pool, _ = S.make_pool(cfg, ps, 4 << 20)
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 1200, size=n)
    starts = rng.integers(0, len(pool) - 1300, size=n)
    streams = [np.ascontiguousarray(pool[int(s): int(s) + int(l)]) for s, l in zip(starts, lens)]
    cuts = [np.arange(len(s) + 1) for s in streams]
    return ps.as_list(), D.DoubleArrayAhoCorasick.new(ps.as_list()), O.OraclePma.build_packed(ps.blob, ps.offs), streams, cuts, 400


def charwise_case(n=800, seed=33):
    cfg = S.config("C4")
    ps = S.make_patterns(cfg, n=5000)
    pool, b = S.make_pool(cfg, ps, 4 << 20)
    rng = np.random.default_rng(seed)
    bi = np.sort(rng.integers(0, len(b) - 400, size=n))
    nt = rng.integers(0, 300, size=n)
    streams, cuts = [], []
    for i in range(n):
        lo, hi = int(b[bi[i]]), int(b[bi[i] + int(nt[i])])
        streams.append(np.ascontiguousarray(pool[lo:hi]))
        cuts.append((b[bi[i]: bi[i] + int(nt[i]) + 1] - lo).astype(np.int64))  # token starts: char boundaries
    pats = [p.decode() for p in ps.as_list()]
    return pats, D.CharwiseDoubleArrayAhoCorasick.new(pats), O.OraclePma.build(pats, charwise=True), streams, cuts, 60


def rounds(streams, cuts, max_step, seed):
    """Ragged chunks (empty ones included) until every stream is consumed: (text, offs int64, chunk starts)."""
    rng = np.random.default_rng(seed)
    at = np.zeros(len(streams), dtype=np.int64)
    while any(at[i] < len(cuts[i]) - 1 for i in range(len(streams))):
        chunks, starts = [], []
        for i, s in enumerate(streams):
            j = min(int(at[i] + rng.integers(0, max_step + 1)), len(cuts[i]) - 1)
            p, q = int(cuts[i][at[i]]), int(cuts[i][j])
            chunks.append(s[p:q])
            starts.append(p)
            at[i] = j
        offs = np.zeros(len(chunks) + 1, dtype=np.int64)
        offs[1:] = np.cumsum([len(c) for c in chunks])
        yield np.concatenate(chunks) if offs[-1] else np.zeros(0, np.uint8), offs, np.array(starts, dtype=np.uint32)


def stepper_matches(opma, mode, streams):
    """The oracle stepper over each whole stream, per stream an (k, 3) uint32 array without matches() of the initial
    state (end 0)."""
    offs = np.zeros(len(streams) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(s) for s in streams])
    ref = opma.scan_batch(STEPPER[mode], np.concatenate(streams), offs, nthreads=16, want_matches=True)
    rm = ref["matches"]
    ro = np.concatenate([[0], np.cumsum(ref["counts"])]).astype(np.int64)
    out = []
    for i in range(len(streams)):
        m = np.stack([rm["start"][ro[i]:ro[i + 1]], rm["end"][ro[i]:ro[i + 1]], rm["value"][ro[i]:ro[i + 1]]], axis=1).astype(np.uint32)
        out.append(m[m[:, 1] != 0])
    return out


def _u32(t):
    return t.cpu().numpy().view(np.uint32)


CASES = ([pytest.param(False, m, k, h, id="bytewise-%s-kernel%d-hot%s" % (m, k, h)) for m in (D.FIND, D.FIND_OVERLAPPING)
          for k in (1, 2, 3, 4) for h in (0, None)]
         + [pytest.param(True, m, k, None, id="charwise-%s-kernel%d" % (m, k)) for m in (D.FIND, D.FIND_OVERLAPPING) for k in (1, 3)])


@pytest.mark.parametrize("cw,mode,kernel,hot", CASES)
def test_every_round_equals_the_matches_stream(cw, mode, kernel, hot):
    """Per round: COUNT = the out_offs differences of scan_stream_device, FIRST = its first tuple per chunk (stream
    coordinates in even rounds, chunk-relative in odd ones), HIST = the bincount of its values under both keys; five
    state tensors carried side by side stay bit for bit equal."""
    import torch

    _, pma, _, streams, cuts, step = charwise_case() if cw else bytewise_case()
    if hot is not None:
        pma.set_option("hot_entries", hot)
    vals = pma.outputs()[0].astype(np.int64)
    n = len(streams)
    st = {k: torch.zeros(n, dtype=torch.int32, device="cuda") for k in ("matches", "count", "first", "value", "output")}
    total = 0
    for r, (text, offs, starts) in enumerate(rounds(streams, cuts, step, seed=5 + kernel)):
        t, o, p = _cuda(text), _cuda(offs), _cuda(starts.view(np.int32))
        pma.set_option("kernel", kernel if (cw or kernel >= 2) else 3)  # the matches path has no stream form on kernel 1
        m = pma.scan_stream_device(mode, t, o, st["matches"], p)
        pma.set_option("kernel", kernel)
        counts = pma.count_stream_device(mode, t, o, st["count"])
        first, found = pma.first_stream_device(mode, t, o, st["first"], pos=p if r % 2 == 0 else None)
        hv = pma.pattern_counts_stream_device(mode, t, o, st["value"], key="value")
        ho = pma.pattern_counts_stream_device(mode, t, o, st["output"], key="output")
        mm = _u32(m.matches).reshape(-1, 3)
        oo = m.offsets.cpu().numpy()
        want_counts = np.diff(oo)
        assert np.array_equal(counts.cpu().numpy(), want_counts), r
        has = want_counts > 0
        assert np.array_equal(found.cpu().numpy(), has), r
        want_first = np.full((n, 3), 0xFFFFFFFF, dtype=np.uint32)
        want_first[has] = mm[oo[:-1][has]]
        if r % 2:
            want_first[has, :2] -= starts[has, None]
        assert np.array_equal(_u32(first).reshape(n, 3), want_first), r
        want_hist = np.bincount(mm[:, 2].astype(np.int64), minlength=hv.numel())
        assert np.array_equal(hv.cpu().numpy(), want_hist), r
        assert np.array_equal(np.bincount(vals, weights=ho.cpu().numpy().astype(np.float64), minlength=hv.numel()), want_hist), r
        for k in ("count", "first", "value", "output"):
            assert torch.equal(st[k], st["matches"]), (r, k)
        total += len(mm)
    assert total > 0


@pytest.mark.parametrize("cw,mode", [(False, D.FIND), (False, D.FIND_OVERLAPPING), (True, D.FIND), (True, D.FIND_OVERLAPPING)])
def test_alternating_forms_equal_the_stepper(cw, mode):
    """COUNT, HIST, FIRST and the matches call take turns on one state tensor; every round's result is the stepper's
    over the whole stream restricted to the chunk, and the final states are the crate's."""
    import torch

    _, pma, opma, streams, cuts, step = charwise_case(n=500) if cw else bytewise_case(n=600)
    ref = stepper_matches(opma, mode, streams)
    n = len(streams)
    state = torch.zeros(n, dtype=torch.int32, device="cuda")
    hist = torch.zeros(int(pma.outputs()[0].max()) + 1, dtype=torch.int64, device="cuda")
    want_hist = np.zeros(hist.numel(), dtype=np.int64)
    for r, (text, offs, starts) in enumerate(rounds(streams, cuts, step, seed=77)):
        t, o, p = _cuda(text), _cuda(offs), _cuda(starts.view(np.int32))
        ends = starts + np.diff(offs).astype(np.uint32)
        want = [ref[i][(ref[i][:, 1] > starts[i]) & (ref[i][:, 1] <= ends[i])] for i in range(n)]
        kind = r % 4
        if kind == 0:
            got = pma.count_stream_device(mode, t, o, state).cpu().numpy()
            assert np.array_equal(got, [len(w) for w in want]), r
        elif kind == 1:
            pma.pattern_counts_stream_device(mode, t, o, state, out=hist)
            for w in want:
                want_hist += np.bincount(w[:, 2].astype(np.int64), minlength=len(want_hist))
        elif kind == 2:
            first, found = pma.first_stream_device(mode, t, o, state, pos=p)
            first, found = _u32(first).reshape(n, 3), found.cpu().numpy()
            for i in range(n):
                assert found[i] == (len(want[i]) > 0), (r, i)
                if len(want[i]):
                    assert tuple(first[i]) == tuple(want[i][0]), (r, i)
        else:
            m = pma.scan_stream_device(mode, t, o, state, p)
            mm, oo = _u32(m.matches).reshape(-1, 3), m.offsets.cpu().numpy()
            for i in range(n):
                assert np.array_equal(mm[oo[i]:oo[i + 1]], want[i]), (r, i)
    assert np.array_equal(hist.cpu().numpy(), want_hist)
    if not cw:
        stv = _u32(state)
        for i in range(0, n, 37):
            assert int(stv[i]) == opma.state_after(bytes(streams[i]), find_mode=(mode == D.FIND)), i


@pytest.mark.parametrize("mode", [D.FIND, D.FIND_OVERLAPPING])
def test_first_positions_wrap_modulo_2_32(mode):
    """d_pos near 2^32: start and end wrap as the matches stream's do; without d_pos they are chunk-relative."""
    import torch

    pma = D.DoubleArrayAhoCorasick.new(["ab", "b", "abcab", "ca"])
    chunks = [b"xxab", b"cab", b"", b"zzzzzzzzzzzzzzzzzzzzzzzzzzzzzzzzzzzzab", b"b"]
    text = np.frombuffer(b"".join(chunks), dtype=np.uint8)
    offs = np.concatenate([[0], np.cumsum([len(c) for c in chunks])]).astype(np.int64)
    pos = np.array([0xFFFFFFFE, 0xFFFFFFFD, 0xFFFFFFFF, 0xFFFFFFF0, 7], dtype=np.uint32)
    t, o, p = _cuda(text), _cuda(offs), _cuda(pos.view(np.int32))
    s_m, s_f, s_r = (torch.zeros(len(chunks), dtype=torch.int32, device="cuda") for _ in range(3))
    m = pma.scan_stream_device(mode, t, o, s_m, p)
    first, found = pma.first_stream_device(mode, t, o, s_f, pos=p)
    rel, found_r = pma.first_stream_device(mode, t, o, s_r)
    mm, oo = _u32(m.matches).reshape(-1, 3), m.offsets.cpu().numpy()
    has = np.diff(oo) > 0
    assert np.array_equal(found.cpu().numpy(), has) and np.array_equal(found_r.cpu().numpy(), has)
    assert has.sum() == 4
    want = np.full((len(chunks), 3), 0xFFFFFFFF, dtype=np.uint32)
    want[has] = mm[oo[:-1][has]]
    assert np.array_equal(_u32(first).reshape(-1, 3), want)
    assert (want[has, 1] < pos[has]).any()  # some of them did wrap
    want[has, :2] -= pos[has, None]
    assert np.array_equal(_u32(rel).reshape(-1, 3), want)
    assert torch.equal(s_f, s_m) and torch.equal(s_r, s_m)


def _sentinels(n, n_hist):
    import torch

    return {"state": torch.arange(1, n + 1, dtype=torch.int32, device="cuda"),
            "counts": torch.full((n,), 0x5A5A5A5A, dtype=torch.int64, device="cuda"),
            "first": torch.full((n, 3), 0x3C3C3C3C, dtype=torch.int32, device="cuda"),
            "found": torch.full((n,), 7, dtype=torch.uint8, device="cuda"),
            "hist": torch.full((max(n_hist, 1),), 11, dtype=torch.int64, device="cuda")}


def _call_all(pma, mode, text, offs, n, text_bytes, buf, n_hist, key=1):
    """The three C calls on raw pointers (key 1: DACH_KEY_VALUE); their return codes."""
    import torch

    L = _lib.load()
    d = pma.device_handle(0)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    v = lambda x: C.c_void_p(x.data_ptr())  # noqa: E731
    tot = C.c_uint64()
    rc_c = L.dach_dev_count_stream(d, mode, v(text), v(offs), n, text_bytes, v(buf["state"]), v(buf["counts"]), C.byref(tot), st)
    rc_f = L.dach_dev_first_stream(d, mode, v(text), v(offs), n, text_bytes, v(buf["state"]), None, v(buf["first"]), v(buf["found"]),
                                   C.byref(tot), st)
    rc_h = L.dach_dev_hist_stream(d, mode, key, v(text), v(offs), n, text_bytes, v(buf["state"]), v(buf["hist"]), n_hist,
                                  C.byref(tot), st)
    torch.cuda.synchronize()
    return rc_c, rc_f, rc_h


def _unchanged(buf, n, n_hist):
    ref = _sentinels(n, n_hist)
    return all(bool((buf[k] == ref[k]).all()) for k in ref)


def test_refusals_leave_every_buffer_as_it_was():
    import torch

    pats = ["ab", "b", "bca"]
    pma = D.DoubleArrayAhoCorasick.new(pats)
    n_hist = len(pats)
    text = _cuda(np.frombuffer(b"abcab" * 40, dtype=np.uint8))
    good = [0, 50, 50, 200]
    for bad, tb in (([0, 50, 20, 200], 200), ([0, 50, 100, 300], 200), ([0, 50, 100, 200], 150)):
        buf = _sentinels(3, n_hist)
        rcs = _call_all(pma, D.FIND_OVERLAPPING, text, torch.tensor(bad, dtype=torch.int64, device="cuda"), 3, tb, buf, n_hist)
        assert rcs == (_lib.INVALID_ARGUMENT,) * 3, (bad, tb)
        assert _unchanged(buf, 3, n_hist), (bad, tb)
    o = torch.tensor(good, dtype=torch.int64, device="cuda")
    # n_hist below the largest value + 1: the histogram call is refused before anything runs
    buf = _sentinels(3, n_hist)
    v = lambda x: C.c_void_p(x.data_ptr())  # noqa: E731
    rc = _lib.load().dach_dev_hist_stream(pma.device_handle(0), D.FIND_OVERLAPPING, 1, v(text), v(o), 3, 200, v(buf["state"]),
                                          v(buf["hist"]), n_hist - 1, None, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert rc == _lib.INVALID_ARGUMENT
    assert _unchanged(buf, 3, n_hist)
    # a leftmost automaton: its mode has no stepper, a Standard mode is the wrong kind
    lm = D.DoubleArrayAhoCorasickBuilder.new().match_kind(D.MatchKind.LeftmostLongest).build(pats)
    for mode, rc in ((D.LEFTMOST_FIND, _lib.INVALID_ARGUMENT), (D.FIND, _lib.MATCH_KIND_MISMATCH)):
        buf = _sentinels(3, n_hist)
        assert _call_all(lm, mode, text, o, 3, 200, buf, n_hist) == (rc,) * 3, mode
        assert _unchanged(buf, 3, n_hist)
    # find with an empty pattern: no lane machine serves it
    empty = D.DoubleArrayAhoCorasick.new([""] + pats)
    buf = _sentinels(3, n_hist + 1)
    assert _call_all(empty, D.FIND, text, o, 3, 200, buf, n_hist + 1) == (_lib.INVALID_ARGUMENT,) * 3
    assert _unchanged(buf, 3, n_hist + 1)
    # option kernel = 0: the lane-per-haystack kernels have no stream form
    pma.set_option("kernel", 0)
    buf = _sentinels(3, n_hist)
    assert _call_all(pma, D.FIND, text, o, 3, 200, buf, n_hist) == (_lib.INVALID_ARGUMENT,) * 3
    assert _unchanged(buf, 3, n_hist)
    pma.set_option("kernel", 3)
    buf = _sentinels(3, n_hist)
    buf["state"].zero_()
    buf["hist"].zero_()
    assert _call_all(pma, D.FIND_OVERLAPPING, text, o, 3, 200, buf, n_hist)[0] == _lib.OK
