"""Counts, first matches and per-pattern histograms of stream chunks (dach_dev_count_stream / dach_dev_first_stream /
dach_dev_hist_stream) on the kernels' lane logic compiled for the CPU (tests/emu_stream_rk), against the
crate's steppers (oracle) driven over each whole stream.  No GPU needed; tests/test_gpu_stream_rk.py runs the device
forms against dach_dev_scan_stream."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import emu_api as EM
import emu_reduce_api as E
import oracle_api as O
from cases import MIXED

FIND, OVERLAPPING = 0, 1
COUNT, FIRST, HIST = 1, 2, 3
HERE = os.path.dirname(os.path.abspath(__file__))
STEPPER = {FIND: O.FIND_STEPPER, OVERLAPPING: O.FIND_OVERLAPPING_STEPPER}
NONE = (0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF)
KEY = {"output": 0, "value": 1}  # dach_hist_key


_LIB = None


def lib():
    """tests/emu_stream_rk/libdach_emu_stream_rk.so, built on first use."""
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-C", os.path.join(HERE, "emu_stream_rk"), "-s"])
        L = C.CDLL(os.path.join(HERE, "emu_stream_rk", "libdach_emu_stream_rk.so"))
        L.emu_rk_stream_wire.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                         C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_int64, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
        L.emu_rk_stream_wire.restype = C.c_int
        L.emu_stream_rk_set_hot_slots.argtypes = [C.c_uint32]
        _LIB = L
    return _LIB


def _call(wire, cw, mode, rk, text, offs, state, pos=None, key=0, hot_n=0, kernel=3, hist_smem=1024, counts=None, first=None,
          found=None, hist=None):
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    n = len(offs) - 1
    tot = C.c_uint64()
    pad = text if text.size else np.zeros(16, dtype=np.uint8)
    p = lambda a: a.ctypes.data if a is not None else None  # noqa: E731
    rc = lib().emu_rk_stream_wire(wire_a.ctypes.data, wire_a.size, int(cw), mode, rk, key, pad.ctypes.data, offs.ctypes.data, n,
                                  state.ctypes.data, p(pos), hot_n, kernel, hist_smem, p(counts), p(first), p(found), p(hist),
                                  hist.size if hist is not None else 0, C.byref(tot))
    return rc, tot.value


def count_stream(wire, cw, mode, text, offs, state, hot_n=0, kernel=3):
    """dach_dev_count_stream through the emulation: (rc, counts, total); ``state`` (uint32, n) updated in place."""
    n = len(offs) - 1
    counts = np.full(max(n, 1), 0xA5A5A5A5A5A5A5A5, dtype=np.uint64)
    rc, tot = _call(wire, cw, mode, COUNT, text, offs, state, hot_n=hot_n, kernel=kernel, counts=counts)
    return rc, counts[:n], tot


def first_stream(wire, cw, mode, text, offs, state, pos=None, hot_n=0, kernel=3):
    """dach_dev_first_stream through the emulation: (rc, first (n, 3) uint32, found bool, n_found)."""
    n = len(offs) - 1
    first = np.full((max(n, 1), 3), 0x5A5A5A5A, dtype=np.uint32)
    found = np.full(max(n, 1), 7, dtype=np.uint8)
    rc, nf = _call(wire, cw, mode, FIRST, text, offs, state, pos=pos, hot_n=hot_n, kernel=kernel, first=first, found=found)
    return rc, first[:n], found[:n].astype(bool), nf


def hist_stream(wire, cw, mode, key, text, offs, state, out, hot_n=0, kernel=3, hist_smem=1024):
    """dach_dev_hist_stream through the emulation: adds into ``out``; (rc, total)."""
    return _call(wire, cw, mode, HIST, text, offs, state, key=KEY[key], hot_n=hot_n, kernel=kernel, hist_smem=hist_smem, hist=out)


def bytewise_streams(seed, empty_pattern=False):
    """Patterns over "abc" (values = their indices), 70 streams of unequal length over "abcd", some empty; every byte is
    a place a chunk may end."""
    rng = np.random.default_rng(900 + seed)
    pats = sorted(set(bytes(rng.integers(97, 100, size=int(rng.integers(1, 7))).tolist()) for _ in range(60)))
    if empty_pattern:
        pats = [b""] + pats
    streams = [bytes(rng.integers(97, 101, size=int(rng.integers(0, 700))).tolist()) for _ in range(70)]
    streams[3] = b""
    cuts = [np.arange(len(s) + 1) for s in streams]
    return pats, streams, cuts


def charwise_streams(seed):
    """Charwise patterns over chars of 1-4 bytes and streams over them (and unmapped chars); chunks end on char
    boundaries only."""
    rng = np.random.default_rng(1900 + seed)
    alpha = 6
    pats = sorted(set("".join(MIXED[int(i)] for i in rng.integers(0, alpha, size=int(rng.integers(1, 6)))) for _ in range(50)))
    syms = MIXED[:alpha] + ["z", "語"]
    streams, cuts = [], []
    for _ in range(50):
        chars = [syms[int(i)] for i in rng.integers(0, len(syms), size=int(rng.integers(0, 300)))]
        streams.append("".join(chars).encode())
        cuts.append(np.concatenate([[0], np.cumsum([len(c.encode()) for c in chars])]).astype(np.int64))
    return pats, streams, cuts


def stepper_matches(opma, mode, streams):
    """The oracle stepper over each whole stream: per stream an (k, 3) uint32 array in report order, without matches()
    of the initial state (end 0), which no consume() produced."""
    lens = [len(s) for s in streams]
    offs = np.zeros(len(streams) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    whole = np.frombuffer(b"".join(streams), dtype=np.uint8)
    ref = opma.scan_batch(STEPPER[mode], whole, offs, want_matches=True)
    rm = ref["matches"]
    ro = np.concatenate([[0], np.cumsum(ref["counts"])]).astype(np.int64)
    out = []
    for i in range(len(streams)):
        m = np.stack([rm["start"][ro[i]:ro[i + 1]], rm["end"][ro[i]:ro[i + 1]], rm["value"][ro[i]:ro[i + 1]]], axis=1).astype(np.uint32)
        out.append(m[m[:, 1] != 0])
    return out


def rounds(streams, cuts, seed, max_step=14):
    """Rounds of ragged chunks: in each round stream i takes its next 0..max_step cut positions (empty chunks included),
    until every stream is consumed.  Yields (text, offs (uint64), chunk starts in stream coordinates)."""
    rng = np.random.default_rng(seed)
    at = np.zeros(len(streams), dtype=np.int64)  # index into cuts[i]
    while any(at[i] < len(cuts[i]) - 1 for i in range(len(streams))):
        chunks, starts = [], []
        for i, s in enumerate(streams):
            j = min(int(at[i] + rng.integers(0, max_step + 1)), len(cuts[i]) - 1)
            p, q = int(cuts[i][at[i]]), int(cuts[i][j])
            chunks.append(s[p:q])
            starts.append(p)
            at[i] = j
        offs = np.zeros(len(chunks) + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(c) for c in chunks])
        yield np.frombuffer(b"".join(chunks), dtype=np.uint8).copy(), offs, np.array(starts, dtype=np.uint32)


def run_case(wire, cw, mode, streams, cuts, opma, n_hist, hot_n=0, kernel=3, seed=0):
    """COUNT, FIRST and HIST (both keys) on four state vectors side by side, and the matches path of the emulation on a
    fifth; every chunk's results against the stepper's matches that end inside the chunk."""
    ref = stepper_matches(opma, mode, streams)
    n = len(streams)
    st = {k: np.zeros(n, dtype=np.uint32) for k in ("count", "first", "value", "output", "matches")}
    hv = np.zeros(n_hist["value"], dtype=np.uint64)
    ho = np.zeros(n_hist["output"], dtype=np.uint64)
    got_total = 0
    for r, (text, offs, starts) in enumerate(rounds(streams, cuts, seed)):
        ends = starts + np.diff(offs).astype(np.uint32)
        rc, counts, total = count_stream(wire, cw, mode, text, offs, st["count"], hot_n, kernel)
        assert rc == 0
        pos = starts if r % 2 == 0 else None  # stream coordinates, or chunk-relative
        rc, first, found, nf = first_stream(wire, cw, mode, text, offs, st["first"], pos, hot_n, kernel)
        assert rc == 0
        rc, tv = hist_stream(wire, cw, mode, "value", text, offs, st["value"], hv, hot_n, kernel)
        assert rc == 0
        rc, to = hist_stream(wire, cw, mode, "output", text, offs, st["output"], ho, hot_n, kernel)
        assert rc == 0 and tv == to == total
        rc, m, oo, _ = EM.scan_stream(wire, mode, text, offs, st["matches"], starts)
        assert rc == 0
        for i in range(n):
            mi = ref[i]
            want = mi[(mi[:, 1] > starts[i]) & (mi[:, 1] <= ends[i])]
            assert int(counts[i]) == len(want), (r, i)
            assert int(oo[i + 1] - oo[i]) == len(want), (r, i)
            assert bool(found[i]) == (len(want) > 0), (r, i)
            if len(want):
                w = want[0].copy()
                if pos is None:
                    w[:2] -= starts[i]
                assert tuple(first[i]) == tuple(w), (r, i)
            else:
                assert tuple(first[i]) == NONE, (r, i)
        assert total == int(counts.sum()) and nf == int(found.sum())
        got_total += total
        for k in ("first", "value", "output", "matches"):
            assert np.array_equal(st[k], st["count"]), (r, k)
    allm = np.concatenate(ref) if n else np.zeros((0, 3), np.uint32)
    assert got_total == len(allm)
    assert np.array_equal(hv, np.bincount(allm[:, 2].astype(np.int64), minlength=len(hv)).astype(np.uint64))
    rec_vals = E.image_outputs(wire, cw)[:, 0]
    assert np.array_equal(np.bincount(rec_vals.astype(np.int64), weights=ho.astype(np.float64), minlength=len(hv)).astype(np.uint64), hv)
    return st["count"]


def _hist_sizes(wire, cw):
    vals = E.image_outputs(wire, cw)[:, 0]
    return {"value": int(vals.max()) + 1 if len(vals) else 0, "output": len(vals)}


@pytest.mark.parametrize("mode", [FIND, OVERLAPPING])
@pytest.mark.parametrize("hot_n,kernel", [(0, 3), (4096, 3), (0, 1), (256, 4)])
def test_bytewise_streams_equal_the_stepper(mode, hot_n, kernel):
    pats, streams, cuts = bytewise_streams(0)
    opma = O.OraclePma.build(pats)
    wire = opma.serialize()
    EM.lib().emu_stream_config(3, hot_n)
    try:
        state = run_case(wire, False, mode, streams, cuts, opma, _hist_sizes(wire, False), hot_n, kernel, seed=11 + mode)
    finally:
        EM.lib().emu_stream_config(3, 4096)
    for i, s in enumerate(streams):
        assert int(state[i]) == opma.state_after(s, find_mode=(mode == FIND)), i


@pytest.mark.parametrize("mode", [FIND, OVERLAPPING])
def test_bytewise_streams_without_a_hot_region(mode):
    """The image laid out without a hot region: state ids need no translation at the boundary."""
    pats, streams, cuts = bytewise_streams(1)
    opma = O.OraclePma.build(pats)
    wire = opma.serialize()
    lib().emu_stream_rk_set_hot_slots(0)
    EM.lib().emu_set_hot_slots(0)
    try:
        state = run_case(wire, False, mode, streams, cuts, opma, _hist_sizes(wire, False), seed=21 + mode)
    finally:
        lib().emu_stream_rk_set_hot_slots(65536)
        EM.lib().emu_set_hot_slots(65536)
    for i, s in enumerate(streams):
        assert int(state[i]) == opma.state_after(s, find_mode=(mode == FIND)), i


def test_empty_pattern_under_find_overlapping():
    pats, streams, cuts = bytewise_streams(2, empty_pattern=True)
    opma = O.OraclePma.build(pats)
    wire = opma.serialize()
    state = run_case(wire, False, OVERLAPPING, streams, cuts, opma, _hist_sizes(wire, False), seed=31)
    for i, s in enumerate(streams):
        assert int(state[i]) == opma.state_after(s), i


@pytest.mark.parametrize("mode", [FIND, OVERLAPPING])
def test_charwise_streams_equal_the_stepper(mode):
    pats, streams, cuts = charwise_streams(mode)
    opma = O.OraclePma.build(pats, charwise=True)
    wire = opma.serialize()
    EM.lib().emu_stream_charwise(1)
    try:
        run_case(wire, True, mode, streams, cuts, opma, _hist_sizes(wire, True), seed=41 + mode)
    finally:
        EM.lib().emu_stream_charwise(0)


def test_refusals_leave_the_state_alone():
    """No Standard lane machine, or a mode the steppers do not have: DACH_INVALID_ARGUMENT, the state untouched."""
    pats, streams, _ = bytewise_streams(3, empty_pattern=True)
    text = np.frombuffer(b"".join(streams[:5]), dtype=np.uint8).copy()
    offs = np.zeros(6, dtype=np.uint64)
    offs[1:] = np.cumsum([len(s) for s in streams[:5]])
    cases = [(O.OraclePma.build(pats).serialize(), FIND, 3),            # find with an empty pattern
             (O.OraclePma.build(pats[1:]).serialize(), FIND, 0),        # kernel = 0
             (O.OraclePma.build(pats[1:]).serialize(), 2, 3)]           # find_overlapping_no_suffix has no stepper
    for wire, mode, kernel in cases:
        state = np.arange(5, dtype=np.uint32) + 1
        assert count_stream(wire, False, mode, text, offs, state, kernel=kernel)[0] == 1
        assert first_stream(wire, False, mode, text, offs, state, kernel=kernel)[0] == 1
        out = np.full(_hist_sizes(wire, False)["value"], 9, dtype=np.uint64)
        assert hist_stream(wire, False, mode, "value", text, offs, state, out, kernel=kernel)[0] == 1
        assert np.array_equal(state, np.arange(5, dtype=np.uint32) + 1) and (out == 9).all()
