"""StdMachine3's direct matches path on the CPU emulation in tests/emu_direct: a lane stores each event into its block
at the landing that makes it, or keeps it pending for the service phase (no block with room, or a list length of 255
or more); placement (k_expand) expands the blocks.  Checked against the oracle on the golden vectors, random batches,
forced segments, stream chunks, ROOT's empty pattern, long lists, the pool / out_cap overflow protocol and items that
end exactly on a block boundary; and against the queue path (tests/emu_events) for the number of blocks taken."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import emu_events_api as Q
import oracle_api as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "search_tests.json"), encoding="utf-8"))
EMU_DIR = os.path.join(HERE, "emu_direct")
MODE = {"find_iter": 0, "find_overlapping_iter": 1, "find_overlapping_no_suffix_iter": 2}
ORC_MODE = {0: O.FIND, 1: O.FIND_OVERLAPPING, 2: O.FIND_OVERLAPPING_NO_SUFFIX}
HOT = (0, 256, 1 << 16)
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", EMU_DIR, "-s"])
        L = C.CDLL(os.path.join(EMU_DIR, "libdach_emu_direct.so"))
        L.emu_direct_scan_wire.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32,
                                           C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                           C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
        L.emu_direct_scan_wire.restype = C.c_int
        _lib = L
    return _lib


def scan(wire, mode, text, offs, hot_n=0, seg_len=0, seg_from=0, pool_blocks=None, out_cap=None, state=None, pos=None):
    """emu_events_api.scan's contract on the direct path: (rc, matches, out_offs, needed, blocks_used)."""
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    text = np.ascontiguousarray(text, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.uint64)
    n = len(offs) - 1
    cap = int(out_cap) if out_cap is not None else 1 << 12
    pad = text if text.size else np.zeros(16, dtype=np.uint8)
    while True:
        pb = int(pool_blocks) if pool_blocks is not None else cap // 30 + n + (text.size // seg_len + 1 if seg_len else 0) + 16
        saved = state.copy() if state is not None else None
        out = np.zeros(max(cap, 1), dtype=Q.MATCH_DTYPE)
        oo = np.zeros(n + 1, dtype=np.uint64)
        need, used = C.c_uint64(), C.c_uint32()
        rc = lib().emu_direct_scan_wire(wire_a.ctypes.data, wire_a.size, mode, pad.ctypes.data, offs.ctypes.data, n, hot_n,
                                        seg_len, seg_from, pb, state.ctypes.data if state is not None else None,
                                        pos.ctypes.data if pos is not None else None, out.ctypes.data, cap, oo.ctypes.data,
                                        C.byref(need), C.byref(used))
        if rc == 6 and out_cap is None and pool_blocks is None:
            if state is not None:
                state[:] = saved
            cap = max(cap * 2, int(need.value))
            continue
        return rc, out[: need.value] if rc == 0 else None, oo, int(need.value), int(used.value)


def triples(m):
    return [(int(a), int(b), int(c)) for a, b, c in zip(m["start"], m["end"], m["value"])]


def rand_patterns(rng, n, alpha, maxlen, allow_empty=False):
    return [bytes(rng.integers(97, 97 + alpha, size=int(rng.integers(0 if allow_empty else 1, maxlen + 1))).tolist())
            for _ in range(n)]


def batch(hays):
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    return np.frombuffer(b"".join(hays), dtype=np.uint8), offs


def _golden():
    for variant, iterator, coll, kind in GOLD["configs"]:
        if variant != "bytewise" or iterator not in MODE or kind != "Standard":
            continue
        for g in GOLD["collections"][coll]:
            for t in GOLD["groups"][g]:
                yield pytest.param(iterator, t, id="%s-%s" % (iterator, t["name"]))


@pytest.mark.parametrize("iterator,t", list(_golden()))
def test_golden_vectors(iterator, t):
    wire = O.OraclePma.build(t["patterns"]).serialize()
    hay = t["haystack"].encode()
    for hot in HOT:
        rc, m, oo, need, _ = scan(wire, MODE[iterator], np.frombuffer(hay, dtype=np.uint8),
                                  np.array([0, len(hay)], dtype=np.uint64), hot_n=hot)
        if rc == Q.NOT_STD3:  # find with an empty pattern, or a ROOT without children: the simple kernel
            return
        assert rc == 0
        assert triples(m) == [(s, e, v) for v, s, e in t["matches"]]


@pytest.mark.parametrize("seed", range(8))
def test_random_batches_and_segments(seed):
    """Forced segments included: their warm-up events must be dropped at the landing."""
    rng = np.random.default_rng(9100 + seed)
    alpha = int(rng.integers(2, 5))
    pats = rand_patterns(rng, int(rng.integers(1, 60)), alpha, 9, allow_empty=(seed % 4 == 0))
    pma = O.OraclePma.build(pats)
    wire = pma.serialize()
    lens = list(rng.integers(0, 400, size=40)) + [0, 64, 128, 1, 63, 65]
    text, offs = batch([bytes(rng.integers(97, 97 + alpha + 1, size=int(L)).tolist()) for L in lens])
    for mode in (0, 1, 2):
        ref = pma.scan_batch(ORC_MODE[mode], text, offs, want_matches=True)
        for hot in HOT:
            for seg_len, seg_from in ((0, 0), (1, 0), (16, 0), (64, 11), (100, 0)):
                rc, m, oo, need, used = scan(wire, mode, text, offs, hot_n=hot, seg_len=seg_len, seg_from=seg_from)
                if rc == Q.NOT_STD3:
                    assert mode == 0 and b"" in pats
                    continue
                assert rc == 0 and need == ref["total"], (mode, hot, seg_len)
                assert m.tobytes() == ref["matches"].tobytes(), (mode, hot, seg_len)
                assert np.array_equal(np.diff(oo.astype(np.int64)), ref["counts"].astype(np.int64))
                # the same blocks as the queue path: one per started BLK_EVENTS events of an item
                q = Q.scan(wire, mode, text, offs, hot_n=hot, seg_len=seg_len, seg_from=seg_from)
                assert q[0] == 0 and q[4] == used, (mode, hot, seg_len)


@pytest.mark.parametrize("mode", [1, 2])
def test_root_empty_pattern_is_the_first_event(mode):
    """ROOT's list at position 0 is the item's pending event when the item starts; every later visit to ROOT is an
    ordinary landing.  Empty haystacks report the empty pattern once; segments after the first do not."""
    pats = [b"", b"a", b"ab", b"b", b"bab"]
    pma = O.OraclePma.build(pats)
    wire = pma.serialize()
    text, offs = batch([b"", b"a", b"abxab", b"x" * 70, b"ab" * 50, b"", b"b"])
    ref = pma.scan_batch(ORC_MODE[mode], text, offs, want_matches=True)
    for hot in HOT:
        for seg_len in (0, 16):
            rc, m, oo, need, _ = scan(wire, mode, text, offs, hot_n=hot, seg_len=seg_len)
            assert rc == 0 and need == ref["total"], (hot, seg_len)
            assert m.tobytes() == ref["matches"].tobytes(), (hot, seg_len)


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("mode", [0, 1])
def test_stream_chunks_equal_the_stepper_over_the_whole_stream(seed, mode):
    rng = np.random.default_rng(9300 + seed)
    alpha = int(rng.integers(1, 5))
    pats = rand_patterns(rng, int(rng.integers(1, 60)), alpha, int(rng.integers(1, 10)))
    streams = [bytes(rng.integers(97, 97 + alpha + (seed % 2), size=int(rng.integers(0, 500))).tolist()) for _ in range(9)]
    pma = O.OraclePma.build(pats)
    wire = pma.serialize()
    orc_mode = O.FIND_STEPPER if mode == 0 else O.FIND_OVERLAPPING_STEPPER
    want = []
    for s in streams:
        ref = pma.scan_batch(orc_mode, np.frombuffer(s, dtype=np.uint8), np.array([0, len(s)], dtype=np.uint64),
                             want_matches=True)
        want.append([x for x in triples(ref["matches"]) if x[1] != 0])
    state = np.zeros(len(streams), dtype=np.uint32)
    pos = np.zeros(len(streams), dtype=np.uint32)
    got = [[] for _ in streams]
    while any(int(pos[i]) < len(s) for i, s in enumerate(streams)):
        chunks = [s[int(pos[i]): int(pos[i]) + int(rng.integers(0, 70))] for i, s in enumerate(streams)]
        text, offs = batch(chunks)
        rc, m, oo, need, _ = scan(wire, mode, text, offs, hot_n=256 if seed % 2 else 0, state=state, pos=pos)
        assert rc == 0
        tr = triples(m)
        for i in range(len(streams)):
            got[i] += tr[int(oo[i]): int(oo[i + 1])]
            pos[i] += len(chunks[i])
    assert got == want
    for i, s in enumerate(streams):
        assert int(state[i]) == pma.state_after(s, find_mode=(mode == 0))


def _long_lists():
    """`a` x k for k = 1..300: past the 254th `a` of a run every event's list is too long for the length byte, so
    every such event waits for the service phase, which reads the chain word."""
    pats = [b"a" * k for k in range(1, 301)] + [b"ba"]
    text, offs = batch([b"a" * 400, b"xa" + b"a" * 260 + b"b" + b"a" * 300, b"", b"ba" * 40, b"a" * 254, b"a" * 255])
    return O.OraclePma.build(pats), text, offs


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_lists_of_255_and_more_wait_for_the_service_phase(mode):
    pma, text, offs = _long_lists()
    wire = pma.serialize()
    ref = pma.scan_batch(ORC_MODE[mode], text, offs, want_matches=True)
    for hot in HOT:
        for seg_len in (0, 64, 300):
            rc, m, oo, need, _ = scan(wire, mode, text, offs, hot_n=hot, seg_len=seg_len, out_cap=ref["total"])
            assert rc == 0 and need == ref["total"], (hot, seg_len)
            assert m.tobytes() == ref["matches"].tobytes(), (hot, seg_len)
            assert np.array_equal(np.diff(oo.astype(np.int64)), ref["counts"].astype(np.int64))


def test_warm_up_events_are_dropped():
    """Patterns `a` and `aaaa` on a run of `a`: a 30-byte segment has exactly 30 events ending inside it after the 3
    of its warm-up, so it fills exactly one event block; a warm-up event stored by mistake would need a second."""
    pma = O.OraclePma.build([b"a", b"aaaa"])
    wire = pma.serialize()
    n_seg = 40
    text = np.frombuffer(b"a" * (30 * n_seg), dtype=np.uint8)
    offs = np.array([0, text.size], dtype=np.uint64)
    ref = pma.scan_batch(O.FIND_OVERLAPPING, text, offs, want_matches=True)
    rc, m, oo, need, used = scan(wire, 1, text, offs, seg_len=30, pool_blocks=n_seg, out_cap=ref["total"])
    assert rc == 0 and used == n_seg and m.tobytes() == ref["matches"].tobytes()
    rc, m, oo, need, _ = scan(wire, 1, text, offs, seg_len=30, pool_blocks=n_seg - 1, out_cap=ref["total"])
    assert rc == 6 and need == ref["total"]


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_needed_stays_exact_when_the_pool_or_out_cap_overflows(mode):
    """Once the pool is exhausted a lane's block is none: its events are counted at the landing and not stored."""
    pma, text, offs = _long_lists()
    wire = pma.serialize()
    total = pma.scan_batch(ORC_MODE[mode], text, offs)["total"]
    for pool_blocks in (0, 1, 2, 5, 17):
        rc, m, oo, need, _ = scan(wire, mode, text, offs, pool_blocks=pool_blocks, out_cap=total)
        assert rc == 6 and need == total, pool_blocks
    rc, m, oo, need, _ = scan(wire, mode, text, offs, out_cap=total - 1)
    assert rc == 6 and need == total
    rc, m, oo, need, used = scan(wire, mode, text, offs, out_cap=total)
    assert rc == 0 and len(m) == total and used > 17


@pytest.mark.parametrize("k", [29, 30, 31, 59, 60, 61, 90])
def test_items_that_end_on_a_block_boundary(k):
    """Pattern `a` on haystacks of k `a`s: k events each.  An item whose last event fills its block exactly takes no
    further block; one more event takes exactly one more."""
    pma = O.OraclePma.build([b"a"])
    wire = pma.serialize()
    n = 33  # more items than a warp has lanes
    text, offs = batch([b"a" * k] * n)
    per_item = (k + 29) // 30
    for mode in (0, 1, 2):
        ref = pma.scan_batch(ORC_MODE[mode], text, offs, want_matches=True)
        rc, m, oo, need, used = scan(wire, mode, text, offs, pool_blocks=n * per_item, out_cap=ref["total"])
        assert rc == 0 and used == n * per_item and m.tobytes() == ref["matches"].tobytes(), mode
        rc, m, oo, need, _ = scan(wire, mode, text, offs, pool_blocks=n * per_item - 1, out_cap=ref["total"])
        assert rc == 6 and need == ref["total"], mode
