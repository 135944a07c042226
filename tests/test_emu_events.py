"""StdMachine3's matches path with event blocks, on the CPU emulation in tests/emu_events: the drain stores
(end, slot | list length) events, blocks are handed out per warp, placement (k_expand) expands them.  Checked
against the oracle on the golden vectors, random batches, segments and stream chunks, and on what only this path
has: output lists of 255 and more (the length byte's escape), warm-up events that must not be stored, and the pool /
out_cap overflow protocol with event blocks."""
import json
import os

import numpy as np
import pytest

import emu_events_api as E
import oracle_api as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "search_tests.json"), encoding="utf-8"))
MODE = {"find_iter": 0, "find_overlapping_iter": 1, "find_overlapping_no_suffix_iter": 2}
ORC_MODE = {0: O.FIND, 1: O.FIND_OVERLAPPING, 2: O.FIND_OVERLAPPING_NO_SUFFIX}
HOT = (0, 256, 1 << 16)


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
        rc, m, oo, need, _ = E.scan(wire, MODE[iterator], np.frombuffer(hay, dtype=np.uint8),
                                    np.array([0, len(hay)], dtype=np.uint64), hot_n=hot)
        if rc == E.NOT_STD3:  # find with an empty pattern, or a ROOT without children: the simple kernel
            return
        assert rc == 0
        assert triples(m) == [(s, e, v) for v, s, e in t["matches"]]


@pytest.mark.parametrize("seed", range(8))
def test_random_batches_and_segments(seed):
    rng = np.random.default_rng(7100 + seed)
    alpha = int(rng.integers(2, 5))
    pats = rand_patterns(rng, int(rng.integers(1, 60)), alpha, 9, allow_empty=(seed == 0))
    pma = O.OraclePma.build(pats)
    wire = pma.serialize()
    lens = list(rng.integers(0, 400, size=40)) + [0, 64, 128, 1, 63, 65]
    text, offs = batch([bytes(rng.integers(97, 97 + alpha + 1, size=int(L)).tolist()) for L in lens])
    for mode in (0, 1, 2):
        ref = pma.scan_batch(ORC_MODE[mode], text, offs, want_matches=True)
        for hot in HOT:
            for seg_len, seg_from in ((0, 0), (1, 0), (16, 0), (64, 11), (100, 0)):
                rc, m, oo, need, _ = E.scan(wire, mode, text, offs, hot_n=hot, seg_len=seg_len, seg_from=seg_from)
                if rc == E.NOT_STD3:
                    assert mode == 0 and b"" in pats
                    continue
                assert rc == 0 and need == ref["total"], (mode, hot, seg_len)
                assert m.tobytes() == ref["matches"].tobytes(), (mode, hot, seg_len)
                assert np.array_equal(np.diff(oo.astype(np.int64)), ref["counts"].astype(np.int64))


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("mode", [0, 1])
def test_stream_chunks_equal_the_stepper_over_the_whole_stream(seed, mode):
    """Streams cut into ragged chunks (empty ones included), scanned round by round with the state carried over and
    positions rebased (k_add_base), report what the crate's stepper reports over the whole stream."""
    rng = np.random.default_rng(7300 + seed)
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
        rc, m, oo, need, _ = E.scan(wire, mode, text, offs, hot_n=256 if seed % 2 else 0, state=state, pos=pos)
        assert rc == 0
        tr = triples(m)
        for i in range(len(streams)):
            got[i] += tr[int(oo[i]): int(oo[i + 1])]
            pos[i] += len(chunks[i])
    assert got == want
    for i, s in enumerate(streams):
        assert int(state[i]) == pma.state_after(s, find_mode=(mode == 0))


def _long_lists():
    """`a` x k for k = 1..300: the state after k `a`s has a list of k patterns, so every event past the 254th
    byte of a run of `a` takes the escape (its length is read from the head record's chain word)."""
    pats = [b"a" * k for k in range(1, 301)] + [b"ba"]
    text, offs = batch([b"a" * 400, b"xa" + b"a" * 260 + b"b" + b"a" * 300, b"", b"ba" * 40, b"a" * 254, b"a" * 255])
    return O.OraclePma.build(pats), text, offs


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_lists_of_255_and_more_take_the_escape(mode):
    pma, text, offs = _long_lists()
    wire = pma.serialize()
    ref = pma.scan_batch(ORC_MODE[mode], text, offs, want_matches=True)
    for hot in HOT:
        for seg_len in (0, 64, 300):
            rc, m, oo, need, _ = E.scan(wire, mode, text, offs, hot_n=hot, seg_len=seg_len, out_cap=ref["total"])
            assert rc == 0 and need == ref["total"], (hot, seg_len)
            assert m.tobytes() == ref["matches"].tobytes(), (hot, seg_len)
            assert np.array_equal(np.diff(oo.astype(np.int64)), ref["counts"].astype(np.int64))


def test_warm_up_events_are_not_stored():
    """Patterns `a` and `aaaa` on a run of `a`: every byte is one event, and a 30-byte segment has exactly 30
    events ending inside it after the 3 of its warm-up, so it fills exactly one event block.  A warm-up event stored
    by mistake would need a second block and overflow a pool of one block per segment."""
    pma = O.OraclePma.build([b"a", b"aaaa"])
    wire = pma.serialize()
    n_seg = 40
    text = np.frombuffer(b"a" * (30 * n_seg), dtype=np.uint8)
    offs = np.array([0, text.size], dtype=np.uint64)
    ref = pma.scan_batch(O.FIND_OVERLAPPING, text, offs, want_matches=True)
    rc, m, oo, need, used = E.scan(wire, 1, text, offs, seg_len=30, pool_blocks=n_seg, out_cap=ref["total"])
    assert rc == 0 and used == n_seg and m.tobytes() == ref["matches"].tobytes()
    rc, m, oo, need, _ = E.scan(wire, 1, text, offs, seg_len=30, pool_blocks=n_seg - 1, out_cap=ref["total"])
    assert rc == 6 and need == ref["total"]


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_needed_stays_exact_when_the_pool_or_out_cap_overflows(mode):
    """Blocks span many service phases (one haystack has hundreds of events, a lane stores at most 10 per
    phase); whatever runs out, the count goes on and `needed` is the exact total."""
    pma, text, offs = _long_lists()
    wire = pma.serialize()
    total = pma.scan_batch(ORC_MODE[mode], text, offs)["total"]
    for pool_blocks in (0, 1, 2, 5, 17):
        rc, m, oo, need, _ = E.scan(wire, mode, text, offs, pool_blocks=pool_blocks, out_cap=total)
        assert rc == 6 and need == total, pool_blocks
    rc, m, oo, need, _ = E.scan(wire, mode, text, offs, out_cap=total - 1)
    assert rc == 6 and need == total
    rc, m, oo, need, used = E.scan(wire, mode, text, offs, out_cap=total)
    assert rc == 0 and len(m) == total and used > 17
