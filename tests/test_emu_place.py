"""The ordered event placement from block descriptors and two-entry output lists, on the CPU restatement in
tests/emu: the pairs table against the chain walk of the outputs for every output record (C2 and C3 automata,
lists of three, 255 and more, ROOT's empty pattern), and the placement against the oracle -- golden vectors, random
batches with forced segments, long lists, a pad of 0 to 3 words before the output, 1 to 8 blocks per warp, and the
pool / out_cap overflow protocol."""
import json
import os

import numpy as np
import pytest

import emu_events_api as Q
from emu_api import lib
import oracle_api as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "search_tests.json"), encoding="utf-8"))
MODE = {"find_iter": 0, "find_overlapping_iter": 1, "find_overlapping_no_suffix_iter": 2}
ORC_MODE = {0: O.FIND, 1: O.FIND_OVERLAPPING, 2: O.FIND_OVERLAPPING_NO_SUFFIX}
CLASS_SHIFT = 30


def tables(wire):
    """(outputs, pairs) of the device image, (n, 4) uint32 each"""
    w = np.frombuffer(wire, dtype=np.uint8)
    n = lib().emu_place_tables(w.ctypes.data, w.size, None, None, 0)
    assert n >= 0, n
    outs = np.zeros((max(n, 1), 4), dtype=np.uint32)
    pairs = np.zeros((max(n, 1), 4), dtype=np.uint32)
    assert lib().emu_place_tables(w.ctypes.data, w.size, outs.ctypes.data, pairs.ctypes.data, n) == n
    return outs[:n], pairs[:n]


def check_pairs(wire):
    outs, pairs = tables(wire)
    for i in range(len(outs)):
        chain = []
        r = i + 1
        while r != 0:
            chain.append((int(outs[r - 1, 0]), int(outs[r - 1, 1])))
            r = int(outs[r - 1, 2])
        assert int(outs[i, 3]) == len(chain)
        want_cls = min(len(chain), 3)
        parent = chain[1] if len(chain) > 1 else (0, 0)
        got = pairs[i]
        assert (int(got[0]), int(got[1])) == chain[0], i
        assert (int(got[2]), int(got[3]) & ((1 << CLASS_SHIFT) - 1)) == parent, i
        assert int(got[3]) >> CLASS_SHIFT == want_cls, i
    return outs, pairs


def scan(wire, mode, text, offs, u=4, pad=0, seg_len=0, seg_from=0, pool_blocks=None, out_cap=None):
    """(rc, matches, out_offs, needed, blocks_used), growing out_cap and the pool until the batch fits unless given"""
    return Q.scan(wire, mode, text, offs, 0, seg_len, seg_from, pool_blocks, out_cap, direct=True, place_u=u, place_pad=pad)


def batch(hays):
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    return np.frombuffer(b"".join(hays), dtype=np.uint8), offs


def _long_lists():
    pats = [b"a" * k for k in range(1, 301)] + [b"ba", b"b"]
    text, offs = batch([b"a" * 400, b"xa" + b"a" * 260 + b"b" + b"a" * 300, b"", b"ba" * 40, b"a" * 254, b"a" * 255,
                        b"b", b"ab"] + [b"a" * k for k in range(1, 64)])
    return O.OraclePma.build(pats), text, offs


@pytest.mark.parametrize("name", ["C2", "C3"])
def test_pairs_equal_the_chain_walk_on_the_bench_automata(name):
    from daachorse_b200 import synth as S

    ps = S.make_patterns(S.config(name))
    wire = O.OraclePma.build_packed(ps.blob, ps.offs).serialize()
    outs, pairs = tables(wire)
    # vectorised form of check_pairs (the C3 image has hundreds of thousands of records)
    chain = outs[:, 3].astype(np.int64)
    par = outs[:, 2].astype(np.int64)
    has = par > 0
    assert np.array_equal(pairs[:, 0], outs[:, 0]) and np.array_equal(pairs[:, 1], outs[:, 1])
    assert np.array_equal(pairs[:, 3] >> CLASS_SHIFT, np.minimum(chain, 3).astype(np.uint32))
    assert np.array_equal(chain[has], chain[par[has] - 1] + 1) and (chain[~has] == 1).all()
    assert np.array_equal(pairs[has, 2], outs[par[has] - 1, 0])
    assert np.array_equal(pairs[has, 3] & ((1 << CLASS_SHIFT) - 1), outs[par[has] - 1, 1])
    assert (pairs[~has, 2] == 0).all() and (pairs[~has, 3] == 1 << CLASS_SHIFT).all()


def test_pairs_of_long_lists_and_the_empty_pattern():
    pma, _, _ = _long_lists()
    _, pairs = check_pairs(pma.serialize())
    assert set((pairs[:, 3] >> CLASS_SHIFT).tolist()) == {1, 2, 3}
    _, pairs = check_pairs(O.OraclePma.build([b"", b"a", b"ab", b"b", b"bab"]).serialize())
    _, pairs = check_pairs(O.OraclePma.build([b""]).serialize())


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
    check_pairs(wire)
    hay = t["haystack"].encode()
    for u, pad in ((1, 0), (4, 3)):
        rc, m, oo, need, _ = scan(wire, MODE[iterator], np.frombuffer(hay, dtype=np.uint8),
                                  np.array([0, len(hay)], dtype=np.uint64), u=u, pad=pad)
        if rc == Q.NOT_STD3:
            return
        assert rc == 0
        assert [(int(a), int(b), int(c)) for a, b, c in zip(m["start"], m["end"], m["value"])] == \
            [(s, e, v) for v, s, e in t["matches"]]


@pytest.mark.parametrize("seed", range(6))
def test_random_batches_every_word_offset(seed):
    rng = np.random.default_rng(9700 + seed)
    alpha = int(rng.integers(2, 5))
    pats = [bytes(rng.integers(97, 97 + alpha, size=int(rng.integers(0 if seed % 3 == 0 else 1, 10))).tolist())
            for _ in range(int(rng.integers(1, 60)))]
    pma = O.OraclePma.build(pats)
    wire = pma.serialize()
    lens = list(rng.integers(0, 400, size=40)) + [0, 64, 128, 1, 63, 65]
    text, offs = batch([bytes(rng.integers(97, 97 + alpha + 1, size=int(L)).tolist()) for L in lens])
    for mode in (0, 1, 2):
        ref = pma.scan_batch(ORC_MODE[mode], text, offs, want_matches=True)
        for u in (1, 2, 4, 8):
            for pad in range(4):
                for seg_len in (0, 16):
                    rc, m, oo, need, _ = scan(wire, mode, text, offs, u=u, pad=pad, seg_len=seg_len)
                    if rc == Q.NOT_STD3:
                        assert mode == 0 and b"" in pats
                        continue
                    assert rc == 0 and need == ref["total"], (mode, u, pad, seg_len)
                    assert m.tobytes() == ref["matches"].tobytes(), (mode, u, pad, seg_len)
                    assert np.array_equal(np.diff(oo.astype(np.int64)), ref["counts"].astype(np.int64))


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_long_lists_and_overflow(mode):
    """Runs longer than the staging buffer are written directly; a pool or out_cap overflow places nothing and keeps
    the count exact."""
    pma, text, offs = _long_lists()
    wire = pma.serialize()
    ref = pma.scan_batch(ORC_MODE[mode], text, offs, want_matches=True)
    for pad in range(4):
        rc, m, oo, need, _ = scan(wire, mode, text, offs, pad=pad, out_cap=ref["total"])
        assert rc == 0 and need == ref["total"] and m.tobytes() == ref["matches"].tobytes(), pad
    for pool_blocks in (0, 1, 5):
        rc, _, _, need, _ = scan(wire, mode, text, offs, pool_blocks=pool_blocks, out_cap=ref["total"])
        assert rc == 6 and need == ref["total"]
    rc, _, _, need, _ = scan(wire, mode, text, offs, out_cap=ref["total"] - 1)
    assert rc == 6 and need == ref["total"]
