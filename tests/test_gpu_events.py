"""Event blocks of StdMachine3's matches path on the device: the scan stores (end, slot | list length) events and
k_expand places them.  Compared with the lane-per-haystack kernel (kernel 0, tuple blocks and k_gather) and the
oracle.  Segments, stream chunks, jobs on two streams and shard groups run this path in test_gpu_parity.py."""
import ctypes as C

import numpy as np
import pytest

import daachorse_b200 as D
import oracle_api as O
from daachorse_b200 import _lib
from daachorse_b200 import synth as S

pytestmark = pytest.mark.gpu
ORC = {D.FIND: O.FIND, D.FIND_OVERLAPPING: O.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX: O.FIND_OVERLAPPING_NO_SUFFIX}


def _long_lists():
    """`a` x k for k = 1..300: past the 254th `a` of a run every event's list is too long for the length byte."""
    pats = [b"a" * k for k in range(1, 301)] + [b"ba"]
    hays = [b"a" * 400, b"xa" + b"a" * 260 + b"b" + b"a" * 300, b"", b"ba" * 40, b"a" * 254, b"a" * 255] * 40
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    return pats, np.frombuffer(b"".join(hays), dtype=np.uint8), offs


def _scan_all(pma, mode, text, offs, options):
    pma.set_option("kernel", 3)
    for k, v in options:
        pma.set_option(k, v)
    r = pma.scan_batch_host(mode, text, offs)
    for k, _ in options:
        pma.set_option(k, {"seg_len": 0, "gather_ordered": 1, "hot_entries": 6144}[k])
    return r


@pytest.mark.parametrize("mode", [D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX])
def test_long_lists_take_the_escape(mode):
    pats, text, offs = _long_lists()
    pma = D.DoubleArrayAhoCorasick.new(pats)
    ref = O.OraclePma.build(pats).scan_batch(ORC[mode], text, offs, want_matches=True)
    pma.set_option("kernel", 0)
    k0 = pma.scan_batch_host(mode, text, offs)
    assert k0.matches.tobytes() == ref["matches"].tobytes()
    for options in ([], [("seg_len", 64)], [("seg_len", 512)], [("gather_ordered", 2)], [("hot_entries", 0)]):
        r = _scan_all(pma, mode, text, offs, options)
        assert r.matches.tobytes() == k0.matches.tobytes(), options
        assert np.array_equal(r.offsets, k0.offsets), options


@pytest.mark.parametrize("seed", range(3))
def test_seeded_c3_batches_equal_kernel_0(seed):
    cfg = S.config("C3")
    ps = S.make_patterns(cfg, n=20000)
    pool, b = S.make_pool(cfg, ps, 8 << 20, seed=seed)
    starts = S.window_starts(b, len(pool), 3000, 4096, seed=seed + 1)
    text, offs = S.materialise_host(pool, starts, 4096)
    pma = D.DoubleArrayAhoCorasick.new(ps.as_list())
    for mode in (D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX):
        pma.set_option("kernel", 0)
        k0 = pma.scan_batch_host(mode, text, offs)
        for options in ([], [("gather_ordered", 2)], [("seg_len", 256), ("gather_ordered", 2)]):
            r = _scan_all(pma, mode, text, offs, options)
            assert r.matches.tobytes() == k0.matches.tobytes(), (mode, options)
            assert np.array_equal(r.offsets, k0.offsets), (mode, options)


def test_needed_is_exact_on_overflow_with_long_lists():
    pats, text, offs = _long_lists()
    pma = D.DoubleArrayAhoCorasick.new(pats)
    total = O.OraclePma.build(pats).scan_batch(O.FIND_OVERLAPPING, text, offs)["total"]
    L = _lib.load()
    d = pma.device_handle()
    n = len(offs) - 1
    out = np.zeros(total, dtype=D.MATCH_DTYPE)
    oo = np.zeros(n + 1, dtype=np.uint64)
    need = C.c_uint64()
    for cap in (0, 10, total - 1):
        rc = L.dach_scan_batch_host(d, D.FIND_OVERLAPPING, text.ctypes.data, offs.ctypes.data, n, out.ctypes.data, cap,
                                    oo.ctypes.data, C.byref(need))
        assert rc == _lib.OUTPUT_OVERFLOW and need.value == total, cap
    rc = L.dach_scan_batch_host(d, D.FIND_OVERLAPPING, text.ctypes.data, offs.ctypes.data, n, out.ctypes.data, total,
                                oo.ctypes.data, C.byref(need))
    assert rc == 0 and need.value == total
