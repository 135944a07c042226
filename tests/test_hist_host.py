"""Per-pattern histograms without a GPU: the entry points fail loudly, the output records are readable, and the
parity helper of tools/bench_reduce.py --output hist."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import daachorse_b200 as D
from daachorse_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench_reduce as bench  # noqa: E402


def test_hist_without_gpu_fails_loudly():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    p = D.DoubleArrayAhoCorasick.new(["a"])
    text = np.frombuffer(b"aa", dtype=np.uint8)
    offs = np.array([0, 2], dtype=np.uint64)
    for f in (lambda: p.pattern_counts_host(D.FIND, text, offs), lambda: p.value_counts_batch(["a"])):
        with pytest.raises(D.DaachorseError) as e:
            f()
        assert e.value.code == _lib.CUDA_ERROR
    L = _lib.load()
    tot = C.c_uint64()
    assert L.dach_dev_hist_batch(None, 0, 1, None, None, 0, 0, None, 0, C.byref(tot), None) == _lib.INVALID_ARGUMENT
    assert L.dach_hist_batch_host(None, 0, 1, None, None, 0, None, 0, C.byref(tot)) == _lib.INVALID_ARGUMENT


def test_output_records():
    p = D.DoubleArrayAhoCorasick.with_values([("ab", 7), ("b", 3), ("ab", 7)])
    v, ln, par = p.outputs()
    assert len(v) == 3 and sorted(v.tolist()) == [3, 7, 7] and sorted(ln.tolist()) == [1, 2, 2]
    assert all(0 <= int(x) <= 3 for x in par)
    for i, q in enumerate(par):  # a parent comes before its child
        assert q == 0 or q - 1 < i
    L = _lib.load()
    assert L.dach_pma_num_outputs(p._h) == 3
    assert L.dach_pma_outputs(p._h, None, None, None, 2) == _lib.INVALID_ARGUMENT
    assert L.dach_pma_outputs(p._h, None, None, None, 3) == _lib.OK
    assert L.dach_pma_outputs(None, None, None, None, 3) == _lib.INVALID_ARGUMENT
    lf = D.DoubleArrayAhoCorasickBuilder.new().match_kind(D.MatchKind.LeftmostFirst).build(["ab", "abc"])
    assert len(lf.outputs()[0]) == 1


def test_bench_hist_parity_helper():
    vals = np.array([0, 2, 2, 5], dtype=np.uint32)
    got = np.bincount(vals, minlength=7).astype(np.uint64)
    p = bench.hist_parity(got, vals, 7)
    assert p == {"hist_equal": True, "total_equal": True}
    got[1] += 1
    assert not bench.hist_parity(got, vals, 7)["hist_equal"]
    assert not bench.hist_parity(got, vals, 7)["total_equal"]
