"""Counts and first matches without a GPU: the entry points fail loudly, and the parity helpers of
tools/bench_reduce.py."""
import os
import sys

import numpy as np
import pytest

import daachorse_b200 as D
from daachorse_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench_reduce as bench  # noqa: E402


def test_count_and_first_without_gpu_fail_loudly():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    p = D.DoubleArrayAhoCorasick.new(["a"])
    text = np.frombuffer(b"aa", dtype=np.uint8)
    offs = np.array([0, 2], dtype=np.uint64)
    for f in (lambda: p.count_batch_host(D.FIND, text, offs), lambda: p.first_batch_host(D.FIND, text, offs),
              lambda: p.is_match("a"), lambda: p.count_batch(["a"])):
        with pytest.raises(D.DaachorseError) as e:
            f()
        assert e.value.code == _lib.CUDA_ERROR
    L = _lib.load()
    import ctypes as C

    d = C.c_void_p()
    assert L.dach_dev_upload(p._h, 0, C.byref(d)) == _lib.CUDA_ERROR
    tot = C.c_uint64()
    assert L.dach_dev_count_batch(None, 0, None, None, 0, 0, None, C.byref(tot), None) == _lib.INVALID_ARGUMENT
    assert L.dach_dev_first_batch(None, 0, None, None, 0, 0, None, None, C.byref(tot), None) == _lib.INVALID_ARGUMENT


def test_bench_parity_helpers():
    m = np.array([(0, 1, 5), (0, 2, 6), (3, 4, 7)], dtype=D.MATCH_DTYPE)
    first, found = bench.first_from_matches(m, [2, 0, 1])
    assert found.tolist() == [True, False, True]
    assert first.tolist() == [[0, 1, 5], [0xFFFFFFFF] * 3, [3, 4, 7]]
    assert bench.reduce_parity("first", None, first, found, None, first[:2], found)["first_equal"]
    assert not bench.reduce_parity("first", None, first, ~found, None, first, found)["found_equal"]
    p = bench.reduce_parity("counts", np.array([2, 0, 1]), None, None, np.array([2, 0, 1], dtype=np.uint64), None, None)
    assert p == {"counts_equal": True, "total_equal": True}
    assert bench.first_end_frac(first, found, [4, 4, 8]) == pytest.approx((1 / 4 + 4 / 8) / 2)
    assert bench.first_end_frac(first, np.zeros(3, bool), [4, 4, 8]) is None
