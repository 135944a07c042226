"""Per-pattern document frequencies without a GPU: the entry points fail loudly, bad keys and short arrays are refused
before any device work, and the Python wrappers check their arguments."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import daachorse_b200 as D
from daachorse_b200 import _lib


def _no_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")


def test_df_without_gpu_fails_loudly():
    _no_gpu()
    p = D.DoubleArrayAhoCorasick.new(["a"])
    text = np.frombuffer(b"aa", dtype=np.uint8)
    offs = np.array([0, 2], dtype=np.uint64)
    for f in (lambda: p.doc_counts_host(D.FIND, text, offs), lambda: p.value_doc_counts_batch(["a"]),
              lambda: p.last_doc_windows()):
        with pytest.raises(D.DaachorseError) as e:
            f()
        assert e.value.code == _lib.CUDA_ERROR


def test_null_handles_bad_keys_and_short_arrays():
    L = _lib.load()
    tot = C.c_uint64()
    assert L.dach_dev_df_batch(None, 0, 1, None, None, 0, 0, None, 0, C.byref(tot), None) == _lib.INVALID_ARGUMENT
    assert L.dach_df_batch_host(None, 0, 1, None, None, 0, None, 0, C.byref(tot)) == _lib.INVALID_ARGUMENT
    assert L.dach_dev_last_df_windows(None, None, None) == _lib.INVALID_ARGUMENT


def test_wrappers_check_arguments():
    p = D.DoubleArrayAhoCorasick.with_values([("a", 3), ("ab", 9)])
    text = np.frombuffer(b"aab", dtype=np.uint8)
    offs = np.array([0, 3], dtype=np.uint64)
    with pytest.raises(D.DaachorseError) as e:
        p.doc_counts_host(D.FIND, text, offs, key="pattern")
    assert e.value.code == _lib.INVALID_ARGUMENT
    for out in (np.zeros(10, np.int64), np.zeros((2, 5), np.uint64), np.zeros(20, np.uint64)[::2]):
        with pytest.raises(D.DaachorseError) as e:
            p.doc_counts_host(D.FIND, text, offs, out=out)
        assert e.value.code == _lib.INVALID_ARGUMENT
    with pytest.raises(D.DaachorseError) as e:
        p.doc_counts_host(D.FIND, text, np.array([0, 4], dtype=np.uint64))  # past the text
    assert e.value.code == _lib.INVALID_ARGUMENT
    with pytest.raises(AssertionError):
        p.doc_counts_host(D.LEFTMOST_FIND, text, offs)


def test_bench_df_parity_helper():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import bench_reduce as bench

    counts = np.array([3, 0, 2], dtype=np.uint64)  # haystack 0: values 0, 2, 2; haystack 2: values 2, 5
    vals = np.array([0, 2, 2, 2, 5], dtype=np.uint32)
    got = np.array([1, 0, 2, 0, 0, 1, 0], dtype=np.uint64)
    assert bench.df_parity(got, counts, vals, 7) == {"df_equal": True, "total_equal": True}
    got[2] += 1
    p = bench.df_parity(got, counts, vals, 7)
    assert not p["df_equal"] and not p["total_equal"]
