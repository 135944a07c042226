"""Masked text without a GPU: argument refusals come before any device work, the entry points fail loudly, and the
reference the mask tests compare against agrees with the per-byte definition."""
import ctypes as C

import numpy as np
import pytest

import daachorse_b200 as D
import emu_mask_api as M
from daachorse_b200 import _lib


def _no_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")


def test_mask_without_gpu_fails_loudly():
    _no_gpu()
    p = D.DoubleArrayAhoCorasick.new(["a"])
    text = np.frombuffer(b"aa", dtype=np.uint8)
    offs = np.array([0, 2], dtype=np.uint64)
    for f in (lambda: p.mask_batch_host(D.FIND, text, offs), lambda: p.mask_batch(["a"])):
        with pytest.raises(D.DaachorseError) as e:
            f()
        assert e.value.code == _lib.CUDA_ERROR
    L = _lib.load()
    assert L.dach_dev_mask_batch(None, 0, None, None, 0, 0, 42, None, None) == _lib.INVALID_ARGUMENT
    assert L.dach_mask_batch_host(None, 0, None, None, 0, 42, None) == _lib.INVALID_ARGUMENT


def test_argument_refusals_come_before_device_work():
    """Every one of these is INVALID_ARGUMENT (not the CUDA_ERROR the first device call would raise here)."""
    import torch

    p = D.DoubleArrayAhoCorasick.new(["a"])
    cw = D.CharwiseDoubleArrayAhoCorasick.new(["a"])
    text = np.frombuffer(b"abab", dtype=np.uint8).copy()
    offs = np.array([0, 4], dtype=np.uint64)
    bad = [
        lambda: p.mask_batch_host(D.FIND, text, offs, out=text),  # in place
        lambda: p.mask_batch_host(D.FIND, text, offs, out=text[1:].copy()),  # too small
        lambda: p.mask_batch_host(D.FIND, text, offs, out=np.zeros(4, dtype=np.int32)),
        lambda: p.mask_batch_host(D.FIND, text, offs, out=np.zeros((2, 2), dtype=np.uint8)),
        lambda: p.mask_batch_host(D.FIND, text, offs, fill=256),
        lambda: p.mask_batch_host(D.FIND, text, offs, fill=-1),
        lambda: p.mask_batch_host(D.FIND, text, offs, fill=b"**"),
        lambda: p.mask_batch_host(D.FIND, text, np.array([0, 9], dtype=np.uint64)),
        lambda: cw.mask_batch_host(D.FIND, text, offs, fill=0x80),
        lambda: cw.mask_batch(["a"], fill="é"),
        lambda: p.mask_batch(["a"], fill=True),
        lambda: p.mask_batch_device(D.FIND, torch.zeros(4, dtype=torch.uint8), torch.zeros(2, dtype=torch.int64), fill=300),
        lambda: cw.mask_batch_device(D.FIND, torch.zeros(4, dtype=torch.uint8), torch.zeros(2, dtype=torch.int64), fill=0xFF),
    ]
    for i, f in enumerate(bad):
        with pytest.raises(D.DaachorseError) as e:
            f()
        assert e.value.code == _lib.INVALID_ARGUMENT, i
    with pytest.raises(AssertionError):
        p.mask_batch_host(D.LEFTMOST_FIND, text, offs)  # the crate asserts on the match kind


def test_offsets_past_the_text_are_refused_with_no_haystack():
    """n = 0 still copies text[0, offs[0]): an offs[0] past the text is refused before the call reads or writes it."""
    p = D.DoubleArrayAhoCorasick.new(["a"])
    text = np.zeros(4, dtype=np.uint8)
    out = np.full(8, 7, dtype=np.uint8)
    for offs, kw in (([100], {}), ([5], {"out": out}), ([0, 2, 5], {"out": out})):
        with pytest.raises(D.DaachorseError) as e:
            p.mask_batch_host(D.FIND, text, np.array(offs, dtype=np.uint64), **kw)
        assert e.value.code == _lib.INVALID_ARGUMENT, offs
    assert (out == 7).all()


def _brute(text, offs, spans, fill):
    out = bytearray(text.tobytes())
    for j in range(len(out)):
        for h, s, e in spans:
            if int(offs[h]) + s <= j < int(offs[h]) + e:
                out[j] = fill
                break
    return np.frombuffer(bytes(out), dtype=np.uint8)


@pytest.mark.parametrize("seed", range(20))
def test_expected_mask_is_the_per_byte_definition(seed):
    rng = np.random.default_rng(400 + seed)
    lens = rng.integers(0, 30, size=int(rng.integers(0, 6)))
    lead, tail = int(rng.integers(0, 4)), int(rng.integers(0, 4))
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64) + np.uint64(lead)
    text = rng.integers(0, 256, size=int(offs[-1]) + tail).astype(np.uint8)
    spans = []
    for h, n in enumerate(lens):
        for _ in range(int(rng.integers(0, 5))):
            e = int(rng.integers(0, n + 1))
            spans.append((h, int(rng.integers(0, e + 1)), e))  # zero-length ones included
    fill = int(rng.integers(0, 256))
    got = M.expected_mask(text, offs, [s for _, s, _ in spans], [e for _, _, e in spans], [h for h, _, _ in spans], fill)
    assert np.array_equal(got, _brute(text, offs, spans, fill))
