"""Counts, first matches, histograms and masked text on jobs, without a GPU: the four entry points are exported and
refuse a null job, jobs cannot be made without a device, and the Job wrappers refuse what the ``*_device`` forms
refuse before anything reaches the library (the library is replaced by fakes that record every call)."""
import ctypes as C
import gc
import os
import re

import pytest

import daachorse_b200 as D
from daachorse_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JOB_RK = ("dach_job_count", "dach_job_first", "dach_job_hist", "dach_job_mask")


def test_job_reductions_are_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "daachorse_b200.h")).read()
    for name in JOB_RK:
        assert re.search(r"^int %s\(dach_job \*job," % name, hdr, re.M), name
        assert name in _lib.SYMBOLS
        assert hasattr(C.CDLL(_lib.LIB_PATH), name)


def test_null_job_is_refused():
    L = _lib.load()
    buf = (C.c_uint64 * 4)()
    p = C.cast(buf, C.c_void_p)
    assert L.dach_job_count(None, 0, p, p, 1, 8, p, None) == _lib.INVALID_ARGUMENT
    assert L.dach_job_first(None, 0, p, p, 1, 8, p, p, None) == _lib.INVALID_ARGUMENT
    assert L.dach_job_hist(None, 0, 1, p, p, 1, 8, p, 4, None) == _lib.INVALID_ARGUMENT
    assert L.dach_job_mask(None, 0, p, p, 1, 8, 42, p, None) == _lib.INVALID_ARGUMENT
    assert L.dach_job_wait(None, C.byref(C.c_uint64())) == _lib.INVALID_ARGUMENT
    assert "null" in _lib.last_error()


def test_jobs_without_gpu_fail_loudly():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    p = D.DoubleArrayAhoCorasick.new(["a"])
    with pytest.raises(D.DaachorseError) as e:
        p.job(0)
    assert e.value.code == _lib.CUDA_ERROR


@pytest.fixture
def fake_job(monkeypatch):
    """A Job whose handle and device image are fakes; every call of the four entry points is recorded."""
    L = _lib.load()
    calls = []
    monkeypatch.setattr(L, "dach_dev_upload", lambda h, dev, out: (setattr(out._obj, "value", 0x1000), _lib.OK)[1])
    monkeypatch.setattr(L, "dach_dev_free", lambda d: None)
    monkeypatch.setattr(L, "dach_job_create", lambda d, out: (setattr(out._obj, "value", 0x2000), _lib.OK)[1])
    monkeypatch.setattr(L, "dach_job_free", lambda j: None)
    for name in JOB_RK:
        monkeypatch.setattr(L, name, lambda *a, _n=name: calls.append(_n) or _lib.OK)

    made = []

    def make(cw=False):
        pma = (D.CharwiseDoubleArrayAhoCorasick if cw else D.DoubleArrayAhoCorasick).new(["ab", "b"])
        made.append((pma, pma.job(0)))
        return made[-1]

    yield make, calls
    assert calls == []  # nothing refused reached the library
    del made[:]
    gc.collect()  # the fake handles go to the fake frees, before the real ones come back


def _refused(f, code=_lib.INVALID_ARGUMENT, match=None):
    with pytest.raises(D.DaachorseError) as e:
        f()
    assert e.value.code == code
    if match:
        assert match in str(e.value), str(e.value)


def test_wrappers_refuse_before_the_library(fake_job):
    import torch

    make, calls = fake_job
    pma, job = make()
    _, cw_job = make(cw=True)
    t = torch.zeros(8, dtype=torch.uint8)
    o = torch.tensor([0, 4, 8], dtype=torch.int64)
    # the match kind: the crate's assertion, as in the *_device forms
    for f in (lambda: job.count(D.LEFTMOST_FIND, t, o), lambda: job.first(D.LEFTMOST_FIND, t, o),
              lambda: job.pattern_counts(D.LEFTMOST_FIND, t, o), lambda: job.mask(D.LEFTMOST_FIND, t, o)):
        with pytest.raises(AssertionError):
            f()
    # keys and fill bytes, checked before the tensors
    _refused(lambda: job.pattern_counts(D.FIND, t, o, key="pattern"), match="key")
    for fill in (256, -1, b"**", True):
        _refused(lambda: job.mask(D.FIND, t, o, fill=fill), match="fill")
    _refused(lambda: cw_job.mask(D.FIND, t, o, fill=0x80), match="ASCII")
    # tensors off the device
    for f in (lambda: job.count(D.FIND, t, o), lambda: job.first(D.FIND, t, o), lambda: job.pattern_counts(D.FIND, t, o),
              lambda: job.mask(D.FIND, t, o)):
        _refused(f, match="CUDA tensor")
    _refused(lambda: job.count(D.FIND, t, torch.zeros(0, dtype=torch.int64)), match="n + 1")
    assert calls == []


def test_job_wrappers_take_the_device_forms_arguments():
    """Same argument names and defaults as the *_device forms, so code can move between the two."""
    import inspect

    pairs = (("count", "count_batch_device"), ("first", "first_batch_device"),
             ("pattern_counts", "pattern_counts_device"), ("mask", "mask_batch_device"))
    for jname, dname in pairs:
        js = inspect.signature(getattr(D.automaton.Job, jname))
        ds = inspect.signature(getattr(D.automaton._Automaton, dname))
        assert [(p.name, p.default) for p in js.parameters.values()] == [(p.name, p.default) for p in ds.parameters.values()], jname
