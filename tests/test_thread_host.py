"""device_handle under host threads: eight threads making their first device call at the same moment share one upload
of the scan image and one handle, and the automaton frees exactly that handle when it is collected.  The upload is
replaced by a slow fake (no GPU needed), so that every thread is inside device_handle while the first upload runs."""
import ctypes as C
import gc
import threading
import time

import daachorse_b200 as D
from daachorse_b200 import _lib


def test_device_handle_uploads_once_under_threads(monkeypatch):
    L = _lib.load()
    pma = D.DoubleArrayAhoCorasick.new(["ab", "bcd", "x"])
    lock = threading.Lock()
    uploads, frees = [], []

    def fake_upload(h, device, out):
        time.sleep(0.05)  # releases the GIL, as the real upload does inside ctypes
        with lock:
            uploads.append(device)
            handle = 0x10000 + 0x100 * len(uploads)
        out._obj.value = handle
        return _lib.OK

    def fake_free(d):
        with lock:
            frees.append(d.value if isinstance(d, C.c_void_p) else d)

    monkeypatch.setattr(L, "dach_dev_upload", fake_upload)
    monkeypatch.setattr(L, "dach_dev_free", fake_free)
    n = 8
    barrier = threading.Barrier(n)
    seen, errors = [None] * n, []

    def worker(i):
        try:
            barrier.wait(timeout=30)
            seen[i] = pma.device_handle(0).value
        except Exception as e:  # reported below; a thread must not die silently
            errors.append(repr(e))

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(n)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=30)
    assert not any(t.is_alive() for t in threads)
    assert errors == []
    assert len(uploads) == 1, uploads
    assert len(set(seen)) == 1 and seen[0] == 0x10100, seen
    assert pma.device_handle(0).value == seen[0] and len(uploads) == 1  # later calls reuse it
    del pma
    gc.collect()
    assert frees == [seen[0]]
