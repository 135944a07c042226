"""ctypes binding of tests/emu_hist/libdach_emu_hist.so: per-pattern histograms (dach_dev_hist_batch) on the kernels'
lane logic compiled for the CPU (test infrastructure only)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
EMU_DIR = os.path.join(_HERE, "emu_hist")
LIB = os.path.join(EMU_DIR, "libdach_emu_hist.so")
KEY = {"output": 0, "value": 1}
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", EMU_DIR, "-s"])
        L = C.CDLL(LIB)
        L.emu_hist_batch_wire.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64,
                                          C.c_uint32, C.c_int, C.c_uint32, C.c_int64, C.c_void_p, C.c_uint64,
                                          C.POINTER(C.c_uint64), C.POINTER(C.c_int)]
        L.emu_hist_batch_wire.restype = C.c_int
        L.emu_hist_event_shares.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64,
                                            C.c_void_p, C.c_int, C.c_void_p]
        L.emu_hist_event_shares.restype = C.c_int
        L.emu_hist_set_hot_slots.argtypes = [C.c_uint32]
        _lib = L
    return _lib


def hist(wire, charwise, mode, key, text, offs, n_hist, hot_n=0, kernel=3, seg_len=0, hist_smem=1024, out=None):
    """dach_dev_hist_batch through the emulation: adds into `out` (np.uint64[n_hist], zeros if None).
    Returns (rc, hist, total, which) -- which: the kernel that ran (3 / 1 / 0), + 8 if parent chains were expanded."""
    L = lib()
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    text = np.ascontiguousarray(text, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.uint64)
    n = len(offs) - 1
    h = np.zeros(max(n_hist, 1), dtype=np.uint64) if out is None else out
    tot = C.c_uint64()
    which = C.c_int(-1)
    pad = text if text.size else np.zeros(16, dtype=np.uint8)
    rc = L.emu_hist_batch_wire(wire_a.ctypes.data, wire_a.size, int(charwise), mode, KEY[key], pad.ctypes.data, offs.ctypes.data,
                               n, hot_n, kernel, seg_len, hist_smem, h.ctypes.data, n_hist, C.byref(tot), C.byref(which))
    return rc, h[:n_hist], tot.value, which.value


def event_shares(wire, charwise, mode, text, offs, tops):
    """The lane machine's events on compact slots: (all events, {k: events on the k most frequent slots},
    {k: events on compact slots < k})."""
    L = lib()
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    text = np.ascontiguousarray(text, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.uint64)
    top = np.ascontiguousarray(tops, dtype=np.uint32)
    out = np.zeros(1 + 2 * len(tops), dtype=np.uint64)
    rc = L.emu_hist_event_shares(wire_a.ctypes.data, wire_a.size, int(charwise), mode, text.ctypes.data, offs.ctypes.data, len(offs) - 1,
                                 top.ctypes.data, len(tops), out.ctypes.data)
    if rc:
        raise ValueError("no lane machine runs this automaton and mode")
    k = len(tops)
    return int(out[0]), dict(zip(tops, map(int, out[1:1 + k]))), dict(zip(tops, map(int, out[1 + k:])))
