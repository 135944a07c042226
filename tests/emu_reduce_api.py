"""ctypes binding of tests/emu_reduce/libdach_emu_reduce.so: COUNT / FIRST scans on the kernels' lane logic compiled
for the CPU (test infrastructure only)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
EMU_DIR = os.path.join(_HERE, "emu_reduce")
LIB = os.path.join(EMU_DIR, "libdach_emu_reduce.so")
MATCH_DTYPE = np.dtype([("start", "<u4"), ("end", "<u4"), ("value", "<u4")])
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", EMU_DIR, "-s"])
        L = C.CDLL(LIB)
        L.emu_reduce_batch_wire.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64,
                                            C.c_uint32, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
        L.emu_reduce_batch_wire.restype = C.c_int
        L.emu_image_outputs.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t]
        L.emu_image_outputs.restype = C.c_longlong
        L.emu_image_segmentable.argtypes = [C.c_void_p, C.c_size_t]
        L.emu_image_segmentable.restype = C.c_int
        L.emu_set_hot_slots.argtypes = [C.c_uint32]
        L.emu_stats.argtypes = [C.c_void_p, C.c_int]
        L.emu_stats.restype = None
        _lib = L
    return _lib


def image_segmentable(wire):
    """HostImage::segmentable of a serialized bytewise automaton (1 / 0; -1: refused)."""
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    return int(lib().emu_image_segmentable(wire_a.ctypes.data, wire_a.size))


def stats(reset=True):
    """EmuStats of the lane machines since the last reset: dict with 'steps', 'probes', ..."""
    names = ("steps", "probes", "hits", "miss_known", "miss_f2root", "learns", "root_falls", "root_stay", "sig_skips",
             "pushes", "cache_hits")
    buf = (C.c_ulonglong * len(names))()
    lib().emu_stats(buf, int(reset))
    return dict(zip(names, list(buf)))


def reduce(wire, charwise, mode, rk, text, offs, hot_n=0, kernel=3, seg_len=0):
    """dach_dev_count_batch (rk = 1) / dach_dev_first_batch (rk = 2) through the emulation.
    Returns (rc, counts or (first, found), total)."""
    L = lib()
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    text = np.ascontiguousarray(text, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.uint64)
    n = len(offs) - 1
    counts = np.zeros(max(n, 1), dtype=np.uint64)
    first = np.zeros(max(n, 1), dtype=MATCH_DTYPE)
    found = np.zeros(max(n, 1), dtype=np.uint8)
    tot = C.c_uint64()
    pad = text if text.size else np.zeros(16, dtype=np.uint8)
    rc = L.emu_reduce_batch_wire(wire_a.ctypes.data, wire_a.size, int(charwise), mode, rk, pad.ctypes.data, offs.ctypes.data, n,
                                 hot_n, kernel, seg_len, counts.ctypes.data, first.ctypes.data, found.ctypes.data, C.byref(tot))
    if rk == 1:
        return rc, counts[:n], tot.value
    return rc, (first[:n], found[:n].astype(bool)), tot.value


def image_outputs(wire, charwise=False):
    """The device image's output records as an (k, 4) uint32 array {value, length, parent, chain}."""
    L = lib()
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    k = L.emu_image_outputs(wire_a.ctypes.data, wire_a.size, int(charwise), None, 0)
    out = np.zeros((max(k, 1), 4), dtype=np.uint32)
    L.emu_image_outputs(wire_a.ctypes.data, wire_a.size, int(charwise), out.ctypes.data, k)
    return out[:k]
