"""ctypes binding of tests/emu_events/libdach_emu_events.so: StdMachine3's matches path with event blocks (the drain
that stores events, k_expand) on the kernels' lane logic compiled for the CPU (test infrastructure only)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
EMU_DIR = os.path.join(_HERE, "emu_events")
LIB = os.path.join(EMU_DIR, "libdach_emu_events.so")
MATCH_DTYPE = np.dtype([("start", "<u4"), ("end", "<u4"), ("value", "<u4")])
NOT_STD3 = -1  # the automaton or mode does not run on StdMachine3
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", EMU_DIR, "-s"])
        L = C.CDLL(LIB)
        L.emu_events_scan_wire.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32,
                                           C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                           C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
        L.emu_events_scan_wire.restype = C.c_int
        _lib = L
    return _lib


def scan(wire, mode, text, offs, hot_n=0, seg_len=0, seg_from=0, pool_blocks=None, out_cap=None, state=None, pos=None):
    """Returns (rc, matches, out_offs, needed, blocks_used).  Without pool_blocks / out_cap both grow until the batch
    fits.  `state` (np.uint32, n): stream chunks, updated in place; `pos` (np.uint32, n): their first positions."""
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    text = np.ascontiguousarray(text, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.uint64)
    n = len(offs) - 1
    cap = int(out_cap) if out_cap is not None else 1 << 12
    pad = text if text.size else np.zeros(16, dtype=np.uint8)
    while True:
        pb = int(pool_blocks) if pool_blocks is not None else cap // 30 + n + (text.size // seg_len + 1 if seg_len else 0) + 16
        saved = state.copy() if state is not None else None
        out = np.zeros(max(cap, 1), dtype=MATCH_DTYPE)
        oo = np.zeros(n + 1, dtype=np.uint64)
        need, used = C.c_uint64(), C.c_uint32()
        rc = lib().emu_events_scan_wire(wire_a.ctypes.data, wire_a.size, mode, pad.ctypes.data, offs.ctypes.data, n, hot_n,
                                        seg_len, seg_from, pb, state.ctypes.data if state is not None else None,
                                        pos.ctypes.data if pos is not None else None, out.ctypes.data, cap, oo.ctypes.data,
                                        C.byref(need), C.byref(used))
        if rc == 6 and out_cap is None and pool_blocks is None:
            if state is not None:
                state[:] = saved
            cap = max(cap * 2, int(need.value))
            continue
        return rc, out[: need.value] if rc == 0 else None, oo, int(need.value), int(used.value)
