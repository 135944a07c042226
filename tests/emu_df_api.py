"""ctypes binding of tests/emu_df/libdach_emu_df.so: per-pattern document frequencies (dach_dev_df_batch) on the kernels'
lane logic compiled for the CPU (test infrastructure only)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
EMU_DIR = os.path.join(_HERE, "emu_df")
LIB = os.path.join(EMU_DIR, "libdach_emu_df.so")
KEY = {"output": 0, "value": 1}
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", EMU_DIR, "-s"])
        L = C.CDLL(LIB)
        L.emu_df_batch_wire.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64,
                                        C.c_uint32, C.c_int, C.c_uint32, C.c_int64, C.c_int, C.c_void_p, C.c_uint64,
                                        C.POINTER(C.c_uint64), C.c_void_p]
        L.emu_df_batch_wire.restype = C.c_int
        _lib = L
    return _lib


def df(wire, charwise, mode, key, text, offs, n_df, hot_n=0, kernel=3, seg_len=0, df_pairs=1 << 16, split=True, out=None):
    """dach_dev_df_batch through the emulation: adds into `out` (np.uint64[n_df], zeros if None).
    Returns (rc, df, total, info) -- info: windows, rescans, which (the kernel that ran, 3 / 1 / 0, + 8 if parent
    chains were expanded), left (set entries still taken after the call), slot_pairs / key_pairs (the most pairs one
    window put into each set)."""
    L = lib()
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    text = np.ascontiguousarray(text, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.uint64)
    n = len(offs) - 1
    h = np.zeros(max(n_df, 1), dtype=np.uint64) if out is None else out
    tot = C.c_uint64()
    info = np.zeros(6, dtype=np.uint64)
    pad = text if text.size else np.zeros(16, dtype=np.uint8)
    rc = L.emu_df_batch_wire(wire_a.ctypes.data, wire_a.size, int(charwise), mode, KEY[key], pad.ctypes.data, offs.ctypes.data, n,
                             hot_n, kernel, seg_len, df_pairs, int(split), h.ctypes.data, n_df, C.byref(tot), info.ctypes.data)
    names = ("windows", "rescans", "which", "left", "slot_pairs", "key_pairs")
    return rc, h[:n_df], tot.value, dict(zip(names, map(int, info)))
