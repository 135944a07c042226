"""COUNT / FIRST scans (dach_dev_count_batch / dach_dev_first_batch) on the CPU emulation of the kernels'
lane logic, tests/emu/libdach_emu.so (test infrastructure only)."""
import ctypes as C

import numpy as np

from emu_api import MATCH_DTYPE, image_outputs, image_segmentable, lib, stats  # noqa: F401


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


