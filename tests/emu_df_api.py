"""Per-pattern document frequencies (dach_dev_df_batch) on the CPU emulation of the kernels' lane logic,
tests/emu/libdach_emu.so (test infrastructure only)."""
import ctypes as C

import numpy as np

from emu_api import lib

KEY = {"output": 0, "value": 1}


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
