"""StdMachine3's matches path with event blocks on the CPU emulation of the kernels' lane logic,
tests/emu/libdach_emu.so (test infrastructure only): the queue kernel or the direct one, placed by k_expand or
by block descriptors (k_blk_desc / k_expand_desc)."""
import ctypes as C

import numpy as np

from emu_api import MATCH_DTYPE, lib  # noqa: F401

NOT_STD3 = -1  # the automaton or mode does not run on StdMachine3


def scan(wire, mode, text, offs, hot_n=0, seg_len=0, seg_from=0, pool_blocks=None, out_cap=None, state=None, pos=None,
         direct=False, place_u=0, place_pad=0):
    """Returns (rc, matches, out_offs, needed, blocks_used).  Without pool_blocks / out_cap both grow until the batch
    fits.  `state` (np.uint32, n): stream chunks, updated in place; `pos` (np.uint32, n): their first positions.
    direct: k_scan_direct instead of the queue kernel; place_u > 0: placed from block descriptors (k_expand_desc),
    place_u blocks per warp, the output place_pad words past a 16-byte boundary."""
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
                                        C.byref(need), C.byref(used), int(direct), place_u, place_pad)
        if rc == 6 and out_cap is None and pool_blocks is None:
            if state is not None:
                state[:] = saved
            cap = max(cap * 2, int(need.value))
            continue
        return rc, out[: need.value] if rc == 0 else None, oo, int(need.value), int(used.value)
