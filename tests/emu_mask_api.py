"""Masked text (dach_dev_mask_batch) on the CPU emulation of the kernels' lane logic, tests/emu/libdach_emu.so
(test infrastructure only), and the reference the mask tests compare against."""
import ctypes as C

import numpy as np

from emu_api import lib


def mask(wire, charwise, mode, text, offs, fill, hot_n=0, kernel=3, seg_len=0, out=None):
    """dach_dev_mask_batch through the emulation: (rc, masked text, which) -- which: the kernel that ran (3 / 1 / 0),
    + 8 if haystacks were cut into segments; -1 if nothing was scanned."""
    L = lib()
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    text = np.ascontiguousarray(text, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.uint64)
    if out is None:
        out = np.full(max(text.size, 1), 0xEE, dtype=np.uint8)
    pad = text if text.size else np.zeros(16, dtype=np.uint8)
    which = C.c_int(-1)
    rc = L.emu_mask_batch_wire(wire_a.ctypes.data, wire_a.size, int(charwise), mode, pad.ctypes.data, offs.ctypes.data, len(offs) - 1,
                               text.size, fill, hot_n, kernel, seg_len, out.ctypes.data, C.byref(which))
    return rc, out[:text.size], which.value


def expected_mask(text, offs, starts, ends, hay, fill):
    """``text`` with bytes [offs[hay[k]] + starts[k], offs[hay[k]] + ends[k]) set to ``fill`` for every match k (a
    difference array over the text: overlapping spans and zero-length matches need no special case)."""
    text = np.asarray(text, dtype=np.uint8)
    offs = np.asarray(offs, dtype=np.uint64).astype(np.int64)
    base = offs[np.asarray(hay, dtype=np.int64)] if len(hay) else np.zeros(0, np.int64)
    s = base + np.asarray(starts, dtype=np.int64)
    e = base + np.asarray(ends, dtype=np.int64)
    keep = e > s
    d = np.bincount(s[keep], minlength=text.size + 1) - np.bincount(e[keep], minlength=text.size + 1)
    out = text.copy()
    out[np.cumsum(d[:-1]) > 0] = fill
    return out


def expected_from_matches(text, offs, matches, counts, fill):
    """expected_mask of a match list in dach_dev_scan_batch's layout: structured (start, end, value) and per-haystack
    counts."""
    hay = np.repeat(np.arange(len(counts)), np.asarray(counts, dtype=np.int64))
    return expected_mask(text, offs, matches["start"], matches["end"], hay, fill)
