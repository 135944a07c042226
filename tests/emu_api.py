"""ctypes binding of tests/emu/libdach_emu.so: the kernels' lane logic compiled for the CPU, every result kind
(test infrastructure only).  The library is built and loaded here once; emu_reduce_api, emu_hist_api, emu_df_api,
emu_mask_api and emu_events_api wrap its other entry points."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
EMU_DIR = os.path.join(_HERE, "emu")
LIB = os.path.join(EMU_DIR, "libdach_emu.so")
MATCH_DTYPE = np.dtype([("start", "<u4"), ("end", "<u4"), ("value", "<u4")])
_lib = None

_P, _SZ, _I, _U32, _U64, _I64 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32, C.c_uint64, C.c_int64
_PU32, _PU64, _PI = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_int)
_SIGNATURES = {  # name: (restype, argtypes)
    "emu_scan_batch_wire": (_I, [_P, _SZ, _I, _I, _P, _P, _U64, _U32, _I, _U32, _U32, _U32, _P, _U64, _P, _PU64]),
    "emu_scan_stream_wire": (_I, [_P, _SZ, _I, _P, _P, _U64, _P, _P, _U32, _P, _U64, _P, _PU64]),
    "emu_events_scan_wire": (_I, [_P, _SZ, _I, _P, _P, _U64, _U32, _U32, _U32, _U32, _P, _P, _P, _U64, _P, _PU64, _PU32,
                                  _I, _U32, _U32]),
    "emu_place_tables": (_I64, [_P, _SZ, _P, _P, _U64]),
    "emu_reduce_batch_wire": (_I, [_P, _SZ, _I, _I, _I, _P, _P, _U64, _U32, _I, _U32, _P, _P, _P, _PU64]),
    "emu_rk_stream_wire": (_I, [_P, _SZ, _I, _I, _I, _I, _P, _P, _U64, _P, _P, _U32, _I, _I64, _P, _P, _P, _P, _U64, _PU64]),
    "emu_hist_batch_wire": (_I, [_P, _SZ, _I, _I, _I, _P, _P, _U64, _U32, _I, _U32, _I64, _P, _U64, _PU64, _PI]),
    "emu_hist_event_shares": (_I, [_P, _SZ, _I, _I, _P, _P, _U64, _P, _I, _P]),
    "emu_df_batch_wire": (_I, [_P, _SZ, _I, _I, _I, _P, _P, _U64, _U32, _I, _U32, _I64, _I, _P, _U64, _PU64, _P]),
    "emu_mask_batch_wire": (_I, [_P, _SZ, _I, _I, _P, _P, _U64, _U64, C.c_uint8, _U32, _I, _U32, _P, _PI]),
    "emu_check_image_transitions": (C.c_longlong, [_P, _SZ, _U32, _PU32, _PU32]),
    "emu_check_image_transitions_charwise": (C.c_longlong, [_P, _SZ]),
    "emu_image_segmentable": (_I, [_P, _SZ]),
    "emu_image_outputs": (C.c_longlong, [_P, _SZ, _I, _P, _SZ]),
    "emu_stats": (None, [_P, _I]),
    "emu_set_hot_slots": (None, [_U32]),
    "emu_stream_config": (None, [_I, _U32]),
    "emu_stream_charwise": (None, [_I]),
}


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", EMU_DIR, "-s"])
        L = C.CDLL(LIB)
        for name, (res, args) in _SIGNATURES.items():
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _lib = L
    return _lib


def stats(reset=True):
    """EmuStats of the lane machines since the last reset: dict with 'steps', 'probes', ..."""
    names = ("steps", "probes", "hits", "miss_known", "miss_f2root", "learns", "root_falls", "root_stay", "sig_skips",
             "pushes", "cache_hits")
    buf = (C.c_ulonglong * len(names))()
    lib().emu_stats(buf, int(reset))
    return dict(zip(names, list(buf)))


def image_segmentable(wire):
    """HostImage::segmentable of a serialized bytewise automaton (1 / 0; -1: refused)."""
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    return int(lib().emu_image_segmentable(wire_a.ctypes.data, wire_a.size))


def image_outputs(wire, charwise=False):
    """The device image's output records as an (k, 4) uint32 array {value, length, parent, chain}."""
    L = lib()
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    k = L.emu_image_outputs(wire_a.ctypes.data, wire_a.size, int(charwise), None, 0)
    out = np.zeros((max(k, 1), 4), dtype=np.uint32)
    L.emu_image_outputs(wire_a.ctypes.data, wire_a.size, int(charwise), out.ctypes.data, k)
    return out[:k]


def check_image_transitions_charwise(wire):
    """The charwise compact image: every (state, mapped code) transition against the crate's; mismatches."""
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    return int(lib().emu_check_image_transitions_charwise(wire_a.ctypes.data, wire_a.size))


def check_image_transitions(wire, want_hot_slots):
    """Every (state, byte) transition of the compact bytewise device image against the crate's transition
    function.  Returns (mismatches, hot_slots, states placed in the hot region)."""
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    hs, hu = C.c_uint32(), C.c_uint32()
    bad = lib().emu_check_image_transitions(wire_a.ctypes.data, wire_a.size, int(want_hot_slots), C.byref(hs), C.byref(hu))
    return int(bad), int(hs.value), int(hu.value)


def scan(wire, charwise, mode, text, offs, hot_n=0, pool_blocks=None, out_cap=None, kernel=3, seg_len=0, seg_from=0):
    """Returns (rc, matches, out_offs, needed)."""
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    text = np.ascontiguousarray(text, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.uint64)
    n = len(offs) - 1
    cap = int(out_cap) if out_cap is not None else 1 << 16
    while True:
        n_items = n + (int(text.size) // seg_len + 1 if seg_len else 0)
        pb = int(pool_blocks) if pool_blocks is not None else cap // 15 + n_items + 16
        out = np.zeros(max(cap, 1), dtype=MATCH_DTYPE)
        oo = np.zeros(n + 1, dtype=np.uint64)
        need = C.c_uint64()
        pad = text if text.size else np.zeros(16, dtype=np.uint8)
        rc = lib().emu_scan_batch_wire(wire_a.ctypes.data, wire_a.size, int(charwise), mode, pad.ctypes.data,
                                       offs.ctypes.data, n, hot_n, kernel, seg_len, seg_from, pb, out.ctypes.data, cap, oo.ctypes.data,
                                       C.byref(need))
        if rc == 6 and out_cap is None and pool_blocks is None:
            cap = max(cap * 2, int(need.value))
            continue
        return rc, out[: need.value] if rc == 0 else None, oo, need.value


def scan_stream(wire, mode, text, offs, state, pos=None, out_cap=1 << 16):
    """dach_dev_scan_stream through the emulation: ``state`` (uint32, n) is updated in place.
    Returns (rc, matches, out_offs, needed)."""
    wire_a = np.frombuffer(wire, dtype=np.uint8)
    text = np.ascontiguousarray(text, dtype=np.uint8)
    offs = np.ascontiguousarray(offs, dtype=np.uint64)
    n = len(offs) - 1
    assert state.dtype == np.uint32 and len(state) == n
    cap = int(out_cap)
    while True:
        saved = state.copy()
        out = np.zeros(max(cap, 1), dtype=MATCH_DTYPE)
        oo = np.zeros(n + 1, dtype=np.uint64)
        need = C.c_uint64()
        pad = text if text.size else np.zeros(16, dtype=np.uint8)
        rc = lib().emu_scan_stream_wire(wire_a.ctypes.data, wire_a.size, mode, pad.ctypes.data, offs.ctypes.data, n,
                                        state.ctypes.data, pos.ctypes.data if pos is not None else None, cap // 15 + n + 16,
                                        out.ctypes.data, cap, oo.ctypes.data, C.byref(need))
        if rc == 6:
            state[:] = saved
            cap = max(cap * 2, int(need.value))
            continue
        return rc, out[: need.value] if rc == 0 else None, oo, need.value
