#!/usr/bin/env python3
"""Per-byte event counts of the bytewise Standard lane machine on samples of the bench workloads, from
the CPU emulation of the kernels' lane code (tests/emu, StdMachine3 with its DACH_STAT counters).
No GPU needed.  Usage: python tools/lane_stats.py [C2|C3|C5 ...]

    python tools/lane_stats.py --events [C3 C3-find C2 C4 ...]

reports instead how the lane machines' output events (what a HIST scan counts per state) spread over the compact
slots: the share on the 1 / 64 / 1024 / 4096 busiest slots and on the leading 1024 / 4096 slots (what option hist_smem
counts in shared memory), from tests/emu_hist.

    python tools/lane_stats.py --lists [C3 C2 ...]

reports the output-list lengths of find_overlapping events (the matches that end at one position of a haystack come
from one event, and there are as many as the landed state's list is long): their distribution, and the share of
events whose list is too long for the length byte StdMachine3 queues with an event (255 or more: the drain reads the
head record's chain word instead), from the oracle's matches.

    python tools/lane_stats.py --pairs [C3 C3-find C2 C4 ...]

reports what a document-frequency window holds (dach_dev_df_batch, DESIGN.md section 4.9): the distinct (haystack,
state) pairs the lane machine puts into the first set and the distinct (haystack, key) pairs of the second, per MiB of
text, on 4 MiB of the workload's own haystacks, from tests/emu_df -- and so how much text one window of option
df_pairs pairs covers."""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np

import emu_api as E
import oracle_api as O
from daachorse_b200 import synth as S

NAMES = "steps probes hits miss_known miss_f2root learns root_falls root_stay sig_skips pushes cache_hits".split()
WHAT = {"steps": "lane iterations", "probes": "record fetches that are probes", "hits": "probes that hit (landings)",
        "miss_known": "own-child probes that missed (signature false positives)", "miss_f2root": "failure probes that missed, next: ROOT",
        "learns": "fetches of a failure state's record", "root_falls": "probes of ROOT's children", "root_stay": "landings in ROOT",
        "sig_skips": "bytes whose own-child probe the signature saved", "pushes": "landings on a state with outputs"}


def run(name, n_hay=256):
    cfg = S.config(name)
    ps = S.make_patterns(cfg)
    pool, b = S.make_pool(cfg, ps, 16 << 20)
    opma = O.OraclePma.build_packed(ps.blob, ps.offs)
    wire = opma.serialize()
    hay_len = min(cfg["hay_len"], 1 << 14)
    starts = S.window_starts(b, len(pool), n_hay, hay_len)
    text, offs = S.materialise_host(pool, starts, hay_len)
    buf = (C.c_ulonglong * len(NAMES))()
    lib = E.lib()
    E.scan(wire, False, 1, text, offs, kernel=3, out_cap=1 << 24)  # sizes the output; counters reset below
    lib.emu_stats(buf, 1)
    rc, m, oo, need = E.scan(wire, False, 1, text, offs, kernel=3, out_cap=max(int(need_cap(text)), 1 << 16))
    lib.emu_stats(buf, 1)
    nb = len(text)
    print("== %s: %d patterns, %d haystacks x %d B, %.4f matches/byte" % (name, len(ps), n_hay, hay_len, need / nb))
    for k, v in zip(NAMES, buf):
        if k in WHAT:
            print("   %-12s %8.4f per byte   %s" % (k, v / nb, WHAT[k]))


def need_cap(text):
    return len(text)  # >= 1 match per byte is far more than any config produces


EVENT_CONFIGS = {"C3": ("C3", 1), "C3-find": ("C3", 0), "C2": ("C2", 1), "C4": ("C4", 3)}


def event_shares(name, n_hay=256):
    import emu_hist_api as H

    synth, mode = EVENT_CONFIGS[name]
    cfg = S.config(synth)
    cw = cfg["variant"] == "charwise"
    ps = S.make_patterns(cfg)
    pool, b = S.make_pool(cfg, ps, 16 << 20)
    kind = 1 if mode == 3 else 0  # C4: LeftmostLongest
    opma = O.OraclePma.build_packed(ps.blob, ps.offs, charwise=cw, match_kind=kind)
    hay_len = min(cfg["hay_len"], 1 << 14)
    starts = S.window_starts(b, len(pool), n_hay, hay_len)
    text, offs = S.materialise_host(pool, starts, hay_len)
    if cw:
        text = S.pad_to_char_boundary(text.reshape(n_hay, hay_len)).reshape(-1)
    tops = [1, 64, 1024, 4096]
    all_, top, lead = H.event_shares(opma.serialize(), cw, mode, text, offs, tops)
    print("== %s: %d patterns, %d haystacks x %d B: %d events, %.4f per byte" % (name, len(ps), n_hay, hay_len, all_, all_ / len(text)))
    print("   busiest slots:  " + "  ".join("top %d %.1f %%" % (k, 100.0 * top[k] / max(all_, 1)) for k in tops))
    print("   leading slots:  " + "  ".join("< %d %.1f %%" % (k, 100.0 * lead[k] / max(all_, 1)) for k in tops[2:]))


def pair_counts(name, mib=4):
    import emu_df_api as F

    synth, mode = EVENT_CONFIGS[name]
    cfg = S.config(synth)
    cw = cfg["variant"] == "charwise"
    ps = S.make_patterns(cfg)
    pool, b = S.make_pool(cfg, ps, 16 << 20)
    kind = 1 if mode == 3 else 0  # C4: LeftmostLongest
    opma = O.OraclePma.build_packed(ps.blob, ps.offs, charwise=cw, match_kind=kind)
    hay_len = cfg["hay_len"]
    n_hay = max(1, (mib << 20) // hay_len)
    starts = S.window_starts(b, len(pool), n_hay, hay_len)
    text, offs = S.materialise_host(pool, starts, hay_len)
    if cw:
        text = S.pad_to_char_boundary(text.reshape(n_hay, hay_len)).reshape(-1)
    rc, _, _, info = F.df(opma.serialize(), cw, mode, "output", text, offs, len(ps), df_pairs=1 << 22)
    assert rc == 0 and info["rescans"] == 0
    per = len(text) / float(1 << 20)
    sp, kp = info["slot_pairs"] / per, info["key_pairs"] / per
    print("== %s: %d patterns, %d haystacks x %d B: per MiB %.0f (haystack, state) pairs, %.0f (haystack, key) pairs; "
          "the default 2^24 pairs cover %.0f MiB" % (name, len(ps), n_hay, hay_len, sp, kp, (1 << 24) / max(sp, kp, 1)))


def list_lengths(name, n_hay=256):
    cfg = S.config(name)
    ps = S.make_patterns(cfg)
    pool, b = S.make_pool(cfg, ps, 16 << 20)
    opma = O.OraclePma.build_packed(ps.blob, ps.offs)
    hay_len = min(cfg["hay_len"], 1 << 14)
    starts = S.window_starts(b, len(pool), n_hay, hay_len)
    text, offs = S.materialise_host(pool, starts, hay_len)
    ref = opma.scan_batch(O.FIND_OVERLAPPING, text, offs, want_matches=True)
    hay = np.repeat(np.arange(n_hay, dtype=np.uint64), ref["counts"].astype(np.int64))
    _, lens = np.unique((hay << np.uint64(32)) | ref["matches"]["end"].astype(np.uint64), return_counts=True)
    n = max(len(lens), 1)
    print("== %s find_overlapping: %d events, %.4f per byte, %.3f matches per event, longest list %d"
          % (name, len(lens), len(lens) / len(text), lens.sum() / n, lens.max() if len(lens) else 0))
    bins = [(1, 1), (2, 2), (3, 4), (5, 16), (17, 254), (255, 1 << 62)]
    print("   list length:  " + "  ".join("%s %.2f %%" % (str(lo) if lo == hi else "%d+" % lo if hi > 1 << 40 else "%d-%d" % (lo, hi),
                                                           100.0 * np.count_nonzero((lens >= lo) & (lens <= hi)) / n) for lo, hi in bins))
    print("   events that take the escape (list >= 255): %.4f %%" % (100.0 * np.count_nonzero(lens >= 255) / n))


if __name__ == "__main__":
    if sys.argv[1:2] == ["--lists"]:
        for nm in (sys.argv[2:] or ["C3", "C2"]):
            list_lengths(nm)
    elif sys.argv[1:2] == ["--pairs"]:
        for nm in (sys.argv[2:] or list(EVENT_CONFIGS)):
            pair_counts(nm)
    elif sys.argv[1:2] == ["--events"]:
        for nm in (sys.argv[2:] or list(EVENT_CONFIGS)):
            event_shares(nm)
    else:
        for nm in (sys.argv[1:] or ["C2", "C3"]):
            run(nm)
