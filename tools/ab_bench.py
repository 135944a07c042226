#!/usr/bin/env python3
"""A/B timing of kernel options on ONE GPU (machines differ by a few percent, so variants are only comparable
inside one run): builds the C3 batch once, then times the device-resident find_overlapping step
for every option set given on the command line.

    python tools/ab_bench.py [--scale 0.25] [--config C3] [--reps 5] "kernel=3" "kernel=3,hot_entries=0" "kernel=2"
    DACH_LIB=tools/alt/lib_x.so python tools/ab_bench.py ...      # an experiment build of the library

Prints one line per option set: whole-step GB/s, scan-kernel GB/s (CUDA events inside the library)."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import daachorse_b200 as D
from daachorse_b200 import synth as S

ap = argparse.ArgumentParser()
ap.add_argument("--scale", type=float, default=0.25)
ap.add_argument("--config", default="C3")
ap.add_argument("--mode", default="overlapping")
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--tag", default=os.environ.get("DACH_LIB", "default"))
ap.add_argument("sets", nargs="*")
a = ap.parse_args()

cfg = S.config(a.config, a.scale)
ps = S.make_patterns(cfg)
pool, b = S.make_pool(cfg, ps, 64 << 20)
starts = S.window_starts(b, len(pool), cfg["n_haystacks"], cfg["hay_len"])
pma = D.DoubleArrayAhoCorasick.new(ps.as_list())
pool_t = torch.from_numpy(pool).cuda()
text_t, offs_t = S.materialise_on_device(pool_t, torch.from_numpy(starts).cuda(), cfg["hay_len"])
del pool_t
mode = {"overlapping": D.FIND_OVERLAPPING, "find": D.FIND, "no_suffix": D.FIND_OVERLAPPING_NO_SUFFIX}[a.mode]
r = pma.scan_batch_device(mode, text_t, offs_t)
out = torch.empty((r.matches.shape[0] + 1024, 3), dtype=torch.int32, device="cuda")
oo = torch.empty(offs_t.numel(), dtype=torch.int64, device="cuda")
base_sum = int(r.matches.to(torch.int64).sum().item())
nb = text_t.numel()
DEFAULTS = {"kernel": 3, "hot_entries": 6144, "threads": 1024, "ctas_per_sm": 1, "l2_hints": 2, "gather_ordered": 1}
for s in (a.sets or ["kernel=3"]):
    opts = dict(DEFAULTS)
    for kv in s.split(","):
        if kv:
            k, v = kv.split("=")
            opts[k] = int(v)
    for k, v in opts.items():
        pma.set_option(k, v)
    ms, ks = [], []
    for i in range(a.reps + 2):
        r = pma.scan_batch_device(mode, text_t, offs_t, out=out, out_offs=oo)
        st = pma.stats()
        if i >= 2:
            ms.append(st["total_ms"])
            ks.append(st["scan_kernel_ms"])
    ok = int(r.matches.to(torch.int64).sum().item()) == base_sum
    print("%-28s %-44s step %7.1f GB/s  kernel %7.1f GB/s (best %7.1f)  %s" % (
        a.tag[-28:], s, nb / (np.mean(ms) * 1e-3) / 1e9, nb / (np.mean(ks) * 1e-3) / 1e9, nb / (min(ks) * 1e-3) / 1e9,
        "sum ok" if ok else "SUM DIFFERS"), flush=True)
