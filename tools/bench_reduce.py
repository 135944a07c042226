#!/usr/bin/env python3
"""tools/bench_reduce.py -- counts and first matches on the bench.py workloads, one H100:

    python tools/bench_reduce.py --output counts [--config C3|C3-find|C2|C4|C5] [--steps K] [--warmup W]
    python tools/bench_reduce.py --output first  ...
    python tools/bench_reduce.py --output hist [--key value|output] ...
    python tools/bench_reduce.py --output df [--key value|output] ...
    python tools/bench_reduce.py --output mask [--fill N] [--alt-mib M] ...
    python tools/bench_reduce.py --stream --output counts|hist [--key value|output] [--config C2|C3|C3-find] ...

One step = one dach_dev_count_batch / dach_dev_first_batch / dach_dev_hist_batch / dach_dev_df_batch on the step's
batch (the batches, automata and seeds of bench.py).  One JSON line, bench.py's fields where they apply:
  value              bytes offered / device time of the call's pipeline (CUDA events inside the library; df: CUDA events
                     around whole steps, since a step is many windows)
  roofline           bench.py's definition, on the COUNT / FIRST scan kernel
  e2e                the same batch through dach_count_batch_host / dach_first_batch_host from pinned host text
  parity             per-haystack counts and their total (counts), or first tuples and found flags (first), against
                     the oracle on the first --parity-frac of the last batch; and the whole step against the full
                     matches scan of the same batch
  first_end_frac     (first) mean first.end / haystack length over the haystacks with a match: how much of what it
                     is offered FIRST reads
  alternatives       (hist) in the same run, GB/s by CUDA events around whole steps: the histogram call, the full
                     matches scan (dach_dev_scan_batch) + torch.bincount of the values, and COUNT; the hist parity
                     checks the value-keyed histogram against np.bincount of the oracle sample's values, and the whole
                     step against the full scan bincounted on the device
  alternatives       (df) in the same run: the document-frequency call, the full matches scan + the haystack index of
                     every match, torch.unique of the (haystack, key) pairs and a bincount, and the histogram call; the
                     df parity checks the value-keyed counts against np.unique of the oracle sample's (haystack, value)
                     pairs, and the whole step against the matches path; windows / rescans of the last call
  alternatives       (--stream) each step is one round: the step's batch is the next chunk of n streams, the state
                     carried from step to step.  GB/s by CUDA events around whole steps of the stream form
                     (dach_dev_count_stream / dach_dev_hist_stream) and of scan_stream_device + torch on the same
                     rounds; parity: counts / histogram and the carried state, stream form vs matches stream
  alternatives       (mask) in the same run: the mask call, COUNT (the same scan without the stores), the copy kernel
                     alone (a mask call with no haystack), and the matches path + a torch span fill in slices of
                     --alt-mib; the mask parity checks the host form on the oracle sample's spans, and the whole step
                     against the torch span fill
  launches_per_step  kernels launched per step
Nothing is written to the tree.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

from bench import CONFIGS, UNIT, ClockSampler, Workload, measured_peaks, metric_name, mode_ids  # noqa: E402


def reduce_parity(output, got_counts, got_first, got_found, ref_counts, ref_first, ref_found):
    """In-run parity of --output counts / first on the oracle sample: per-haystack counts (and their total), or first
    tuples and found flags.  got_* / ref_*: numpy arrays over the same haystacks; the first tuples may cover a prefix."""
    if output == "counts":
        return {"counts_equal": bool(np.array_equal(got_counts.astype(np.uint64), ref_counts.astype(np.uint64))),
                "total_equal": int(got_counts.astype(np.uint64).sum()) == int(ref_counts.astype(np.uint64).sum())}
    k = len(ref_first)
    return {"found_equal": bool(np.array_equal(got_found.astype(bool), ref_found.astype(bool))),
            "first_equal": got_first[:k].astype(np.uint32).tobytes() == ref_first.astype(np.uint32).tobytes()}


def hist_parity(got_hist, ref_values, n_hist):
    """In-run parity of --output hist (value key) on the oracle sample: the histogram against np.bincount of the
    oracle's match values, and its total against their number."""
    ref = np.bincount(np.asarray(ref_values, dtype=np.int64), minlength=n_hist).astype(np.uint64)
    got = np.asarray(got_hist).astype(np.uint64)
    return {"hist_equal": bool(len(got) == len(ref) and np.array_equal(got, ref)),
            "total_equal": int(got.sum()) == int(len(ref_values))}


def df_parity(got_df, ref_counts, ref_values, n_df):
    """In-run parity of --output df (value key) on the oracle sample: the counts against a bincount of np.unique of the
    oracle's (haystack, value) pairs, and their total against the number of those pairs."""
    hay = np.repeat(np.arange(len(ref_counts), dtype=np.uint64), np.asarray(ref_counts, dtype=np.int64))
    pairs = np.unique((hay << np.uint64(32)) | np.asarray(ref_values, dtype=np.uint64))
    ref = np.bincount((pairs & np.uint64(0xffffffff)).astype(np.int64), minlength=n_df).astype(np.uint64)
    got = np.asarray(got_df).astype(np.uint64)
    return {"df_equal": bool(len(got) == len(ref) and np.array_equal(got, ref)), "total_equal": int(got.sum()) == int(len(pairs))}


def first_from_matches(matches, counts):
    """(first tuples (k, 3) u32, found (k,)) of haystacks whose runs of `matches` have lengths `counts`; all-ones
    where a haystack has none."""
    counts = np.asarray(counts, dtype=np.int64)
    m = np.asarray(matches).reshape(-1, 3) if not hasattr(matches, "dtype") or matches.dtype.names is None else \
        np.stack([matches["start"], matches["end"], matches["value"]], axis=1)
    first = np.full((len(counts), 3), 0xFFFFFFFF, dtype=np.uint32)
    found = counts > 0
    starts = np.concatenate([[0], np.cumsum(counts)])[:-1]
    first[found] = m[starts[found]].astype(np.uint32)
    return first, found


def first_end_frac(first, found, hay_lens):
    """mean of first.end / haystack length over the haystacks with a match (None if there is none): the share of a
    haystack FIRST had to read."""
    found = np.asarray(found, dtype=bool)
    if not found.any():
        return None
    ends = np.asarray(first, dtype=np.uint32).reshape(-1, 3)[found, 1].astype(np.float64)
    lens = np.asarray(hay_lens, dtype=np.float64)[found]
    return float(np.mean(ends / np.maximum(lens, 1)))


def run_reduce_output(args, W, pma, batches, dmode, omode, n, hay_len, step_bytes, resident, dev, t_setup):
    """--output counts / first on one GPU: every step is one dach_dev_count_batch / dach_dev_first_batch on the step's
    batch.  value = bytes offered / device time of the call's pipeline (CUDA events inside the library)."""
    import torch

    setup_s = time.time() - t_setup
    if args.stream:
        return run_stream_output(args, W, pma, batches, dmode, n, hay_len, step_bytes, resident, dev, setup_s)
    if args.output == "df":
        return run_df_output(args, W, pma, batches, dmode, omode, n, hay_len, step_bytes, resident, dev, setup_s)
    if args.output == "mask":
        return run_mask_output(args, W, pma, batches, dmode, omode, n, hay_len, step_bytes, resident, dev, setup_s)
    if args.output == "hist":
        return run_hist_output(args, W, pma, batches, dmode, omode, n, hay_len, step_bytes, resident, dev, setup_s)
    counts_t = torch.empty(n, dtype=torch.int64, device=dev)
    first_t = torch.empty((n, 3), dtype=torch.int32, device=dev)
    found_t = torch.empty(n, dtype=torch.bool, device=dev)

    def step(s):
        t, o = batches[s % len(batches)]
        if args.output == "counts":
            pma.count_batch_device(dmode, t, o, out=counts_t)
        else:
            pma.first_batch_device(dmode, t, o, out=first_t, found=found_t)
        st = pma.stats()
        return st["scan_kernel_ms"], st["total_ms"]

    for s in range(args.warmup):
        step(s)
    torch.cuda.synchronize()
    sampler = ClockSampler(dev.index)
    sampler.start()
    time.sleep(0.2)
    n_before = len(sampler.rows)
    launches1 = pma.stats()["launches"]
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    times = [step(args.warmup + s) for s in range(args.steps)]
    ev1.record()
    torch.cuda.synchronize()
    time.sleep(0.25)
    clocks = sampler.stop(skip=n_before)
    launches2 = pma.stats()["launches"]
    wall_ms = ev0.elapsed_time(ev1) / args.steps
    k_ms = float(np.mean([t[0] for t in times]))
    dev_ms = float(np.mean([t[1] for t in times]))
    value = step_bytes / (dev_ms * 1e-3) / 1e9
    last_batch = (args.warmup + args.steps - 1) % len(batches)
    t_last, o_last = batches[last_batch]
    # the full scan of the same batch (untimed): its per-haystack runs are what counts / first must equal
    r = pma.scan_batch_device(dmode, t_last, o_last)
    full_counts = torch.diff(r.offsets)
    extra = {}
    if args.output == "counts":
        step_ok = bool(torch.equal(counts_t, full_counts))
        extra["total"] = int(counts_t.sum().item())
    else:
        fd = full_counts > 0
        step_ok = bool(torch.equal(found_t, fd)) and bool(torch.equal(first_t[fd], r.matches[r.offsets[:-1][fd]]))
        extra["n_found"] = int(found_t.sum().item())
        hl = torch.diff(o_last).cpu().numpy()
        extra["first_end_frac"] = first_end_frac(first_t.cpu().numpy().view(np.uint32), found_t.cpu().numpy(), hl)
    del r, full_counts
    parity = None
    if not args.no_cpu:
        import oracle_api as O

        threads = O.cpu_budget()["threads"]
        ns = max(1, min(n, int(n * args.parity_frac)))
        nt = max(1, ns // 4)
        opma = W.oracle()
        lo = W.batch_ranges()[last_batch][0]
        ptext, poffs = W.host_batch(lo, lo + ns)
        ref = opma.scan_batch(omode, ptext, poffs, nthreads=threads, want_hashes=False)
        ref_t = opma.scan_batch(omode, ptext[: int(poffs[nt])], poffs[: nt + 1], nthreads=threads, want_matches=True)
        ref_first, _ = first_from_matches(ref_t["matches"], ref_t["counts"])
        parity = reduce_parity(args.output, counts_t[:ns].cpu().numpy(), first_t[:ns].cpu().numpy().view(np.uint32),
                               found_t[:ns].cpu().numpy(), ref["counts"], ref_first, ref["counts"] > 0)
        parity.update({"haystacks_checked": ns, "share_of_batch": ns / n, "first_tuples_checked": nt if args.output == "first" else 0,
                       "what": "last timed step vs the oracle on the first %d haystacks of its batch" % ns})
    parity = dict(parity or {}, step_equals_full_scan=step_ok)
    e2e = None
    if not args.no_e2e:
        t0_, o0_ = batches[0]
        h_text_t = torch.empty(t0_.numel(), dtype=torch.uint8).pin_memory()  # as the matches path: pinned host text
        h_text_t.copy_(t0_)
        h_text = h_text_t.numpy()
        h_offs = o0_.cpu().numpy().astype(np.uint64)
        e2e_ms = []
        for i in range(1 + args.e2e_steps):
            t0 = time.perf_counter()
            if args.output == "counts":
                pma.count_batch_host(dmode, h_text, h_offs)
            else:
                pma.first_batch_host(dmode, h_text, h_offs)
            if i >= 1:
                e2e_ms.append((time.perf_counter() - t0) * 1e3)
        st = pma.stats()
        e2e = {"value": h_text.size / (np.mean(e2e_ms) * 1e-3) / 1e9, "unit": UNIT, "h2d_bytes_per_step": int(st["h2d_bytes"]),
               "d2h_bytes_per_step": int(st["d2h_bytes"]), "ms_per_step": float(np.mean(e2e_ms)),
               "workload": "the step batch's %d haystacks x %d B through the host entry point: pinned host text -> device -> "
                           "scan -> per-haystack results to pageable host arrays" % (n, hay_len)}
        del h_text_t
    peak, peak_src = measured_peaks()
    achieved = step_bytes / (k_ms * 1e-3) / 1e9
    roofline = {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak, "traffic": None,
                "kernel": "k_scan_machine_rk (%s)" % args.output, "kernel_ms": k_ms, "algorithmic_bytes_per_launch": step_bytes,
                "peak_source": peak_src,
                "note": "algorithmic bytes = 1 B read per haystack byte offered; kernel_ms = mean CUDA-event time of the scan kernel"}
    return {
        "metric": metric_name(W.spec) + ", " + args.output, "output": args.output, "value": value, "unit": UNIT, "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": wall_ms, "device_ms_per_step": dev_ms, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "config": {"workload": "%s: %s, %s, %d haystacks x %d B per step, %d batch(es) resident (%.2f GiB)" % (
                       args.config, W.spec["what"], W.mode_name, n, hay_len, len(batches), resident / 2**30),
                   "n_patterns": len(W.ps), "hay_len": hay_len, "bytes_per_gpu": step_bytes, "options": args.option,
                   "setup_s": setup_s},
        **extra, "roofline": roofline, "parity": parity, "e2e": e2e,
        "gpu_launches": int(launches2 - launches1), "launches_per_step": (launches2 - launches1) / args.steps, "clocks": clocks,
    }


def _card():
    import subprocess

    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        name, plim = [x.strip() for x in q.split(",")[:2]]
        return {"name": name, "power_limit": plim}
    except Exception:
        import torch

        return {"name": torch.cuda.get_device_name(0), "power_limit": None}


def run_hist_output(args, W, pma, batches, dmode, omode, n, hay_len, step_bytes, resident, dev, setup_s):
    """--output hist: every step is one dach_dev_hist_batch on the step's batch, added into one device histogram (the
    additive contract: a corpus accumulates).  The same run times the full matches scan + torch.bincount of its values
    and COUNT on the same batches, step by step, by CUDA events around whole steps."""
    import torch

    vals = pma.outputs()[0]
    n_hist = (int(vals.max()) + 1 if len(vals) else 0) if args.key == "value" else len(vals)
    hist_t = torch.zeros(n_hist, dtype=torch.int64, device=dev)
    counts_t = torch.empty(n, dtype=torch.int64, device=dev)
    r0 = pma.scan_batch_device(dmode, *batches[0])
    cap = int(max(r0.matches.shape[0], 1) * 1.25) + 1024
    del r0
    out_m = torch.empty((cap, 3), dtype=torch.int32, device=dev)
    out_o = torch.empty(n + 1, dtype=torch.int64, device=dev)

    def hist_step(s):
        t, o = batches[s % len(batches)]
        pma.pattern_counts_device(dmode, t, o, key=args.key, out=hist_t)
        st = pma.stats()
        return st["scan_kernel_ms"], st["total_ms"]

    def matches_step(s):
        t, o = batches[s % len(batches)]
        r = pma.scan_batch_device(dmode, t, o, out=out_m, out_offs=out_o)
        return torch.bincount(r.matches[:, 2].long(), minlength=n_hist)

    def count_step(s):
        t, o = batches[s % len(batches)]
        pma.count_batch_device(dmode, t, o, out=counts_t)

    def timed(fn):
        for s in range(args.warmup):
            fn(s)
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        res = [fn(args.warmup + s) for s in range(args.steps)]
        ev1.record()
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1) / args.steps, res

    sampler = ClockSampler(dev.index)
    sampler.start()
    time.sleep(0.2)
    n_before = len(sampler.rows)
    launches1 = pma.stats()["launches"]
    hist_ms, times = timed(hist_step)
    launches2 = pma.stats()["launches"]
    matches_ms, _ = timed(matches_step)
    count_ms, _ = timed(count_step)
    time.sleep(0.25)
    clocks = sampler.stop(skip=n_before)
    k_ms = float(np.mean([t[0] for t in times]))
    dev_ms = float(np.mean([t[1] for t in times]))
    value = step_bytes / (dev_ms * 1e-3) / 1e9
    gbs = lambda ms: step_bytes / (ms * 1e-3) / 1e9  # noqa: E731
    # the whole last step against the full scan of the same batch, bincounted on the device
    last_batch = (args.warmup + args.steps - 1) % len(batches)
    t_last, o_last = batches[last_batch]
    one = pma.pattern_counts_device(dmode, t_last, o_last, key=args.key)
    r = pma.scan_batch_device(dmode, t_last, o_last)
    full = torch.bincount(r.matches[:, 2].long(), minlength=int(vals.max()) + 1 if len(vals) else 0)
    if args.key == "output":
        full = full[torch.from_numpy(vals.astype(np.int64)).to(dev)]  # new(): one value per record
    step_ok = bool(torch.equal(one, full))
    total = int(one.sum().item())
    del r, full
    parity = None
    if not args.no_cpu:
        import oracle_api as O

        threads = O.cpu_budget()["threads"]
        ns = max(1, min(n, int(n * args.parity_frac)))
        opma = W.oracle()
        lo = W.batch_ranges()[last_batch][0]
        ptext, poffs = W.host_batch(lo, lo + ns)
        ref = opma.scan_batch(omode, ptext, poffs, nthreads=threads, want_matches=True)
        nv = int(vals.max()) + 1 if len(vals) else 0
        got = pma.pattern_counts_host(dmode, ptext, poffs, key="value")
        parity = hist_parity(got, ref["matches"]["value"], nv)
        parity.update({"haystacks_checked": ns, "share_of_batch": ns / n,
                       "what": "value-keyed histogram of the first %d haystacks of the last batch vs np.bincount of the "
                               "oracle's match values" % ns})
    parity = dict(parity or {}, step_equals_full_scan=step_ok)
    e2e = None
    if not args.no_e2e:
        t0_, o0_ = batches[0]
        h_text_t = torch.empty(t0_.numel(), dtype=torch.uint8).pin_memory()
        h_text_t.copy_(t0_)
        h_text = h_text_t.numpy()
        h_offs = o0_.cpu().numpy().astype(np.uint64)
        e2e_ms = []
        for i in range(1 + args.e2e_steps):
            t0 = time.perf_counter()
            pma.pattern_counts_host(dmode, h_text, h_offs, key=args.key)
            if i >= 1:
                e2e_ms.append((time.perf_counter() - t0) * 1e3)
        st = pma.stats()
        e2e = {"value": h_text.size / (np.mean(e2e_ms) * 1e-3) / 1e9, "unit": UNIT, "h2d_bytes_per_step": int(st["h2d_bytes"]),
               "d2h_bytes_per_step": int(st["d2h_bytes"]), "ms_per_step": float(np.mean(e2e_ms)),
               "workload": "the step batch's %d haystacks x %d B through the host entry point: pinned host text -> device -> "
                           "scan -> one histogram of %d x 8 B to the host" % (n, hay_len, n_hist)}
        del h_text_t
    peak, peak_src = measured_peaks()
    achieved = step_bytes / (k_ms * 1e-3) / 1e9
    roofline = {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak, "traffic": None,
                "kernel": "k_scan_machine_rk (hist)", "kernel_ms": k_ms, "algorithmic_bytes_per_launch": step_bytes,
                "peak_source": peak_src,
                "note": "algorithmic bytes = 1 B read per haystack byte offered; kernel_ms = mean CUDA-event time of the scan kernel"}
    return {
        "metric": metric_name(W.spec) + ", hist (%s key)" % args.key, "output": "hist", "key": args.key, "value": value, "unit": UNIT,
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": hist_ms, "device_ms_per_step": dev_ms,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "config": {"workload": "%s: %s, %s, %d haystacks x %d B per step, %d batch(es) resident (%.2f GiB)" % (
                       args.config, W.spec["what"], W.mode_name, n, hay_len, len(batches), resident / 2**30),
                   "n_patterns": len(W.ps), "hay_len": hay_len, "bytes_per_gpu": step_bytes, "options": args.option,
                   "setup_s": setup_s, "n_hist": n_hist},
        "total": total,
        "alternatives": {"unit": UNIT, "what": "CUDA events around %d whole steps each, same batches" % args.steps,
                         "hist": gbs(hist_ms), "matches_plus_bincount": gbs(matches_ms), "count": gbs(count_ms),
                         "hist_ms": hist_ms, "matches_plus_bincount_ms": matches_ms, "count_ms": count_ms},
        "card": _card(), "roofline": roofline, "parity": parity, "e2e": e2e,
        "gpu_launches": int(launches2 - launches1), "launches_per_step": (launches2 - launches1) / args.steps, "clocks": clocks,
    }


def run_stream_output(args, W, pma, batches, dmode, n, hay_len, step_bytes, resident, dev, setup_s):
    """--stream --output counts / hist: every step is one round of n streams -- the step's batch is the next chunk of
    each -- with the state tensor carried from step to step.  The same run plays the same rounds from the same start
    through scan_stream_device (stream positions, a preallocated output) and derives what the stream form returns from
    its matches; both are timed by CUDA events around whole steps.  Parity: per-stream counts summed over all rounds,
    the accumulated histogram and the carried state, stream form against the matches stream."""
    import torch

    if dmode not in (0, 1):
        raise SystemExit("--stream: the config's iterator has no stepper (find_iter / find_overlapping_iter only)")
    vals = pma.outputs()[0]
    n_hist = (int(vals.max()) + 1 if len(vals) else 0) if args.key == "value" else len(vals)
    value_of_record = torch.from_numpy(vals.astype(np.int64)).to(dev)
    rounds = args.warmup + args.steps
    pos = [torch.full((n,), (((s * hay_len) + 2**31) % 2**32) - 2**31, dtype=torch.int32, device=dev) for s in range(rounds)]  # u32 bits
    r0 = pma.scan_batch_device(dmode, *batches[0])
    cap = int(max(r0.matches.shape[0], 1) * 1.25) + 1024
    del r0
    out_m = torch.empty((cap, 3), dtype=torch.int32, device=dev)
    out_o = torch.empty(n + 1, dtype=torch.int64, device=dev)
    counts_t = torch.empty(n, dtype=torch.int64, device=dev)

    def play(fn):
        """all rounds from a fresh state; the timed window covers the last args.steps of them"""
        state = torch.zeros(n, dtype=torch.int32, device=dev)
        acc = torch.zeros(n if args.output == "counts" else n_hist, dtype=torch.int64, device=dev)
        for s in range(args.warmup):
            fn(s, state, acc)
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        res = [fn(args.warmup + s, state, acc) for s in range(args.steps)]
        ev1.record()
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1) / args.steps, res, state, acc

    def stream_step(s, state, acc):
        t, o = batches[s % len(batches)]
        if args.output == "counts":
            acc += pma.count_stream_device(dmode, t, o, state, out=counts_t)
        else:
            pma.pattern_counts_stream_device(dmode, t, o, state, key=args.key, out=acc)
        st = pma.stats()
        return st["scan_kernel_ms"], st["total_ms"]

    def matches_step(s, state, acc):
        t, o = batches[s % len(batches)]
        r = pma.scan_stream_device(dmode, t, o, state, pos[s], out=out_m, out_offs=out_o)
        if args.output == "counts":
            acc += torch.diff(r.offsets)
        else:
            h = torch.bincount(r.matches[:, 2].long(), minlength=int(vals.max()) + 1 if len(vals) else 0)
            acc += h if args.key == "value" else h[value_of_record]  # new(): one value per record

    sampler = ClockSampler(dev.index)
    sampler.start()
    time.sleep(0.2)
    n_before = len(sampler.rows)
    launches1 = pma.stats()["launches"]
    stream_ms, times, st_a, acc_a = play(stream_step)
    launches2 = pma.stats()["launches"]
    matches_ms, _, st_b, acc_b = play(matches_step)
    time.sleep(0.25)
    clocks = sampler.stop(skip=n_before)
    k_ms = float(np.mean([t[0] for t in times]))
    dev_ms = float(np.mean([t[1] for t in times]))
    gbs = lambda ms: step_bytes / (ms * 1e-3) / 1e9  # noqa: E731
    what = "counts" if args.output == "counts" else "hist"
    parity = {"%s_equal" % what: bool(torch.equal(acc_a, acc_b)), "state_equal": bool(torch.equal(st_a, st_b)),
              "total": int(acc_a.sum().item()), "rounds": rounds,
              "what": "stream form vs scan_stream_device over the same %d rounds from state 0: %s and the carried state" % (
                  rounds, "per-stream counts summed over the rounds" if what == "counts" else "the accumulated histogram")}
    return {
        "metric": metric_name(W.spec) + ", stream %s" % (what if what == "counts" else "hist (%s key)" % args.key),
        "output": args.output, "stream": True, "value": gbs(stream_ms), "unit": UNIT, "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": stream_ms, "device_ms_per_step": dev_ms, "scan_kernel_ms": k_ms,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "config": {"workload": "%s: %s, %s, %d streams, one %d B chunk each per step (the step's batch), %d batch(es) resident "
                               "(%.2f GiB)" % (args.config, W.spec["what"], W.mode_name, n, hay_len, len(batches), resident / 2**30),
                   "n_patterns": len(W.ps), "hay_len": hay_len, "bytes_per_gpu": step_bytes, "options": args.option,
                   "setup_s": setup_s},
        "alternatives": {"unit": UNIT, "what": "CUDA events around %d whole steps each, same rounds" % args.steps,
                         "stream_" + what: gbs(stream_ms), "scan_stream_plus_torch": gbs(matches_ms),
                         "stream_%s_ms" % what: stream_ms, "scan_stream_plus_torch_ms": matches_ms},
        "card": _card(), "parity": parity,
        "gpu_launches": int(launches2 - launches1), "launches_per_step": (launches2 - launches1) / rounds, "clocks": clocks,
    }


def run_df_output(args, W, pma, batches, dmode, omode, n, hay_len, step_bytes, resident, dev, setup_s):
    """--output df: every step is one dach_dev_df_batch on the step's batch, added into one device array.  The same run
    times the matches path + torch (haystack index per match, torch.unique of (haystack, key), bincount) and the
    histogram call on the same batches, step by step, by CUDA events around whole steps."""
    import torch

    vals = pma.outputs()[0]
    n_df = (int(vals.max()) + 1 if len(vals) else 0) if args.key == "value" else len(vals)
    df_t = torch.zeros(n_df, dtype=torch.int64, device=dev)
    hist_t = torch.zeros(n_df, dtype=torch.int64, device=dev)
    r0 = pma.scan_batch_device(dmode, *batches[0])
    cap = int(max(r0.matches.shape[0], 1) * 1.25) + 1024
    del r0
    out_m = torch.empty((cap, 3), dtype=torch.int32, device=dev)
    out_o = torch.empty(n + 1, dtype=torch.int64, device=dev)
    hay_ids = torch.arange(n, device=dev)
    key_of_value = torch.from_numpy(np.argsort(vals, kind="stable").astype(np.int64)).to(dev)  # new(): record of value v

    def df_step(s):
        t, o = batches[s % len(batches)]
        pma.doc_counts_device(dmode, t, o, key=args.key, out=df_t)
        st = pma.stats()
        return st["scan_kernel_ms"], st["total_ms"], pma.last_doc_windows()

    def matches_df(t, o):
        r = pma.scan_batch_device(dmode, t, o, out=out_m, out_offs=out_o)
        keys = r.matches[:, 2].long()
        if args.key == "output":
            keys = key_of_value[keys]
        hay = torch.repeat_interleave(hay_ids[: o.numel() - 1], torch.diff(r.offsets.long()))
        return torch.bincount(torch.unique(hay * n_df + keys) % n_df, minlength=n_df)

    def matches_step(s):
        return matches_df(*batches[s % len(batches)])

    def hist_step(s):
        t, o = batches[s % len(batches)]
        pma.pattern_counts_device(dmode, t, o, key=args.key, out=hist_t)

    def timed(fn):
        for s in range(args.warmup):
            fn(s)
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        res = [fn(args.warmup + s) for s in range(args.steps)]
        ev1.record()
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1) / args.steps, res

    sampler = ClockSampler(dev.index)
    sampler.start()
    time.sleep(0.2)
    n_before = len(sampler.rows)
    launches1 = pma.stats()["launches"]
    df_ms, times = timed(df_step)
    launches2 = pma.stats()["launches"]
    matches_ms, _ = timed(matches_step)
    hist_ms, _ = timed(hist_step)
    time.sleep(0.25)
    clocks = sampler.stop(skip=n_before)
    # a step is many windows, each timed inside the library; the step is timed by the events around it
    k_ms = float(np.mean([t[0] for t in times]))
    windows = [t[2] for t in times]
    gbs = lambda ms: step_bytes / (ms * 1e-3) / 1e9  # noqa: E731
    value = gbs(df_ms)
    # the whole last step against the matches path of the same batch, and the histogram invariants
    last_batch = (args.warmup + args.steps - 1) % len(batches)
    t_last, o_last = batches[last_batch]
    one = pma.doc_counts_device(dmode, t_last, o_last, key=args.key)
    step_ok = bool(torch.equal(one, matches_df(t_last, o_last)))
    h = pma.pattern_counts_device(dmode, t_last, o_last, key=args.key)
    vs_hist = {"df_le_hist": bool((one <= h).all()), "same_support": bool(torch.equal(one > 0, h > 0)),
               "df_le_n": bool(int(one.max()) <= n) if n_df else True}
    total = int(one.sum().item())
    parity = None
    if not args.no_cpu:
        import oracle_api as O

        threads = O.cpu_budget()["threads"]
        ns = max(1, min(n, int(n * args.parity_frac)))
        opma = W.oracle()
        lo = W.batch_ranges()[last_batch][0]
        ptext, poffs = W.host_batch(lo, lo + ns)
        ref = opma.scan_batch(omode, ptext, poffs, nthreads=threads, want_matches=True)
        nv = int(vals.max()) + 1 if len(vals) else 0
        got = pma.doc_counts_host(dmode, ptext, poffs, key="value")
        parity = df_parity(got, ref["counts"], ref["matches"]["value"], nv)
        parity.update({"haystacks_checked": ns, "share_of_batch": ns / n,
                       "what": "value-keyed document frequencies of the first %d haystacks of the last batch vs np.unique "
                               "of the oracle's (haystack, value) pairs" % ns})
    parity = dict(parity or {}, step_equals_matches_path=step_ok, **vs_hist)
    e2e = None
    if not args.no_e2e:
        t0_, o0_ = batches[0]
        h_text_t = torch.empty(t0_.numel(), dtype=torch.uint8).pin_memory()
        h_text_t.copy_(t0_)
        h_text = h_text_t.numpy()
        h_offs = o0_.cpu().numpy().astype(np.uint64)
        e2e_ms = []
        for i in range(1 + args.e2e_steps):
            t0 = time.perf_counter()
            pma.doc_counts_host(dmode, h_text, h_offs, key=args.key)
            if i >= 1:
                e2e_ms.append((time.perf_counter() - t0) * 1e3)
        st = pma.stats()
        e2e = {"value": h_text.size / (np.mean(e2e_ms) * 1e-3) / 1e9, "unit": UNIT, "h2d_bytes_per_step": int(st["h2d_bytes"]),
               "d2h_bytes_per_step": int(st["d2h_bytes"]), "ms_per_step": float(np.mean(e2e_ms)), "windows": pma.last_doc_windows(),
               "workload": "the step batch's %d haystacks x %d B through the host entry point: pinned host text -> device -> "
                           "scan -> %d x 8 B to the host" % (n, hay_len, n_df)}
        del h_text_t
    return {
        "metric": metric_name(W.spec) + ", df (%s key)" % args.key, "output": "df", "key": args.key, "value": value, "unit": UNIT,
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": df_ms,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "config": {"workload": "%s: %s, %s, %d haystacks x %d B per step, %d batch(es) resident (%.2f GiB)" % (
                       args.config, W.spec["what"], W.mode_name, n, hay_len, len(batches), resident / 2**30),
                   "n_patterns": len(W.ps), "hay_len": hay_len, "bytes_per_gpu": step_bytes, "options": args.option,
                   "setup_s": setup_s, "n_df": n_df},
        "total": total, "last_window_scan_kernel_ms": k_ms,
        "windows_per_step": float(np.mean([w[0] for w in windows])), "rescans_per_step": float(np.mean([w[1] for w in windows])),
        "alternatives": {"unit": UNIT, "what": "CUDA events around %d whole steps each, same batches" % args.steps,
                         "df": gbs(df_ms), "matches_plus_torch_unique": gbs(matches_ms), "hist": gbs(hist_ms),
                         "df_ms": df_ms, "matches_plus_torch_unique_ms": matches_ms, "hist_ms": hist_ms},
        "card": _card(), "parity": parity, "e2e": e2e,
        "gpu_launches": int(launches2 - launches1), "launches_per_step": (launches2 - launches1) / args.steps, "clocks": clocks,
    }


def torch_span_fill(pma, dmode, t, o, fill, out, slice_haystacks, cap):
    """The matches path plus torch: every slice of `slice_haystacks` haystacks scanned into a match list, its spans
    turned into a byte mask (a difference array and a cumsum) and filled into `out`, a copy of the text."""
    import torch

    out.copy_(t)
    n = o.numel() - 1
    out_m = torch.empty((cap, 3), dtype=torch.int32, device=t.device)
    for a in range(0, n, slice_haystacks):
        b = min(n, a + slice_haystacks)
        lo, hi = int(o[a]), int(o[b])
        os_ = o[a:b + 1] - lo
        r = pma.scan_batch_device(dmode, t[lo:hi], os_, out=out_m)
        m = r.matches.long()
        hay = torch.repeat_interleave(torch.arange(b - a, device=t.device), torch.diff(r.offsets))
        s, e = os_[hay] + m[:, 0], os_[hay] + m[:, 1]
        d = torch.zeros(hi - lo + 1, dtype=torch.int32, device=t.device)
        d.index_add_(0, s, torch.ones_like(s, dtype=torch.int32))
        d.index_add_(0, e, torch.full_like(e, -1, dtype=torch.int32))
        out[lo:hi].masked_fill_(torch.cumsum(d[:-1], 0) > 0, fill)
    return out


def run_mask_output(args, W, pma, batches, dmode, omode, n, hay_len, step_bytes, resident, dev, setup_s):
    """--output mask: every step is one dach_dev_mask_batch on the step's batch.  The same run times, by CUDA events
    around whole steps on the same batches: COUNT (the same scan without the stores), the copy kernel alone (a mask call
    with no haystack), and the matches path plus a torch span fill in slices of --alt-mib."""
    import torch

    fill = args.fill
    masked = torch.empty(step_bytes, dtype=torch.uint8, device=dev)
    alt = torch.empty(step_bytes, dtype=torch.uint8, device=dev)
    counts_t = torch.empty(n, dtype=torch.int64, device=dev)
    slice_h = max(1, (args.alt_mib << 20) // hay_len)
    t0_, o0_ = batches[0]
    r0 = pma.scan_batch_device(dmode, t0_[: int(o0_[min(n, slice_h)])], o0_[: min(n, slice_h) + 1])
    cap = int(max(r0.matches.shape[0], 1) * 1.25) + 1024
    del r0

    def mask_step(s):
        t, o = batches[s % len(batches)]
        pma.mask_batch_device(dmode, t, o, fill=fill, out=masked[: t.numel()])
        st = pma.stats()
        return st["scan_kernel_ms"], st["total_ms"]

    def count_step(s):
        t, o = batches[s % len(batches)]
        pma.count_batch_device(dmode, t, o, out=counts_t)

    def copy_step(s):
        t, o = batches[s % len(batches)]
        pma.mask_batch_device(dmode, t, o[:1], fill=fill, out=masked[: t.numel()])

    def torch_step(s):
        t, o = batches[s % len(batches)]
        torch_span_fill(pma, dmode, t, o, fill, alt[: t.numel()], slice_h, cap)

    def timed(fn):
        """ms per step over args.steps steps after args.warmup, the steps' results, and the kernels they launched"""
        for s in range(args.warmup):
            fn(s)
        torch.cuda.synchronize()
        l0 = pma.stats()["launches"]
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        res = [fn(args.warmup + s) for s in range(args.steps)]
        ev1.record()
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1) / args.steps, res, pma.stats()["launches"] - l0

    sampler = ClockSampler(dev.index)
    sampler.start()
    time.sleep(0.2)
    n_before = len(sampler.rows)
    mask_ms, times, launches = timed(mask_step)
    count_ms, _, _ = timed(count_step)
    copy_ms, _, _ = timed(copy_step)
    torch_ms, _, _ = timed(torch_step)
    time.sleep(0.25)
    clocks = sampler.stop(skip=n_before)
    k_ms = float(np.mean([t[0] for t in times]))
    dev_ms = float(np.mean([t[1] for t in times]))
    gbs = lambda ms: step_bytes / (ms * 1e-3) / 1e9  # noqa: E731
    # the whole last step against the torch span fill of the same batch
    last_batch = (args.warmup + args.steps - 1) % len(batches)
    t_last, o_last = batches[last_batch]
    one = pma.mask_batch_device(dmode, t_last, o_last, fill=fill, out=masked[: t_last.numel()])
    ref = torch_span_fill(pma, dmode, t_last, o_last, fill, alt[: t_last.numel()], slice_h, cap)
    step_ok = bool(torch.equal(one, ref))
    masked_bytes = int((one != t_last).sum().item())
    parity = None
    if not args.no_cpu:
        import oracle_api as O
        import emu_mask_api as EM

        threads = O.cpu_budget()["threads"]
        ns = max(1, min(n, int(n * args.parity_frac)))
        opma = W.oracle()
        lo = W.batch_ranges()[last_batch][0]
        ptext, poffs = W.host_batch(lo, lo + ns)
        r = opma.scan_batch(omode, ptext, poffs, nthreads=threads, want_matches=True)
        want = EM.expected_from_matches(ptext, poffs, r["matches"], r["counts"], fill)
        got = pma.mask_batch_host(dmode, ptext, poffs, fill=fill)
        parity = {"mask_equal": bool(np.array_equal(got, want)), "haystacks_checked": ns, "share_of_batch": ns / n,
                  "what": "host mask of the first %d haystacks of the last batch vs the oracle's matches turned into spans" % ns}
    parity = dict(parity or {}, step_equals_torch_span_fill=step_ok)
    peak, peak_src = measured_peaks()
    achieved = step_bytes / (k_ms * 1e-3) / 1e9
    roofline = {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak, "traffic": None,
                "kernel": "k_scan_machine_rk (mask)", "kernel_ms": k_ms, "algorithmic_bytes_per_launch": step_bytes,
                "peak_source": peak_src,
                "note": "algorithmic bytes = 1 B read per haystack byte offered; kernel_ms = mean CUDA-event time of the scan kernel"}
    return {
        "metric": metric_name(W.spec) + ", mask", "output": "mask", "value": gbs(dev_ms), "unit": UNIT,
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": mask_ms, "device_ms_per_step": dev_ms,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "config": {"workload": "%s: %s, %s, %d haystacks x %d B per step, %d batch(es) resident (%.2f GiB)" % (
                       args.config, W.spec["what"], W.mode_name, n, hay_len, len(batches), resident / 2**30),
                   "n_patterns": len(W.ps), "hay_len": hay_len, "bytes_per_gpu": step_bytes, "options": args.option,
                   "setup_s": setup_s, "fill": fill, "alt_mib": args.alt_mib},
        "masked_bytes_last_step": masked_bytes,
        "alternatives": {"unit": UNIT, "what": "CUDA events around %d whole steps each, same batches" % args.steps,
                         "mask": gbs(mask_ms), "count": gbs(count_ms), "copy_only": gbs(copy_ms),
                         "matches_plus_torch_fill": gbs(torch_ms), "mask_ms": mask_ms, "count_ms": count_ms,
                         "copy_ms": copy_ms, "matches_plus_torch_fill_ms": torch_ms},
        "card": _card(), "roofline": roofline, "parity": parity,
        "gpu_launches": int(launches), "launches_per_step": launches / args.steps, "clocks": clocks,
    }


def device_batches(W, dev):
    """The workload's batches on the device as bench.py makes them: [(text, offs)], and the bytes of text resident."""
    import torch

    from daachorse_b200 import synth as S

    hay_len = W.hay_len
    pool_t = torch.from_numpy(W.pool).to(dev)
    starts_t = torch.from_numpy(W.starts).to(dev)
    ranges = W.batch_ranges()
    if "window" in W.spec:
        text_all, offs_all = S.materialise_on_device(pool_t, starts_t, hay_len)
        return [(text_all[lo * hay_len: hi * hay_len], offs_all[: hi - lo + 1]) for lo, hi in ranges], text_all.numel()
    batches = []
    for lo, hi in ranges:
        t, o = S.materialise_on_device(pool_t, starts_t[lo:hi], hay_len)
        if W.spec["synth"] == "C4":
            S.pad_to_char_boundary_device(t, hi - lo, hay_len)
        batches.append((t, o))
    return batches, sum(b[0].numel() for b in batches)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--output", required=True, choices=["counts", "first", "hist", "df", "mask"])
    ap.add_argument("--fill", type=int, default=ord("*"), help="--output mask: the fill byte")
    ap.add_argument("--alt-mib", type=int, default=256, help="--output mask: slice of the matches-plus-torch baseline")
    ap.add_argument("--stream", action="store_true", help="--output counts / hist on stream chunks: one round per step")
    ap.add_argument("--key", default="value", choices=["value", "output"], help="--output hist / df: key")
    ap.add_argument("--config", default="C3", choices=sorted(CONFIGS))
    ap.add_argument("--steps", type=int, default=None)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the config's batch (debug only)")
    ap.add_argument("--pool-mib", type=int, default=None)
    ap.add_argument("--e2e-steps", type=int, default=3)
    ap.add_argument("--parity-frac", type=float, default=0.04, help="share of a batch checked against the oracle")
    ap.add_argument("--option", action="append", default=[], help="kernel option name=value")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-cpu", action="store_true", help="no oracle parity")
    args = ap.parse_args()
    if args.steps is None:
        args.steps = CONFIGS[args.config]["steps"]
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if args.stream and args.output not in ("counts", "hist"):
        ap.error("--stream takes --output counts or hist")

    import torch

    assert torch.cuda.is_available(), "bench_reduce.py needs a CUDA device (no CPU fallback)"
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    t_setup = time.time()
    W = Workload(args.config, args.scale, 0, args.pool_mib)
    dmode, omode = mode_ids(W.mode_name)
    hay_len = W.hay_len
    pma = W.automaton()
    for kv in args.option:
        k, v = kv.split("=")
        pma.set_option(k, int(v))
    batches, resident = device_batches(W, dev)
    n = W.window
    torch.cuda.synchronize()
    line = run_reduce_output(args, W, pma, batches, dmode, omode, n, hay_len, n * hay_len, resident, dev, t_setup)
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
