#!/usr/bin/env python3
"""tools/bench_jobs_rk.py -- COUNT and HIST as a two-job pipeline against one synchronous call per step, one H100:

    python tools/bench_jobs_rk.py [--config C2|C3] [--output counts|hist] [--steps K] [--warmup W] [--repeats R]

The batches, automata and seeds are those of bench.py and tools/bench_reduce.py (find_overlapping on C2 and C3).  Both
forms run the same steps on the same batches, one output buffer per step parity (s mod 2):
  sync      one dach_dev_count_batch / dach_dev_hist_batch per step (the call synchronises its stream; HIST: the step's
            histogram is zeroed on that stream first)
  pipeline  two jobs on two streams, in bench.py's run_pipeline order: step s+1 is enqueued (dach_job_count /
            dach_job_hist) before step s is waited for (dach_job_wait); HIST zeroes the step's histogram on its job's
            stream first
GB/s = bytes offered per step x steps / host wall time between two device synchronisations, per form; the forms
alternate --repeats times in one run, and the line reports every repeat.  Parity: after the timed runs, both forms run
once more and every step's counts or histogram and its total are compared, pipeline against sync.  One JSON line, with
the card's name and power limit.  Nothing is written to the tree.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench import CONFIGS, Workload, mode_ids, run_pipeline  # noqa: E402
from bench_reduce import _card, device_batches  # noqa: E402


def make_forms(pma, dmode, batches, output, dev):
    """(sync_step, job_enqueue, job_finish, outs): the step callbacks of both forms and their two output buffers.  The
    synchronous step calls the C ABI directly, as the job wrappers do, so that both forms report the call's total."""
    import ctypes as C

    import torch

    from daachorse_b200 import _lib
    from daachorse_b200.automaton import HIST_KEYS

    L = _lib.load()
    n = batches[0][1].numel() - 1
    if output == "counts":
        outs = [torch.empty(n, dtype=torch.int64, device=dev) for _ in range(2)]
    else:
        outs = [torch.zeros(pma._hist_len("value"), dtype=torch.int64, device=dev) for _ in range(2)]
    jobs = [pma.job(dev.index) for _ in range(2)]
    streams = [torch.cuda.Stream(dev) for _ in range(2)]

    def batch(s):
        return batches[s % len(batches)]

    def sync_step(s):
        t, o = batch(s)
        d = pma.device_handle(dev.index)
        tot = C.c_uint64()
        st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        out = outs[s % 2]
        if output == "counts":
            rc = L.dach_dev_count_batch(d, dmode, C.c_void_p(t.data_ptr()), C.c_void_p(o.data_ptr()), o.numel() - 1, t.numel(),
                                        C.c_void_p(out.data_ptr()), C.byref(tot), st)
        else:
            out.zero_()
            rc = L.dach_dev_hist_batch(d, dmode, HIST_KEYS["value"], C.c_void_p(t.data_ptr()), C.c_void_p(o.data_ptr()),
                                       o.numel() - 1, t.numel(), C.c_void_p(out.data_ptr()), out.numel(), C.byref(tot), st)
        assert rc == _lib.OK, _lib.last_error()
        return tot.value

    def job_enqueue(s):
        t, o = batch(s)
        job, st = jobs[s % 2], streams[s % 2]
        if output == "counts":
            job.count(dmode, t, o, out=outs[s % 2], stream=st)
        else:
            with torch.cuda.stream(st):
                outs[s % 2].zero_()
            job.pattern_counts(dmode, t, o, out=outs[s % 2], stream=st)

    def job_finish(s):
        return jobs[s % 2].wait()

    for st in streams:
        st.wait_stream(torch.cuda.current_stream(dev))
    return sync_step, job_enqueue, job_finish, outs


def run_sync(sync_step, steps, on_step=None):
    for s in range(steps):
        tot = sync_step(s)
        if on_step:
            on_step(s, tot)


def run_jobs(job_enqueue, job_finish, steps, on_step=None):
    def finish(s):
        tot = job_finish(s)
        if on_step:
            on_step(s, tot)
        return tot

    run_pipeline(steps, 2, job_enqueue, lambda s: None, finish)


def timed(fn, dev):
    import torch

    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize(dev)
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3", choices=["C2", "C3"])
    ap.add_argument("--output", default="counts", choices=["counts", "hist"])
    ap.add_argument("--steps", type=int, default=None)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3, help="timed runs of each form, alternating")
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the config's batch (debug only)")
    args = ap.parse_args()
    if args.steps is None:
        args.steps = CONFIGS[args.config]["steps"]
    if args.steps < 2:
        ap.error("--steps must be at least 2 (a pipeline of one step has nothing to overlap)")

    import torch

    assert torch.cuda.is_available(), "bench_jobs_rk.py needs a CUDA device (no CPU fallback)"
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    W = Workload(args.config, args.scale, 0, None)
    dmode, _ = mode_ids(W.mode_name)
    pma = W.automaton()
    batches, _ = device_batches(W, dev)
    step_bytes = W.window * W.hay_len
    torch.cuda.synchronize()
    sync_step, job_enqueue, job_finish, outs = make_forms(pma, dmode, batches, args.output, dev)

    run_sync(sync_step, args.warmup)
    run_jobs(job_enqueue, job_finish, args.warmup)
    gbs = lambda sec: step_bytes * args.steps / sec / 1e9  # noqa: E731
    sync_gbs, pipe_gbs = [], []
    for _ in range(args.repeats):
        sync_gbs.append(gbs(timed(lambda: run_sync(sync_step, args.steps), dev)))
        pipe_gbs.append(gbs(timed(lambda: run_jobs(job_enqueue, job_finish, args.steps), dev)))

    # parity: the same steps once more, every step's output and total, pipeline against sync
    ref = {}

    def keep_sync(s, tot):
        ref[s] = (outs[s % 2].clone(), tot)

    def check_job(s, tot):
        want, wtot = ref[s]
        parity.append(bool(torch.equal(outs[s % 2], want)) and tot == wtot)

    run_sync(sync_step, args.steps, keep_sync)
    torch.cuda.synchronize()
    parity = []
    run_jobs(job_enqueue, job_finish, args.steps, check_job)
    line = {
        "config": args.config, "mode": W.mode_name, "output": args.output, "steps": args.steps, "warmup": args.warmup,
        "step_mib": round(step_bytes / 2**20, 1), "unit": "GB/s",
        "sync": [round(x, 2) for x in sync_gbs], "pipeline": [round(x, 2) for x in pipe_gbs],
        "pipeline_over_sync": round(float(sum(pipe_gbs) / sum(sync_gbs)), 4),
        "parity_steps": parity, "parity": all(parity) and len(parity) == args.steps,
        "total_last_step": ref[args.steps - 1][1], "card": _card(),
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
