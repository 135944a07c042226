"""Standalone time of the placement of one scanned batch (enqueue_place: k_expand or k_expand_desc, k_final_offsets).

    python tools/bench_place.py [--configs C3,C3-find,C2] [--repeats 20] [--json OUT]

For each config of bench.py (its first batch, at its shape) and each placement (option expand_desc 0 = k_expand
over the block map, 1 = block descriptors and two-entry lists), one job scans the batch once; then the job is placed
`repeats` times into the same buffers, each placement between two CUDA events on its own.  A placement only reads
the job's pool, so placing it again places the same thing.  Bytes: the event blocks read (256 B per block, counted
as ceil(events / 30) per haystack -- a lower bound, segments add partial blocks) plus the 12-byte tuples written.
The two placements' results are compared byte for byte.  Prints one JSON line per (config, placement).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi unavailable: %s" % e


def events_of(matches, offsets):
    """distinct (haystack, end) pairs of a match list: one event each"""
    import torch

    m = matches.shape[0]
    if m == 0:
        return 0, 0
    ends = matches[:, 1]
    new = torch.ones(m, dtype=torch.bool, device=matches.device)
    new[1:] = ends[1:] != ends[:-1]
    starts = offsets[:-1][offsets[:-1] < m]
    new[starts] = True
    ev_at = torch.cumsum(new.to(torch.int64), 0)
    # events per haystack: ev_at at its last match minus ev_at before its first
    lo, hi = offsets[:-1], offsets[1:]
    has = hi > lo
    before = torch.where(lo > 0, ev_at[(lo - 1).clamp(min=0)], torch.zeros_like(lo))
    per = torch.where(has, ev_at[(hi - 1).clamp(min=0)] - before, torch.zeros_like(lo))
    blocks = int(((per + 29) // 30).sum())
    return int(ev_at[-1]), blocks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C3,C3-find,C2")
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import torch

    import bench as B
    import daachorse_b200 as D
    from daachorse_b200 import synth as S

    assert torch.cuda.is_available(), "bench_place.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    rows = []
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name in args.configs.split(","):
        W = B.Workload(name, 1.0, 0)
        dmode, _ = B.mode_ids(W.mode_name)
        pma = W.automaton()
        lo, hi = W.batch_ranges()[0]
        t, o = S.materialise_on_device(torch.from_numpy(W.pool).to(dev), torch.from_numpy(W.starts[lo:hi]).to(dev), W.hay_len)
        ref = pma.scan_batch_device(dmode, t, o)
        total = int(ref.matches.shape[0])
        n_ev, n_blk = events_of(ref.matches, ref.offsets)
        cap = total + 4096
        out_m = torch.zeros((cap, 3), dtype=torch.int32, device=dev)
        out_o = torch.zeros(o.numel(), dtype=torch.int64, device=dev)
        st = torch.cuda.Stream(dev)
        results = {}
        for desc in (0, 1):
            pma.set_option("expand_desc", desc)
            job = pma.job(0)
            torch.cuda.synchronize()
            job.scan(dmode, t, o, cap, stream=st)
            job.place(out_m, out_o, stream=st)
            assert job.wait() == total
            results[desc] = (out_m[:total].clone(), out_o.clone())
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.repeats)]
            for a, b in ev:
                a.record(st)
                job.place(out_m, out_o, stream=st)
                b.record(st)
                job.wait()
            ms = sorted(a.elapsed_time(b) for a, b in ev)
            med = ms[len(ms) // 2]
            nbytes = 256 * n_blk + 12 * total
            row = {"config": name, "expand_desc": desc, "matches": total, "events": n_ev, "blocks_min": n_blk,
                   "place_ms_median": round(med, 3), "place_ms_min": round(ms[0], 3), "place_ms_max": round(ms[-1], 3),
                   "gbs": round(nbytes / (med * 1e-3) / 1e9, 1), "bytes": nbytes}
            rows.append(row)
            print(json.dumps(row), flush=True)
            del job
        same = torch.equal(results[0][0], results[1][0]) and torch.equal(results[0][1], results[1][1])
        same_ref = torch.equal(results[1][0], ref.matches) and torch.equal(results[1][1], ref.offsets)
        print(json.dumps({"config": name, "identical": bool(same), "identical_to_scan_batch": bool(same_ref)}), flush=True)
        pma.set_option("expand_desc", 1)
        del pma, t, o, ref, out_m, out_o, results
        torch.cuda.empty_cache()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
