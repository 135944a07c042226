#!/usr/bin/env python3
"""A compact pass over every kernel for compute-sanitizer (memcheck / racecheck / initcheck are 10-100x slower than
native, so this is a subset of tests/test_gpu_parity.py that still launches every kernel the library has):

    compute-sanitizer --tool memcheck  --error-exitcode 1 python tools/sanitize.py
    compute-sanitizer --tool racecheck --error-exitcode 1 python tools/sanitize.py

Golden vectors (all iterators x bytewise / charwise), random batches on every kernel option, text buffers at odd
addresses and with no slack after the last byte (the 8-byte text loads must not touch anything outside), stream
chunks, event blocks with output lists of 255 and more (stored at the landing and through the event queue; k_expand in
pool and output order), counts and first matches, per-pattern histograms (both keys, shared-memory counters on and off), document frequencies (both keys, the smallest pair table), asynchronous jobs (the matches and the four
reductions), a two-rank shard group on one device.  Every result is checked against the oracle."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import daachorse_b200 as D
import emu_mask_api as EM
import oracle_api as O
from daachorse_b200 import shard

GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "search_tests.json"), encoding="utf-8"))
MODE = {"find_iter": D.FIND, "find_overlapping_iter": D.FIND_OVERLAPPING,
        "find_overlapping_no_suffix_iter": D.FIND_OVERLAPPING_NO_SUFFIX, "leftmost_find_iter": D.LEFTMOST_FIND}
ORC = {D.FIND: O.FIND, D.FIND_OVERLAPPING: O.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX: O.FIND_OVERLAPPING_NO_SUFFIX,
       D.LEFTMOST_FIND: O.LEFTMOST_FIND}
KIND = {"Standard": 0, "LeftmostLongest": 1, "LeftmostFirst": 2}
n_scans = 0


def golden():
    global n_scans
    for variant, iterator, coll, kind in GOLD["configs"]:
        if iterator not in MODE:
            continue
        cw = variant == "charwise"
        B = D.CharwiseDoubleArrayAhoCorasickBuilder if cw else D.DoubleArrayAhoCorasickBuilder
        for g in GOLD["collections"][coll]:
            for t in GOLD["groups"][g][::3]:
                pma = B.new().match_kind(KIND[kind]).build(t["patterns"])
                got = [(m.value(), m.start(), m.end()) for m in getattr(pma, iterator)(t["haystack"])]
                assert got == [tuple(x) for x in t["matches"]], t["name"]
                n_scans += 1


def random_case(seed, cw, kind):
    rng = np.random.default_rng(seed)
    table = ["a", "b", "é", "あ", "𝄞", "z"]
    pats = sorted({"".join(table[int(i)] for i in rng.integers(0, 4, size=int(rng.integers(1, 6)))) for _ in range(60)})
    hays = ["".join(table[int(i)] for i in rng.integers(0, 5, size=int(rng.integers(0, 300)))).encode() for _ in range(96)]
    if not cw:
        pats = [p.encode() for p in pats]
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    text = np.frombuffer(b"".join(hays), dtype=np.uint8)
    B = D.CharwiseDoubleArrayAhoCorasickBuilder if cw else D.DoubleArrayAhoCorasickBuilder
    return B.new().match_kind(kind).build(pats), O.OraclePma.build(pats, charwise=cw, match_kind=kind), text, offs


def random_batches():
    global n_scans
    dev = torch.device("cuda", 0)
    for cw in (False, True):
        for kind in (0, 1):
            pma, opma, text, offs = random_case(10 * kind + cw, cw, kind)
            for mode in ([D.LEFTMOST_FIND] if kind else [D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX]):
                ref = opma.scan_batch(ORC[mode], text, offs, want_matches=True)
                for opts in ({"kernel": 3}, {"kernel": 3, "event_queue": 1}, {"kernel": 4}, {"kernel": 3, "hot_entries": 512}, {"kernel": 2},
                             {"kernel": 1}, {"kernel": 0}, {"kernel": 3, "seg_len": 64}, {"kernel": 4, "threads": 256}):
                    for k, v in opts.items():
                        pma.set_option(k, v)
                    r = pma.scan_batch_host(mode, text, offs)
                    assert r.matches.tobytes() == ref["matches"].tobytes(), (cw, kind, mode, opts)
                    n_scans += 1
                    pma.set_option("seg_len", 0)
                    pma.set_option("hot_entries", 0)
                    pma.set_option("threads", 1024)
                    pma.set_option("event_queue", 0)
                pma.set_option("kernel", 3)
                # device-resident text at an odd address, the last haystack ending exactly at the end of the allocation
                pad = 3
                buf = torch.empty(text.size + pad, dtype=torch.uint8, device=dev)
                buf[pad:] = torch.from_numpy(text.copy()).to(dev)
                r = pma.scan_batch_device(mode, buf[pad:], torch.from_numpy(offs.astype(np.int64)).to(dev))
                m = r.matches.cpu().numpy().astype(np.uint32)
                assert m.tobytes() == ref["matches"].tobytes(), ("odd address", cw, kind, mode)
                n_scans += 1


def event_blocks():
    """StdMachine3's event blocks with lists too long for the length byte, placed by k_expand in pool order and in
    output order, whole and in segments."""
    global n_scans
    pats = [b"a" * k for k in range(1, 301)] + [b"ba"]
    hays = [b"a" * 400, b"xa" + b"a" * 260 + b"b" + b"a" * 300, b"", b"ba" * 40] * 8
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    text = np.frombuffer(b"".join(hays), dtype=np.uint8)
    pma, opma = D.DoubleArrayAhoCorasick.new(pats), O.OraclePma.build(pats)
    for mode in (D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX):
        ref = opma.scan_batch(ORC[mode], text, offs, want_matches=True)
        for opts in ({"gather_ordered": 0}, {"gather_ordered": 2}, {"gather_ordered": 2, "seg_len": 64}, {"event_queue": 1},
                     {"event_queue": 1, "seg_len": 64}, {"gather_ordered": 2, "expand_desc": 0},
                     {"gather_ordered": 2, "expand_u": 8}):
            for k, v in opts.items():
                pma.set_option(k, v)
            r = pma.scan_batch_host(mode, text, offs)
            assert r.matches.tobytes() == ref["matches"].tobytes(), (mode, opts)
            n_scans += 1
            pma.set_option("seg_len", 0)
            pma.set_option("event_queue", 0)
            pma.set_option("expand_desc", 1)
            pma.set_option("expand_u", 2)
        pma.set_option("gather_ordered", 1)


def counts_and_first():
    """dach_count_batch_host / dach_first_batch_host on every kernel that serves them, the device forms on text at an
    odd address; against the oracle's per-haystack runs."""
    global n_scans
    dev = torch.device("cuda", 0)
    for cw in (False, True):
        for kind in (0, 1):
            pma, opma, text, offs = random_case(20 + 10 * kind + cw, cw, kind)
            for mode in ([D.LEFTMOST_FIND] if kind else [D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX]):
                ref = opma.scan_batch(ORC[mode], text, offs, want_matches=True)
                counts = ref["counts"].astype(np.uint64)
                starts = np.concatenate([[0], np.cumsum(counts)])[:-1].astype(np.int64)
                found = counts > 0
                for opts in ({"kernel": 3}, {"kernel": 3, "hot_entries": 512}, {"kernel": 0}, {"kernel": 3, "seg_len": 64}):
                    for k, v in opts.items():
                        pma.set_option(k, v)
                    c, _ = pma.count_batch_host(mode, text, offs)
                    f, fd = pma.first_batch_host(mode, text, offs)
                    assert np.array_equal(c, counts) and np.array_equal(fd, found), (cw, kind, mode, opts)
                    assert f[fd].tobytes() == ref["matches"][starts[found]].tobytes(), (cw, kind, mode, opts)
                    n_scans += 2
                    pma.set_option("seg_len", 0)
                    pma.set_option("hot_entries", 0)
                pma.set_option("kernel", 3)
                pad = 3
                buf = torch.empty(text.size + pad, dtype=torch.uint8, device=dev)
                buf[pad:] = torch.from_numpy(text.copy()).to(dev)
                o = torch.from_numpy(offs.astype(np.int64)).to(dev)
                assert np.array_equal(pma.count_batch_device(mode, buf[pad:], o).cpu().numpy().astype(np.uint64), counts)
                assert np.array_equal(pma.first_batch_device(mode, buf[pad:], o)[1].cpu().numpy(), found)
                n_scans += 2


def histograms():
    """dach_hist_batch_host / dach_dev_hist_batch, both keys, with the shared-memory counters on and off, on every kernel
    that serves them; against np.bincount of the oracle's match values."""
    global n_scans
    dev = torch.device("cuda", 0)
    for cw in (False, True):
        for kind in (0, 1):
            pma, opma, text, offs = random_case(40 + 10 * kind + cw, cw, kind)
            vals = pma.outputs()[0].astype(np.int64)
            for mode in ([D.LEFTMOST_FIND] if kind else [D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX]):
                ref = opma.scan_batch(ORC[mode], text, offs, want_matches=True)
                want = np.bincount(ref["matches"]["value"].astype(np.int64), minlength=int(vals.max()) + 1).astype(np.uint64)
                for opts in ({"kernel": 3, "hist_smem": 1024}, {"kernel": 3, "hist_smem": 0}, {"kernel": 3, "hist_smem": 64, "seg_len": 64},
                             {"kernel": 0}):
                    for k, v in opts.items():
                        pma.set_option(k, v)
                    assert np.array_equal(pma.pattern_counts_host(mode, text, offs), want), (cw, kind, mode, opts)
                    assert np.array_equal(pma.pattern_counts_host(mode, text, offs, key="output"), want[vals]), (cw, kind, mode, opts)
                    n_scans += 2
                    pma.set_option("seg_len", 0)
                pma.set_option("kernel", 3)
                pma.set_option("hist_smem", 1024)
                pad = 3
                buf = torch.empty(text.size + pad, dtype=torch.uint8, device=dev)
                buf[pad:] = torch.from_numpy(text.copy()).to(dev)
                o = torch.from_numpy(offs.astype(np.int64)).to(dev)
                assert np.array_equal(pma.pattern_counts_device(mode, buf[pad:], o).cpu().numpy().astype(np.uint64), want)
                n_scans += 1


def doc_frequencies():
    """dach_df_batch_host / dach_dev_df_batch, both keys, on every kernel that serves them, with the default pair table
    and the smallest (every window overflows until it is small enough); against np.unique of the oracle's (haystack,
    value) pairs."""
    global n_scans
    dev = torch.device("cuda", 0)
    for cw in (False, True):
        for kind in (0, 1):
            pma, opma, text, offs = random_case(60 + 10 * kind + cw, cw, kind)
            vals = pma.outputs()[0].astype(np.int64)
            for mode in ([D.LEFTMOST_FIND] if kind else [D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX]):
                ref = opma.scan_batch(ORC[mode], text, offs, want_matches=True)
                hay = np.repeat(np.arange(len(offs) - 1, dtype=np.uint64), ref["counts"].astype(np.int64))
                pairs = np.unique((hay << np.uint64(32)) | ref["matches"]["value"].astype(np.uint64))
                want = np.bincount((pairs & np.uint64(0xffffffff)).astype(np.int64), minlength=int(vals.max()) + 1).astype(np.uint64)
                for opts in ({"kernel": 3}, {"kernel": 3, "seg_len": 64}, {"kernel": 3, "df_pairs": 1}, {"kernel": 0, "df_pairs": 1},
                             {"kernel": 0}):
                    for k, v in opts.items():
                        pma.set_option(k, v)
                    assert np.array_equal(pma.doc_counts_host(mode, text, offs), want), (cw, kind, mode, opts)
                    assert np.array_equal(pma.doc_counts_host(mode, text, offs, key="output"), want[vals]), (cw, kind, mode, opts)
                    n_scans += 2
                    pma.set_option("seg_len", 0)
                    pma.set_option("df_pairs", 1 << 24)
                pma.set_option("kernel", 3)
                pad = 3
                buf = torch.empty(text.size + pad, dtype=torch.uint8, device=dev)
                buf[pad:] = torch.from_numpy(text.copy()).to(dev)
                o = torch.from_numpy(offs.astype(np.int64)).to(dev)
                assert np.array_equal(pma.doc_counts_device(mode, buf[pad:], o).cpu().numpy().astype(np.uint64), want)
                n_scans += 1


def masked_text():
    """dach_mask_batch_host / dach_dev_mask_batch on every machine that serves them (StdMachine3 with and without
    segments, LmMachine, CwMachine, the lane-per-haystack loops); against the oracle's matches turned into spans, and
    the device form's output at an odd offset from its text."""
    global n_scans
    dev = torch.device("cuda", 0)
    for cw in (False, True):
        for kind in (0, 1):
            pma, opma, text, offs = random_case(80 + 10 * kind + cw, cw, kind)
            for mode in ([D.LEFTMOST_FIND] if kind else [D.FIND, D.FIND_OVERLAPPING, D.FIND_OVERLAPPING_NO_SUFFIX]):
                ref = opma.scan_batch(ORC[mode], text, offs, want_matches=True)
                want = EM.expected_from_matches(text, offs, ref["matches"], ref["counts"], 0x2A)
                for opts in ({"kernel": 3}, {"kernel": 3, "seg_len": 64}, {"kernel": 0}):
                    for k, v in opts.items():
                        pma.set_option(k, v)
                    assert np.array_equal(pma.mask_batch_host(mode, text, offs), want), (cw, kind, mode, opts)
                    n_scans += 1
                    pma.set_option("seg_len", 0)
                pma.set_option("kernel", 3)
                pad = 3
                buf = torch.empty(text.size + pad, dtype=torch.uint8, device=dev)
                buf[pad:] = torch.from_numpy(text.copy()).to(dev)
                out = torch.empty(text.size + 7, dtype=torch.uint8, device=dev)
                o = torch.from_numpy(offs.astype(np.int64)).to(dev)
                pma.mask_batch_device(mode, buf[pad:], o, out=out[7:])
                assert np.array_equal(out[7:].cpu().numpy(), want)
                n_scans += 1


def job_reductions():
    """dach_job_count / _first / _hist / _mask, one compact case each on two jobs and two streams (StdMachine3 in
    segments and the lane-per-haystack loops); against the oracle."""
    global n_scans
    dev = torch.device("cuda", 0)
    pma, opma, text, offs = random_case(90, False, 0)
    mode = D.FIND_OVERLAPPING
    ref = opma.scan_batch(ORC[mode], text, offs, want_matches=True)
    counts = ref["counts"].astype(np.int64)
    found = counts > 0
    starts = np.concatenate([[0], np.cumsum(counts)])[:-1]
    vals = pma.outputs()[0].astype(np.int64)
    hist = np.bincount(ref["matches"]["value"].astype(np.int64), minlength=int(vals.max()) + 1)
    mask = EM.expected_from_matches(text, offs, ref["matches"], ref["counts"], 0x2A)
    t = torch.from_numpy(text.copy()).to(dev)
    o = torch.from_numpy(offs.astype(np.int64)).to(dev)
    jobs = [pma.job(0), pma.job(0)]
    sts = [torch.cuda.Stream(dev), torch.cuda.Stream(dev)]
    torch.cuda.synchronize()
    for opts in ({"kernel": 3, "seg_len": 64}, {"kernel": 0}):
        for k, v in opts.items():
            pma.set_option(k, v)
        for i, (job, st) in enumerate(zip(jobs, sts)):
            c = job.count(mode, t, o, stream=st)
            assert job.wait() == int(counts.sum()) and np.array_equal(c.cpu().numpy(), counts), opts
            f, fd = job.first(mode, t, o, stream=st)
            assert job.wait() == int(found.sum()) and np.array_equal(fd.cpu().numpy(), found), opts
            assert f.cpu().numpy().astype(np.uint32)[found].tobytes() == ref["matches"][starts[found]].tobytes(), opts
            h = job.pattern_counts(mode, t, o, key="value" if i == 0 else "output", stream=st)
            assert job.wait() == len(ref["matches"]), opts
            assert np.array_equal(h.cpu().numpy(), hist if i == 0 else hist[vals]), opts
            m = job.mask(mode, t, o, fill=0x2A, stream=st)
            assert job.wait() == 0 and np.array_equal(m.cpu().numpy(), mask), opts
            n_scans += 4
        pma.set_option("seg_len", 0)
    pma.set_option("kernel", 3)


def streams_jobs_groups():
    global n_scans
    dev = torch.device("cuda", 0)
    pma, opma, text, offs = random_case(77, False, 0)
    t = torch.from_numpy(text.copy()).to(dev)
    o = torch.from_numpy(offs.astype(np.int64)).to(dev)
    n = len(offs) - 1
    whole = pma.scan_batch_device(D.FIND_OVERLAPPING, t, o)
    # stream chunks: two rounds, the matches call and the count / first / histogram calls on states of their own
    state, s_count, s_first, s_hist = (torch.zeros(n, dtype=torch.int32, device=dev) for _ in range(4))
    hist = torch.zeros(pma._hist_len("value"), dtype=torch.int64, device=dev)
    half = (offs[:-1] + (offs[1:] - offs[:-1]) // 2).astype(np.int64)
    for lo, hi in ((offs[:-1].astype(np.int64), half), (half, offs[1:].astype(np.int64))):
        lens = hi - lo
        co = np.zeros(n + 1, dtype=np.int64)
        co[1:] = np.cumsum(lens)
        ct = np.concatenate([text[int(a): int(b)] for a, b in zip(lo, hi)]) if co[-1] else np.zeros(0, np.uint8)
        tt = torch.from_numpy(ct.copy()).to(dev) if len(ct) else torch.zeros(16, dtype=torch.uint8, device=dev)[:0]
        cot = torch.from_numpy(co).to(dev)
        pos = torch.from_numpy(lo.astype(np.int32)).to(dev)
        r = pma.scan_stream_device(D.FIND_OVERLAPPING, tt, cot, state, pos)
        counts = pma.count_stream_device(D.FIND_OVERLAPPING, tt, cot, s_count)
        first, found = pma.first_stream_device(D.FIND_OVERLAPPING, tt, cot, s_first, pos=pos)
        pma.pattern_counts_stream_device(D.FIND_OVERLAPPING, tt, cot, s_hist, out=hist)
        assert torch.equal(counts, r.offsets[1:] - r.offsets[:-1])
        assert torch.equal(found, counts > 0) and torch.equal(first[found], r.matches[r.offsets[:-1][found]])
        n_scans += 4
    for s in (s_count, s_first, s_hist):
        assert torch.equal(s, state)
    for i in range(0, n, 7):
        assert int(state[i].item()) == opma.state_after(text[int(offs[i]): int(offs[i + 1])].tobytes())
    # jobs on two streams
    jobs = [pma.job(0), pma.job(0)]
    sts = [torch.cuda.Stream(dev), torch.cuda.Stream(dev)]
    outs = [torch.zeros((whole.matches.shape[0] + 3, 3), dtype=torch.int32, device=dev) for _ in range(2)]
    oos = [torch.zeros(n + 1, dtype=torch.int64, device=dev) for _ in range(2)]
    torch.cuda.synchronize()
    for k in range(2):
        jobs[k].scan(D.FIND_OVERLAPPING, t, o, outs[k].shape[0], stream=sts[k])
        jobs[k].place(outs[k], oos[k], stream=sts[1 - k])
    for k in range(2):
        assert jobs[k].wait() == whole.matches.shape[0]
        assert torch.equal(outs[k][: whole.matches.shape[0]], whole.matches) and torch.equal(oos[k], whole.offsets)
        n_scans += 1
    # a two-rank shard group on one device
    bounds = shard.byte_balanced_ranges(offs, 2)
    cap = int(whole.matches.shape[0]) + 16
    groups = [shard.PeerGroup(r, 2, 0, cap, n, exchange=None) for r in range(2)]
    for g in groups:
        g.connect([x.handle for x in groups])
    for step in range(2):
        for r in (0, 1):  # the sanitizer serialises kernels: a rank that waits for a lower rank must be issued after it
            lo, hi = bounds[r], bounds[r + 1]
            tt = t[int(offs[lo]): int(offs[hi])]
            oo = (o[lo: hi + 1] - o[lo]).contiguous()
            jobs[r].scan(D.FIND_OVERLAPPING, tt, oo, cap, stream=sts[r])
            groups[r].place(jobs[r], lo, r == 1, stream=sts[r])
        groups[1].finish(stream=sts[1])
        total = groups[0].finish(stream=sts[0])
        m, oo = groups[0].result(total)
        assert total == whole.matches.shape[0] and torch.equal(m, whole.matches) and torch.equal(oo, whole.offsets)
        n_scans += 2
    for g in groups:
        g.close()


if __name__ == "__main__":
    golden()
    random_batches()
    event_blocks()
    counts_and_first()
    histograms()
    doc_frequencies()
    masked_text()
    job_reductions()
    streams_jobs_groups()
    torch.cuda.synchronize()
    print("sanitize.py: %d scans, all equal to the oracle" % n_scans)
