"""Every scan path at the edges of the automaton, against the oracle on the same patterns and bytes:

  A  double-array layouts: num_free_blocks 1, 2, 3, 16 and 64 (more vacant slots whose CHECK bytes the compact image
     must keep), bytewise and charwise, every match kind, the NUL-heavy set and a C2-sized dictionary;
  B  hot-region sizes of the compact image (DACH_HOT_SLOTS at upload): none, one block, 4096, the default and 2^22
     slots, with stream state ids carried across chunk cuts in the renumbered and in the crate's numbering;
  C  values across u32: 0, 1, 2^24 - 1, 2^24, 2^31, 0xFFFFFFFE and 0xFFFFFFFF, duplicate patterns and lists of two
     or more, the KEY_VALUE refusal and FIRST at a real match of value 0xFFFFFFFF;
  D  the 2^24 edge of the compact image (build_image in dev_image.cpp): a relaid-out image whose new ids reach
     2^24 - 1, the largest compact image (2^24 slots, no hot region), the smallest automaton without one (every
     batch call on the lane-per-haystack kernels, every stream call refused), and the charwise comparison n < 2^24.

"All result kinds": scan_batch_host and scan_batch_device, COUNT, FIRST, HIST and DF under both keys, mask; for
Standard automata the four stream forms on ragged chunks, final states equal to the crate's."""
import gc
import resource

import numpy as np
import pytest

import daachorse_b200 as D
import emu_mask_api as EM
import oracle_api as O
from cases import filler_case, layout_cases, layout_params, mixed_width_case, nul_heavy_case
from daachorse_b200 import _lib
from daachorse_b200 import synth as S
from test_gpu_df import doc_freq
from test_gpu_stream_rk import rounds, stepper_matches

pytestmark = pytest.mark.gpu
ORC = {0: O.FIND, 1: O.FIND_OVERLAPPING, 2: O.FIND_OVERLAPPING_NO_SUFFIX, 3: O.LEFTMOST_FIND}
DEFAULTS = {"kernel": 3, "hot_entries": -2, "event_queue": 0, "expand_desc": 1, "gather_ordered": 1, "seg_len": 0}
# one option off its default at a time; gather_ordered 2 forces the ordered placement, where expand_desc applies
STD_MACHINES = ([{}] + [{"kernel": k} for k in (0, 1, 2, 4)] + [{"hot_entries": 0}, {"event_queue": 1},
                {"gather_ordered": 2, "expand_desc": 0}, {"gather_ordered": 2, "expand_desc": 1},
                {"gather_ordered": 2, "event_queue": 1}, {"seg_len": 64}])
LANE_MACHINES = [{}, {"kernel": 0}, {"kernel": 1}]
FILL = ord("*")
S32, S64 = 0x5A5A5A5A, 0x5A5A5A5A5A5A5A5A
G24 = 1 << 24


def _torch():
    import torch

    return torch


def _cuda(a, dtype=None):
    torch = _torch()
    a = np.ascontiguousarray(a)
    if a.size == 0:
        return torch.zeros(16, dtype=dtype or torch.uint8, device="cuda")[:0]
    return torch.from_numpy(a).cuda()


def _u32(t):
    return t.cpu().numpy().view(np.uint32).reshape(-1, 3)


def _release():
    torch = _torch()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


class Case:
    """One automaton in the product and in the oracle, built from the same patterns, values and layout."""

    def __init__(self, pats, cw=False, kind=0, nfb=16, values=None):
        self.cw, self.kind = cw, kind
        B = D.CharwiseDoubleArrayAhoCorasickBuilder if cw else D.DoubleArrayAhoCorasickBuilder
        b = B.new().match_kind(kind).num_free_blocks(nfb)
        self.pma = b.build(pats) if values is None else b.build_with_values(list(zip(pats, values)))
        self.opma = O.OraclePma.build(pats, charwise=cw, match_kind=kind, num_free_blocks=nfb, values=values)
        self.n = self.pma.num_elements()
        assert self.n == self.opma.num_elements()
        self.modes = (3,) if kind else (0, 1, 2)
        self.machines = STD_MACHINES if (not cw and not kind) else LANE_MACHINES
        vals, lens, _ = self.pma.outputs()
        keys = (vals.astype(np.int64) << 32) | lens.astype(np.int64)
        assert len(np.unique(keys)) == len(keys), "the output key is derived from (value, length): keep them unique"
        self.known = np.sort(keys)
        self.rec = np.argsort(keys, kind="stable")
        self.n_out, self.max_val = len(vals), int(vals.max())

    def configure(self, opts):
        for k, v in DEFAULTS.items():
            self.pma.set_option(k, opts.get(k, v))

    def oracle(self, mode, text, offs):
        ref = self.opma.scan_batch(ORC[mode], np.ascontiguousarray(text), offs, want_matches=True)
        return ref["matches"], np.concatenate([[0], np.cumsum(ref["counts"].astype(np.int64))]).astype(np.int64)

    def rec_of(self, m):
        """Output record of every match (start, end, value)."""
        k = (m["value"].astype(np.int64) << 32) | (m["end"].astype(np.int64) - m["start"].astype(np.int64))
        at = np.searchsorted(self.known, k)
        assert np.array_equal(self.known[np.minimum(at, len(self.known) - 1)], k)
        return self.rec[at]

    def keyed(self, want):
        """(key, bins, key of every match); KEY_VALUE only where a histogram of max value + 1 bins is affordable."""
        out = [("output", self.n_out, self.rec_of(want))]
        if self.max_val <= G24:
            out.append(("value", self.max_val + 1, want["value"].astype(np.int64)))
        return out


def check_batch(c, text, offs, tag, machines=None, reductions=True):
    """Matches on every machine of `c` (device, sentinel-filled output with slack; host once), then COUNT, FIRST,
    HIST and DF (both keys, added into pre-filled buffers) and mask on every machine that serves them."""
    torch = _torch()
    machines = c.machines if machines is None else machines
    t, o = _cuda(text), _cuda(offs.astype(np.int64))
    n = len(offs) - 1
    for mode in c.modes:
        want, wo = c.oracle(mode, text, offs)
        total = int(wo[-1])
        counts = np.diff(wo)
        has = counts > 0
        r = c.pma.scan_batch_host(mode, text, offs)
        assert r.matches.tobytes() == want.tobytes() and np.array_equal(r.offsets.astype(np.int64), wo), (tag, mode, "host")
        keyed = c.keyed(want)
        want_mask = EM.expected_from_matches(text, offs, want, counts, FILL)
        for opts in machines:
            if opts.get("seg_len") and mode not in (1, 2):
                continue
            c.configure(opts)
            out = torch.full((total + 64, 3), S32, dtype=torch.int32, device="cuda")
            oo = torch.full((n + 17,), S64, dtype=torch.int64, device="cuda")
            r = c.pma.scan_batch_device(mode, t, o, out=out, out_offs=oo)
            assert r.matches.shape[0] == total, (tag, mode, opts)
            assert _u32(out[:total]).tobytes() == want.view(np.uint32).tobytes(), (tag, mode, opts)
            assert bool((out[total:] == S32).all()), (tag, mode, opts, "d_out written past needed")
            assert np.array_equal(oo[: n + 1].cpu().numpy(), wo), (tag, mode, opts)
            if not reductions or "event_queue" in opts or "gather_ordered" in opts:
                continue  # placement options: the reductions have no placement
            assert np.array_equal(c.pma.count_batch_device(mode, t, o).cpu().numpy(), counts), (tag, mode, opts)
            first, found = c.pma.first_batch_device(mode, t, o)
            assert np.array_equal(found.cpu().numpy(), has), (tag, mode, opts)
            assert _u32(first)[has].tobytes() == want[wo[:-1][has]].view(np.uint32).tobytes(), (tag, mode, opts)
            assert (_u32(first)[~has] == 0xFFFFFFFF).all(), (tag, mode, opts)
            for key, k, keys in keyed:
                for name, call, ref in (("hist", c.pma.pattern_counts_device, np.bincount(keys, minlength=k)),
                                        ("df", c.pma.doc_counts_device, doc_freq(counts, keys, k).astype(np.int64))):
                    pre = torch.arange(1, k + 9, dtype=torch.int64, device="cuda") * 1000
                    got = (call(mode, t, o, key=key, out=pre.clone()) - pre).cpu().numpy()
                    assert np.array_equal(got[:k], ref), (tag, mode, opts, name, key)
                    assert not got[k:].any(), (tag, mode, opts, name, key, "written past the key range")
            masked = c.pma.mask_batch_device(mode, t, o, fill=FILL)
            assert np.array_equal(masked.cpu().numpy(), want_mask), (tag, mode, opts, "mask")
        c.configure({})
        if reductions:  # the host forms once, on the default machine
            assert np.array_equal(c.pma.count_batch_host(mode, text, offs)[0], counts), (tag, mode)
            f, g = c.pma.first_batch_host(mode, text, offs)
            assert np.array_equal(g, has) and f[has].tobytes() == want[wo[:-1][has]].tobytes(), (tag, mode)
            for key, k, keys in keyed:
                assert np.array_equal(c.pma.pattern_counts_host(mode, text, offs, key=key), np.bincount(keys, minlength=k)), (tag, mode, key)
                assert np.array_equal(c.pma.doc_counts_host(mode, text, offs, key=key), doc_freq(counts, keys, k)), (tag, mode, key)
            assert np.array_equal(c.pma.mask_batch_host(mode, text, offs, fill=FILL), want_mask), (tag, mode)


def _hays(text, offs):
    return [np.ascontiguousarray(text[int(offs[i]): int(offs[i + 1])]) for i in range(len(offs) - 1)]


def _char_cuts(s):
    return np.concatenate([np.flatnonzero((s & 0xC0) != 0x80), [len(s)]]).astype(np.int64)


def check_streams(c, streams, tag, step=700, seed=1):
    """The four stream forms on ragged chunks of `streams`, each with its own state tensor: matches equal the oracle
    stepper over each whole stream, COUNT / FIRST / HIST equal each round's matches, the states stay equal and end
    where the crate's automaton does (bytewise: OraclePma.state_after)."""
    torch = _torch()
    cuts = [_char_cuts(s) if c.cw else np.arange(len(s) + 1) for s in streams]
    n = len(streams)
    for mode in (D.FIND, D.FIND_OVERLAPPING):
        want = stepper_matches(c.opma, mode, streams)
        st = {k: torch.zeros(n, dtype=torch.int32, device="cuda") for k in ("matches", "count", "first", "hist")}
        hist = torch.zeros(c.n_out, dtype=torch.int64, device="cuda")
        got = [[] for _ in streams]
        for r, (text, offs, starts) in enumerate(rounds(streams, cuts, step, seed)):
            t, o, p = _cuda(text), _cuda(offs), _cuda(starts.view(np.int32))
            m = c.pma.scan_stream_device(mode, t, o, st["matches"], p)
            mm, oo = _u32(m.matches), m.offsets.cpu().numpy()
            for i in range(n):
                got[i].append(mm[oo[i]: oo[i + 1]])
            assert np.array_equal(c.pma.count_stream_device(mode, t, o, st["count"]).cpu().numpy(), np.diff(oo)), (tag, mode, r)
            first, found = c.pma.first_stream_device(mode, t, o, st["first"], pos=p)
            has = np.diff(oo) > 0
            assert np.array_equal(found.cpu().numpy(), has), (tag, mode, r)
            assert np.array_equal(_u32(first)[has], mm[oo[:-1][has]]), (tag, mode, r)
            c.pma.pattern_counts_stream_device(mode, t, o, st["hist"], key="output", out=hist)
            for k in ("count", "first", "hist"):
                assert torch.equal(st[k], st["matches"]), (tag, mode, r, k)
        all_want = np.concatenate(want)
        for i in range(n):
            assert np.concatenate(got[i]).tobytes() == want[i].tobytes(), (tag, mode, i)
        w = np.zeros(len(all_want), dtype=O.MATCH_DTYPE)
        w["start"], w["end"], w["value"] = all_want[:, 0], all_want[:, 1], all_want[:, 2]
        assert np.array_equal(hist.cpu().numpy(), np.bincount(c.rec_of(w), minlength=c.n_out)), (tag, mode)
        if not c.cw:
            final = st["matches"].cpu().numpy().view(np.uint32)
            for i, s in enumerate(streams):
                assert int(final[i]) == c.opma.state_after(s.tobytes(), find_mode=mode == D.FIND), (tag, mode, i)


def check_streams_refused(c, text, offs):
    """An automaton without a compact image has no stream form: every stream call returns DACH_INVALID_ARGUMENT and
    leaves the state and every output buffer as it was."""
    torch = _torch()
    t, o = _cuda(text), _cuda(offs.astype(np.int64))
    n = len(offs) - 1
    for mode in (D.FIND, D.FIND_OVERLAPPING):
        state = torch.full((n,), 5, dtype=torch.int32, device="cuda")
        out = torch.full((64, 3), S32, dtype=torch.int32, device="cuda")
        oo = torch.full((n + 1,), S64, dtype=torch.int64, device="cuda")
        cnt = torch.full((n,), S64, dtype=torch.int64, device="cuda")
        first = torch.full((n, 3), S32, dtype=torch.int32, device="cuda")
        found = torch.full((n,), 0x5A, dtype=torch.uint8, device="cuda")
        hist = torch.arange(c.n_out, dtype=torch.int64, device="cuda") + 7
        calls = (lambda: c.pma.scan_stream_device(mode, t, o, state, out=out, out_offs=oo),
                 lambda: c.pma.count_stream_device(mode, t, o, state, out=cnt),
                 lambda: c.pma.first_stream_device(mode, t, o, state, out=first, found=found),
                 lambda: c.pma.pattern_counts_stream_device(mode, t, o, state, key="output", out=hist))
        for i, call in enumerate(calls):
            with pytest.raises(D.DaachorseError) as e:
                call()
            assert e.value.code == _lib.INVALID_ARGUMENT, (mode, i)
        torch.cuda.synchronize()
        assert bool((state == 5).all()), "a refused stream call moved the state"
        assert bool((out == S32).all()) and bool((oo == S64).all()) and bool((cnt == S64).all())
        assert bool((first == S32).all()) and bool((found == 0x5A).all())
        assert torch.equal(hist, torch.arange(c.n_out, dtype=torch.int64, device="cuda") + 7)


# ---- A: double-array layouts ------------------------------------------------------------------------------------------
def _cjk_patterns():
    return [p.decode() for p in S.make_patterns(S.config("C4"), n=5000).as_list()]


LAYOUT_CASES = layout_cases()


@pytest.mark.parametrize("case,nfb", layout_params(LAYOUT_CASES),
                         ids=["%s-nfb%d" % (LAYOUT_CASES[i][0], k) for i, k in layout_params(LAYOUT_CASES)])
def test_a_layouts(case, nfb):
    name, pats, cw, kind, text, offs = LAYOUT_CASES[case]
    c = Case(pats, cw, kind, nfb)
    if nfb != 16:
        ref = Case(pats, cw, kind, 16)
        assert c.opma.serialize() != ref.opma.serialize(), (name, nfb, "the layout equals the 16-block one")
        assert c.pma.serialize() == c.opma.serialize(), (name, nfb)
        if nfb == 1 and not cw:  # the charwise arrays keep their size and move states
            assert c.n > ref.n, (name, nfb, "no more slots than with 16 free blocks")
    check_batch(c, text, offs, (name, nfb))
    if not kind:
        hays = _hays(text, offs)[:200]
        check_streams(c, hays, (name, nfb), step=300)


# ---- B: hot-region sizes ------------------------------------------------------------------------------------------------
def _hot_cases():
    out = []
    pats, text, offs = nul_heavy_case(0, n_patterns=20000, n_hay=300)
    out.append(("nul-heavy", pats, False, text, offs))
    cfg = S.config("C3")
    ps = S.make_patterns(cfg, n=20000)
    pool, _ = S.make_pool(cfg, ps, 1 << 20)
    rng = np.random.default_rng(23)
    lens = rng.integers(0, 3000, size=300)
    lens[::17] = 0
    starts = rng.integers(0, len(pool) - 3000, size=300)
    hays = [pool[int(s): int(s) + int(n)].tobytes() for s, n in zip(starts, lens)]
    offs = np.concatenate([[0], np.cumsum([len(h) for h in hays])]).astype(np.uint64)
    out.append(("c3-20000", ps.as_list(), False, np.frombuffer(b"".join(hays), dtype=np.uint8).copy(), offs))
    _, cpats, ctext, coffs = mixed_width_case(9)
    out.append(("charwise-mixed", list(cpats) + _cjk_patterns()[:2000], True, ctext, coffs))
    return out


HOT_CASES = _hot_cases()
HOT_SIZES = [0, 256, 4096, 65536, 1 << 22]


@pytest.mark.parametrize("case", range(len(HOT_CASES)), ids=[c[0] for c in HOT_CASES])
def test_b_hot_region_sizes(case, monkeypatch):
    name, pats, cw, text, offs = HOT_CASES[case]
    sizes = {}
    for hs in HOT_SIZES:
        monkeypatch.setenv("DACH_HOT_SLOTS", str(hs))
        c = Case(pats, cw, 0)  # a fresh automaton: the variable is read when the image is uploaded
        sizes[hs] = c.pma.stats()["image_bytes"]
        monkeypatch.delenv("DACH_HOT_SLOTS")
        check_batch(c, text, offs, (name, hs))
        check_streams(c, _hays(text, offs)[:150], (name, hs), step=250)
        n = c.n
        del c
    print(name, "image bytes per hot-region size:", sizes)
    if cw:  # the charwise image has no hot region
        assert len(set(sizes.values())) == 1
    else:
        # per slot of the region: 16 bytes of records, 4 of output positions and 4 of ids; the region is at most the
        # automaton rounded up to whole 256-slot blocks
        assert sizes[0] < sizes[256] < sizes[4096]
        grow = sorted(sizes.items())
        for (h0, b0), (h1, b1) in zip(grow, grow[1:]):
            top = (n + 255) & ~255
            assert b1 - b0 == 24 * (min(h1, top) - min(h0, top)), (h0, h1, b0, b1)


# ---- C: values across u32 -----------------------------------------------------------------------------------------------
SPECIAL = [0, 1, G24 - 1, G24, 1 << 31, 0xFFFFFFFE, 0xFFFFFFFF]
SMALL = {1 << 31: 2, 0xFFFFFFFE: G24 - 2, 0xFFFFFFFF: 3}  # the values above 2^24, replaced one for one


def _value_case(cw, seed=0):
    """Patterns of group g have length g + 1 and take the special values in turn, so (value, length) names an output
    record; the first two of every group are the same pattern (duplicates with distinct values), and the groups are
    suffixes of each other, so that lists of two and more occur.  Charwise symbols are all two bytes long."""
    rng = np.random.default_rng(300 + seed)
    sym = ["é", "ß"] if cw else [b"a", b"b"]
    pats, vals = [], []
    for g in range(10):
        row = [rng.integers(0, 2, size=g + 1) for _ in SPECIAL]
        row[1] = row[0]
        for i, r in enumerate(row):
            pats.append(("" if cw else b"").join(sym[int(x)] for x in r))
            vals.append(SPECIAL[(i + g) % len(SPECIAL)])
    hays = [("" if cw else b"").join(sym[int(x)] for x in rng.integers(0, 2, size=int(rng.integers(0, 60)))) for _ in range(200)]
    hays += ["z" * 5 if cw else b"zzzzz", "" if cw else b""]
    hb = [h.encode() if cw else h for h in hays]
    offs = np.concatenate([[0], np.cumsum([len(h) for h in hb])]).astype(np.uint64)
    return pats, vals, np.frombuffer(b"".join(hb), dtype=np.uint8).copy(), offs


@pytest.mark.parametrize("cw", [False, True], ids=["bytewise", "charwise"])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_c_values_across_u32(cw, kind):
    pats, vals, text, offs = _value_case(cw)
    c = Case(pats, cw, kind, values=vals)
    assert c.max_val == 0xFFFFFFFF
    check_batch(c, text, offs, ("values", cw, kind))
    if not kind:
        check_streams(c, _hays(text, offs), ("values", cw), step=20)


@pytest.mark.parametrize("cw", [False, True], ids=["bytewise", "charwise"])
def test_c_value_key_up_to_2_pow_24(cw):
    """KEY_VALUE with a histogram of 2^24 + 1 bins: values 0, 1, 2^24 - 1 and 2^24 in their own bins."""
    pats, vals, text, offs = _value_case(cw, seed=1)
    vals = [SMALL.get(v, v) for v in vals]
    c = Case(pats, cw, 0, values=vals)
    assert c.max_val == G24 and len(c.keyed(c.oracle(1, text, offs)[0])) == 2
    check_batch(c, text, offs, ("value key", cw), machines=[{}, {"kernel": 0}])


def test_c_value_key_refused_when_the_histogram_is_short():
    """n_hist <= max value: dach_dev_hist_batch / dach_dev_df_batch with KEY_VALUE refuse before anything runs and
    leave the caller's buffer as it was (the Python forms size their own buffer, so the C ABI is called directly)."""
    import ctypes as C

    torch = _torch()
    pats, vals, text, offs = _value_case(False, seed=1)
    vals = [SMALL.get(v, v) for v in vals]
    c = Case(pats, False, 0, values=vals)
    L = _lib.load()
    d = c.pma.device_handle(0)
    t, o = _cuda(text), _cuda(offs.astype(np.int64))
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    total = C.c_uint64()
    for fn in (L.dach_dev_hist_batch, L.dach_dev_df_batch):
        for k in (G24, 1000):
            prior = torch.arange(k, dtype=torch.int64, device="cuda") * 3 + 1
            h = prior.clone()
            rc = fn(d, 1, 1, C.c_void_p(t.data_ptr()), C.c_void_p(o.data_ptr()), len(offs) - 1, t.numel(), C.c_void_p(h.data_ptr()),
                    k, C.byref(total), st)
            torch.cuda.synchronize()
            assert rc == _lib.INVALID_ARGUMENT and torch.equal(h, prior), (fn, k)
        for key, k in ((1, G24 + 1), (0, c.n_out)):  # the exact sizes are accepted
            h = torch.zeros(k, dtype=torch.int64, device="cuda")
            assert fn(d, 1, key, C.c_void_p(t.data_ptr()), C.c_void_p(o.data_ptr()), len(offs) - 1, t.numel(), C.c_void_p(h.data_ptr()),
                      k, C.byref(total), st) == 0
    for fn in (L.dach_hist_batch_host, L.dach_df_batch_host):
        h = np.arange(1000, dtype=np.uint64) + 5
        rc = fn(d, 1, 1, C.c_void_p(text.ctypes.data), C.c_void_p(offs.ctypes.data), len(offs) - 1, C.c_void_p(h.ctypes.data), 1000,
                C.byref(total))
        assert rc == _lib.INVALID_ARGUMENT and np.array_equal(h, np.arange(1000, dtype=np.uint64) + 5), fn


@pytest.mark.parametrize("cw", [False, True], ids=["bytewise", "charwise"])
def test_c_first_match_of_value_all_ones(cw):
    """A real first match (0, 1, 0xFFFFFFFF) has the same bits as "no match": only `found` tells them apart."""
    torch = _torch()
    pat = "é" if cw else b"q"
    c = Case([pat, ("ßß" if cw else b"rr")], cw, 0, values=[0xFFFFFFFF, 7])
    hays = [(pat.encode() if cw else pat), b"", b"zz", (pat.encode() if cw else pat) * 3]
    text = np.frombuffer(b"".join(hays), dtype=np.uint8).copy()
    offs = np.concatenate([[0], np.cumsum([len(h) for h in hays])]).astype(np.uint64)
    w = len(hays[0])
    for opts in c.machines:
        c.configure(opts)
        for mode in c.modes:
            f, g = c.pma.first_batch_device(mode, _cuda(text), _cuda(offs.astype(np.int64)))
            assert g.cpu().numpy().tolist() == [True, False, False, True], (mode, opts)
            assert _u32(f).tolist() == [[0, w, 0xFFFFFFFF]] + [[0xFFFFFFFF] * 3] * 2 + [[0, w, 0xFFFFFFFF]], (mode, opts)
    c.configure({})
    f, g = c.pma.first_batch_host(0, text, offs)
    assert g.tolist() == [True, False, False, True] and int(f[0]["value"]) == 0xFFFFFFFF
    state = torch.zeros(len(hays), dtype=torch.int32, device="cuda")
    f, g = c.pma.first_stream_device(0, _cuda(text), _cuda(offs.astype(np.int64)), state)
    assert g.cpu().numpy().tolist() == [True, False, False, True]
    assert _u32(f)[0].tolist() == [0, w, 0xFFFFFFFF]


# ---- D: the 2^24 edge -------------------------------------------------------------------------------------------------
def _peak_rss_gib():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20


def _image_regime(c):
    """'wide' (no compact image), 'compact' or 'hot' (compact with a hot region of H slots), from image_bytes:
    wide records 16 n, outputs and pair table 32 per record, the ROOT row 1024; the bytewise compact image adds 24 N + 4 n
    for N = n + H compact slots (records, output positions, both id maps), the charwise one 20 n and the mapper."""
    b = c.pma.stats()["image_bytes"]
    rest = b - 16 * c.n - 32 * c.n_out - 1024
    if c.cw:
        if rest >= 20 * c.n:
            assert rest - 20 * c.n < 4 * 0x110000
            return "compact", 0
        assert 0 <= rest < 4 * 0x110000
        return "wide", 0
    if rest == 0:
        return "wide", 0
    H = (rest - 4 * c.n) // 24 - c.n
    assert 24 * (c.n + H) + 4 * c.n == rest, (b, c.n)
    return ("hot" if H else "compact"), H


EDGE = [  # (id, slots, charwise, kind, regime, hot slots)
    ("bytewise-a", G24 - 65536, False, 0, "hot", 65536),
    ("bytewise-b", G24, False, 0, "compact", 0),
    ("bytewise-c", G24 + 256, False, 0, "wide", 0),
    ("charwise-compact", G24 - 256, True, 0, "compact", 0),
    ("charwise-wide", G24, True, 0, "wide", 0),
    ("leftmost-b", G24, False, 1, "compact", 0),
]


@pytest.fixture(scope="module", params=EDGE, ids=[e[0] for e in EDGE])
def edge(request):
    name, slots, cw, kind, regime, H = request.param
    pats, text, offs = filler_case(slots, cw, kind)
    c = Case(pats, cw, kind)
    del pats
    assert c.n == slots, (name, c.n)
    c.pma.device_handle(0)
    print("%s: %d slots, peak host RSS %.2f GiB after building both automata and the image" % (name, c.n, _peak_rss_gib()))
    yield name, c, text, offs, regime, H
    c.pma = c.opma = None
    _release()


def test_d_slots_and_regime(edge):
    name, c, text, offs, regime, H = edge
    assert _image_regime(c) == (regime, H), name


def test_d_every_result_kind(edge):
    name, c, text, offs, regime, H = edge
    machines = c.machines if regime != "wide" else [{}, {"kernel": 0}]
    check_batch(c, text, offs, name, machines=machines)


def test_d_streams(edge):
    name, c, text, offs, regime, H = edge
    if c.kind:
        pytest.skip("streams are the Standard iterators' steppers")
    if regime == "wide":
        check_streams_refused(c, text, offs)
    else:  # ragged chunks cut mid-filler: the carried state is a slot near the top of the id range
        check_streams(c, _hays(text, offs), name, step=1500)
