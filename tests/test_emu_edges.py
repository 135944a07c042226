"""Edges of the scan's contract on the CPU emulation of the lane logic (tests/emu: matches, events, COUNT / FIRST,
HIST and DF), against the oracle:

  * the 2^32 address line: StdMachine3 keeps the low 32 bits of the text address as its cursor and adds the carry back
    when it forms an address (Lane3::ap, block_of).  Text mapped across 0x1_0000_0000 puts haystacks, segments and
    their warm-up on both sides of that line, for matches, COUNT, FIRST, HIST and DF (both keys, with a pair table so
    small that windows are scanned again as halves);
  * `needed` past 2^32 matches in one haystack: the per-item match counts are u32.  A count that wraps must not come
    back as a small `needed` with DACH_OUTPUT_OVERFLOW (no capacity would help); the scan is refused and `needed` is
    exact.
"""
import ctypes as C
import mmap

import numpy as np
import pytest

import emu_api as EA
import emu_df_api as EF
import emu_events_api as EV
import emu_hist_api as EH
import emu_reduce_api as ER
import oracle_api as O
from test_emu_df import doc_freq

INVALID_ARGUMENT, OUTPUT_OVERFLOW = 1, 6
ORC = {0: O.FIND, 1: O.FIND_OVERLAPPING, 2: O.FIND_OVERLAPPING_NO_SUFFIX, 3: O.LEFTMOST_FIND}

LINE = 1 << 32
MAP_AT = LINE - (1 << 20)  # 1 MiB below the line ...
MAP_LEN = 2 << 20          # ... to 1 MiB above it
MAP_FIXED_NOREPLACE = 0x100000


@pytest.fixture(scope="module")
def across_the_line():
    """2 MiB of anonymous memory at [2^32 - 1 MiB, 2^32 + 1 MiB) as a numpy uint8 array; skipped where the
    address is taken or the kernel refuses the fixed mapping."""
    libc = C.CDLL(None, use_errno=True)
    libc.mmap.restype = C.c_void_p
    libc.mmap.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_long]
    libc.munmap.argtypes = [C.c_void_p, C.c_size_t]
    p = libc.mmap(MAP_AT, MAP_LEN, mmap.PROT_READ | mmap.PROT_WRITE,
                  mmap.MAP_PRIVATE | mmap.MAP_ANONYMOUS | MAP_FIXED_NOREPLACE, -1, 0)
    if p in (None, C.c_void_p(-1).value):
        pytest.skip("cannot map memory across the 4 GiB address line here")
    if p != MAP_AT:  # a kernel without MAP_FIXED_NOREPLACE takes the address as a hint only
        libc.munmap(p, MAP_LEN)
        pytest.skip("cannot map memory across the 4 GiB address line here")
    buf = np.ctypeslib.as_array((C.c_uint8 * MAP_LEN).from_address(p))
    assert buf.ctypes.data == MAP_AT
    try:
        yield buf
    finally:
        del buf
        libc.munmap(MAP_AT, MAP_LEN)


def _line_batches(rng):
    """(lo, offs) windows of the mapping, offsets relative to `lo`: haystacks that start 1-17, 255 and 4096 bytes below
    the line and end above it, one that ends exactly at it and one that starts there, and long ones whose segments'
    warm-up crosses it."""
    L = LINE - MAP_AT
    out = []
    for d in list(range(1, 18)) + [255, 4096]:
        lo = L - d - 64
        out.append((lo, np.array([0, 64, 64 + d + int(rng.integers(1, 400)), 64 + d + 500], dtype=np.uint64)))
    out.append((L - 700, np.array([0, 300, 700, 1100, 1117], dtype=np.uint64)))  # ends at the line, starts at it
    lo = L - 3000
    out.append((lo, np.array([0, 2990, 2990 + 1500, 2990 + 1500 + 7, 2990 + 1500 + 700], dtype=np.uint64)))
    out.append((L - 9000, np.array([0, 9000 - 37, 9000 + 5000], dtype=np.uint64)))
    return out


def _spy(module, fn_name, arg):
    """Wraps the library module's binding calls so that the text pointer handed to `fn_name` (argument `arg`) is
    recorded."""
    real = module.lib()
    seen = []

    class Spy:
        def __getattr__(self, name):
            f = getattr(real, name)
            if name != fn_name:
                return f

            def call(*a):
                seen.append(a[arg])
                return f(*a)
            return call

    return Spy(), seen


def _oracle(opma, mode, text, offs):
    ref = opma.scan_batch(ORC[mode], np.array(text), offs, want_matches=True)
    return ref["matches"], ref["counts"].astype(np.uint64)


@pytest.mark.parametrize("cw", [False, True], ids=["bytewise", "charwise"])
def test_address_line_in_the_emulations(across_the_line, cw, monkeypatch):
    buf = across_the_line
    rng = np.random.default_rng(7 + cw)
    buf[:] = rng.integers(97, 101, size=buf.size).astype(np.uint8)  # ASCII: valid UTF-8 everywhere
    pats = sorted({bytes(rng.integers(97, 101, size=int(rng.integers(1, 9))).tolist()) for _ in range(120)})
    pats = [p.decode() for p in pats] if cw else pats
    spies = {}
    for mod, fn, arg in ((EA, "emu_scan_batch_wire", 4), (EV, "emu_events_scan_wire", 3),
                         (ER, "emu_reduce_batch_wire", 5), (EH, "emu_hist_batch_wire", 5), (EF, "emu_df_batch_wire", 5)):
        spy, seen = _spy(mod, fn, arg)
        monkeypatch.setattr(EA, "_lib", spy)  # the one library every binding loads through
        spies[mod.__name__] = seen
    kinds = (0,) if cw else (0, 1, 2)
    for kind in kinds + ((1, 2) if cw else ()):
        opma = O.OraclePma.build(pats, charwise=cw, match_kind=kind)
        wire = opma.serialize()
        recs = ER.image_outputs(wire, cw)  # DF by output record: the record of each value (the pattern index)
        rec_of = np.zeros(len(pats), dtype=np.int64)
        rec_of[recs[:, 0].astype(np.int64)] = np.arange(len(recs))
        modes = (3,) if kind else (0, 1, 2)
        for lo, offs in _line_batches(rng):
            text = buf[lo: lo + int(offs[-1])]
            assert text.ctypes.data == MAP_AT + lo
            crosses = MAP_AT + lo < LINE < MAP_AT + lo + text.size
            assert crosses or text.ctypes.data + text.size == LINE or text.ctypes.data == LINE
            for mode in modes:
                want, counts = _oracle(opma, mode, text, offs)
                wo = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
                runs = [dict(kernel=0)]
                if cw:
                    runs += [dict(kernel=1)]
                elif kind:
                    runs += [dict(kernel=1)]  # LmMachine
                else:
                    runs += [dict(kernel=1), dict(kernel=2), dict(kernel=3, hot_n=0), dict(kernel=3, hot_n=4096), dict(kernel=4)]
                    if mode != 0:
                        runs += [dict(kernel=3, hot_n=4096, seg_len=s) for s in (64, 256)]
                for kw in runs:
                    rc, m, oo, need = EA.scan(wire, cw, mode, text, offs, **kw)
                    assert rc == 0 and need == len(want), (kind, mode, lo, kw)
                    assert m.tobytes() == want.tobytes(), (kind, mode, lo, kw)
                    assert np.array_equal(oo, wo), (kind, mode, lo, kw)
                if not cw and not kind:  # StdMachine3's event path
                    for kw in [dict(hot_n=h) for h in (0, 4096)] + ([dict(hot_n=4096, seg_len=s) for s in (64, 256)] if mode else []):
                        rc, m, oo, need, _ = EV.scan(wire, mode, text, offs, **kw)
                        assert rc == 0 and m.tobytes() == want.tobytes() and np.array_equal(oo, wo), (mode, lo, kw)
                for kernel in (0, 3):
                    rc, got, total = ER.reduce(wire, cw, mode, 1, text, offs, kernel=kernel)
                    assert rc == 0 and np.array_equal(got, counts) and total == len(want), (kind, mode, lo, kernel)
                    rc, (first, found), nf = ER.reduce(wire, cw, mode, 2, text, offs, kernel=kernel)
                    assert rc == 0 and nf == int((counts > 0).sum())
                    assert np.array_equal(found, counts > 0), (kind, mode, lo, kernel)
                    idx = wo[:-1][found].astype(np.int64)  # each haystack's first match in the oracle's list
                    assert first[found].tobytes() == want[idx].tobytes(), (kind, mode, lo, kernel)
                    nv = len(pats)
                    rc, h, total, _ = EH.hist(wire, cw, mode, "value", text, offs, nv + 5, kernel=kernel)
                    assert rc == 0 and total == len(want)
                    assert np.array_equal(h[:nv], np.bincount(want["value"], minlength=nv).astype(np.uint64))
                    assert not h[nv:].any()
                    for key, k, keys in (("value", nv, want["value"].astype(np.int64)), ("output", len(recs), rec_of[want["value"]])):
                        ref = doc_freq(np.repeat(np.arange(len(counts)), counts.astype(np.int64)), keys, k)
                        for pairs in (1, 1 << 16):  # 1: the smallest table, windows re-scanned as halves across the line
                            rc, got, total, _ = EF.df(wire, cw, mode, key, text, offs, k + 5, kernel=kernel, df_pairs=pairs,
                                                      out=np.full(k + 5, 7, dtype=np.uint64))
                            assert rc == 0 and total == int(ref.sum()), (kind, mode, lo, kernel, key, pairs)
                            assert np.array_equal(got[:k] - np.uint64(7), ref), (kind, mode, lo, kernel, key, pairs)
                            assert (got[k:] == 7).all(), (kind, mode, lo, kernel, key, pairs, "df written past the key range")
    # every binding handed the kernels' lane logic the mapped text itself, not a copy
    for name, seen in spies.items():
        if name == "emu_events_api" and cw:
            continue
        assert seen, name
        assert all(MAP_AT <= int(p) < MAP_AT + MAP_LEN for p in seen), name


# ---- needed past 2^32 ------------------------------------------------------------------------------------------------
# One haystack of N x "a" and the patterns "a", "aa", ..., "a" x 64: find_overlapping yields 64 N - 2016 matches.
ABOVE = 67108896  # 2^32 + 32 matches
BELOW = ABOVE - 1  # 2^32 - 32 matches


def _runs_of_a(n, cw):
    pats = ["a" * k for k in range(1, 65)]
    wire = O.OraclePma.build(pats if cw else [p.encode() for p in pats], charwise=cw).serialize()
    return wire, np.full(n, 97, dtype=np.uint8), np.array([0, n], dtype=np.uint64)


@pytest.mark.parametrize("path,n", [("kernel0", ABOVE), ("kernel3_whole", BELOW), ("charwise_kernel1", ABOVE),
                                    ("events", ABOVE)])
def test_needed_past_2_pow_32_matches_is_exact(path, n):
    """A haystack that is not cut into segments counts its matches in a u32 per item.  Below 2^32 the scan overflows a
    small buffer with the exact `needed`; above it the scan is refused (DACH_INVALID_ARGUMENT: no capacity can hold
    such a list) with the exact `needed` -- before, the count wrapped and the scan reported OUTPUT_OVERFLOW with
    needed == 32."""
    exact = 64 * n - 2016
    assert (exact > 0xffffffff) == (n == ABOVE)
    cw = path.startswith("charwise")
    wire, text, offs = _runs_of_a(n, cw)
    if path == "events":
        rc, _, _, need, _ = EV.scan(wire, 1, text, offs, hot_n=4096, seg_len=0, pool_blocks=64, out_cap=1024)
    else:
        kernel = {"kernel0": 0, "kernel3_whole": 3, "charwise_kernel1": 1}[path]
        rc, _, _, need = EA.scan(wire, cw, 1, text, offs, hot_n=4096 if kernel == 3 else 0, pool_blocks=64, out_cap=1024,
                                 kernel=kernel, seg_len=0)
    assert need == exact
    assert rc == (INVALID_ARGUMENT if exact > 0xffffffff else OUTPUT_OVERFLOW)
