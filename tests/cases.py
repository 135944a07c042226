"""Seeded test inputs shared by the CPU (emulation) and GPU parity tests."""
import numpy as np

MIXED = ["a", "b", "é", "あ", "𝄞", "c", "ß", "漢"]


def mixed_width_case(seed):
    """Charwise patterns / haystacks over chars of 1-4 bytes, empty patterns included; haystacks also
    contain unmapped chars."""
    rng = np.random.default_rng(5000 + seed)
    kind = seed % 3
    alpha = int(rng.integers(1, 8))
    npat, mx = int(rng.integers(1, 80)), int(rng.integers(1, 9))
    pats = ["".join(MIXED[int(i)] for i in rng.integers(0, alpha, size=int(rng.integers(0 if seed % 5 == 0 else 1, mx + 1))))
            for _ in range(npat)]
    syms = MIXED[:alpha] + (["z", "語"] if seed % 3 else [])
    hays = ["".join(syms[int(i)] for i in rng.integers(0, len(syms), size=int(rng.integers(0, 200)))).encode()
            for _ in range(60)]
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    return kind, pats, np.frombuffer(b"".join(hays), dtype=np.uint8), offs


def seeded_reduce_case(cw, kind):
    """The seeded batches of the reduction tests (HIST, DF, launch shapes): (patterns, text, offs).  Bytewise: 300
    patterns over "abcd" and 700 haystacks of up to 3000 bytes over "abcde"; charwise: mixed_width_case(9 + kind)."""
    rng = np.random.default_rng(80 + 3 * kind + cw)
    if cw:
        kind_, pats, text, offs = mixed_width_case(9 + kind)
        assert kind_ == kind
        return pats, text, offs
    pats = [bytes(rng.integers(97, 101, size=int(rng.integers(1, 7))).tolist()) for _ in range(300)]
    lens = rng.integers(0, 3000, size=700)
    offs = np.zeros(len(lens) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    text = rng.integers(97, 102, size=int(offs[-1])).astype(np.uint8)
    return pats, text, offs


def nul_heavy_case(kind, n_patterns=120000, n_hay=1500, max_len=600):
    """Binary patterns of 3..12 bytes and haystacks drawn mostly from 0x00: with more than ~16k patterns the
    automaton is larger than the default hot region of the compact image, so many states sit in the shifted
    part next to the holes re-placed families leave behind (dev_image.cpp)."""
    rng = np.random.default_rng(31337 + kind)
    pats = sorted(set(bytes(rng.choice([0, 0, 1, 2, 3, 255], size=int(rng.integers(3, 13))).tolist())
                      for _ in range(n_patterns)))
    lens = rng.integers(0, max_len, size=n_hay)
    offs = np.zeros(n_hay + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens)
    text = rng.choice(np.array([0, 0, 0, 1, 2, 3, 255], dtype=np.uint8), size=int(offs[-1]))
    return pats, np.ascontiguousarray(text), offs


def layout_cases():
    """Dictionaries whose double array depends on num_free_blocks: (name, patterns, charwise, kind, text, offs).  The
    batches of seeded_reduce_case with 4000 C2 (bytewise) or 5000 C4 (charwise) patterns added, the NUL-heavy set of
    20 000 patterns (52 224 slots with 16 free blocks, 88 320 with 1) and the 10 000 C2 patterns."""
    from daachorse_b200 import synth as S

    c2 = S.make_patterns(S.config("C2")).as_list()
    c4 = [p.decode() for p in S.make_patterns(S.config("C4"), n=5000).as_list()]
    out = []
    for cw in (False, True):
        for kind in (0, 1, 2):
            pats, text, offs = seeded_reduce_case(cw, kind)
            out.append(("%s-kind%d" % ("charwise" if cw else "bytewise", kind), list(pats) + (c4 if cw else c2[:4000]), cw, kind,
                        text, offs))
    for kind in (0, 1):
        pats, text, offs = nul_heavy_case(kind, n_patterns=20000, n_hay=300)
        out.append(("nul-heavy-kind%d" % kind, pats, False, kind, text, offs))
    rng = np.random.default_rng(17)
    hays = [b"".join(c2[int(i)] for i in rng.integers(0, len(c2), size=int(rng.integers(0, 60)))) for _ in range(400)]
    offs = np.concatenate([[0], np.cumsum([len(h) for h in hays])]).astype(np.uint64)
    out.append(("c2", c2, False, 0, np.frombuffer(b"".join(hays), dtype=np.uint8).copy(), offs))
    return out


def layout_params(cases):
    """(case index, num_free_blocks) for 16 and for every count of 1, 2, 3 and 64 whose array differs from the one
    with 16 free blocks: at these sizes 1 always does, 2, 3 and 64 mostly do not (the builder rarely fails to place a
    family in the last two blocks), and a layout equal to the default tests nothing new."""
    import oracle_api as O

    out = []
    for i, (_, pats, cw, kind, _, _) in enumerate(cases):
        ref = O.OraclePma.build(pats, charwise=cw, match_kind=kind).serialize()
        out.append((i, 16))
        out += [(i, k) for k in (1, 2, 3, 64)
                if O.OraclePma.build(pats, charwise=cw, match_kind=kind, num_free_blocks=k).serialize() != ref]
    return out


FILLER_K = 4096  # filler patterns per automaton
FILLER_SUFFIX_EVERY = 64  # every 64th filler also has its last 3 symbols as a pattern
CJK0 = 0x4E00  # charwise fillers use the 128 code points U+4E00..U+4E7F (3 UTF-8 bytes each)


def _cjk_bytes(idx):
    """UTF-8 of U+4E00 + idx, idx an integer array of shape (..., m) with values below 128: shape (..., 3 m) uint8."""
    cp = CJK0 + idx.astype(np.uint32)
    b = np.stack([0xE0 | (cp >> 12), 0x80 | ((cp >> 6) & 0x3F), 0x80 | (cp & 0x3F)], axis=-1).astype(np.uint8)
    return b.reshape(idx.shape[:-1] + (3 * idx.shape[-1],))


def _trim(j):
    """Trim pattern j: "z" and three base-25 digits over "a".."y"; each one adds one or two states to the trie."""
    return bytes([122, 97 + j // 625 % 25, 97 + j // 25 % 25, 97 + j % 25])


def _filler_patterns(cw, L, T, seed):
    """(patterns, filler rows): FILLER_K fillers of L symbols over 0x80-0xFF (charwise: over U+4E00..U+4E7F), the
    3-symbol suffixes of every FILLER_SUFFIX_EVERY-th one, 300 ASCII patterns over "abcd" and T trim patterns."""
    rng = np.random.default_rng(91000 + seed)
    if cw:
        rows = _cjk_bytes(rng.integers(0, 128, size=(FILLER_K, L)))
        sym = 3
    else:
        rows = rng.integers(0x80, 0x100, size=(FILLER_K, L)).astype(np.uint8)
        sym = 1
    fillers = [r.tobytes() for r in rows]
    suffixes = sorted({f[-3 * sym:] for f in fillers[::FILLER_SUFFIX_EVERY]})
    ascii_ = [bytes(rng.integers(97, 101, size=int(rng.integers(1, 7))).tolist()) for _ in range(300)]
    return fillers + suffixes + ascii_ + [_trim(j) for j in range(T)], rows


# (target slots, charwise, match kind) -> (filler length L, trim patterns T), found once by building the oracle's
# automaton for growing T until num_elements() == target.  A builder change that moves the count fails the tests
# that use these cases (they assert the count) instead of silently testing another regime.
FILLER_SIZES = {
    ((1 << 24) - 65536, False, 0): (4080, 3056),
    (1 << 24, False, 0): (4096, 3056),
    ((1 << 24) + 256, False, 0): (4096, 3243),
    (1 << 24, False, 1): (4096, 3056),
    ((1 << 24) - 256, True, 0): (4096, 3219),
    (1 << 24, True, 0): (4096, 3409),
}
# Bytewise fillers whose depth-3 states sit in the highest slots, by filler length.  The builder places each filler's
# chain in consecutive slots, in an order of its own, so these whole fillers walk to within 4 400 slots of the top
# (slot 16 772 892 of 2^24; 16 707 360 of 2^24 - 65 536).
FILLER_TOP = {4080: [2464, 3609, 1716, 2975], 4096: [2223, 1856, 890, 1336]}


def filler_case(target_slots, charwise=False, kind=0, seed=0):
    """An automaton of exactly `target_slots` slots, and haystacks that walk to its deepest states:
    (patterns, text, offs).  Patterns as _filler_patterns (bytes; UTF-8 for charwise).  Haystacks: whole fillers
    (their last states are the deepest, and breadth-first placement puts them at the end of the array), fillers cut
    short, ASCII text over "abcde", mixtures of the three, and empty haystacks; charwise ones are cut at char
    boundaries."""
    L, T = FILLER_SIZES[(target_slots, bool(charwise), kind)]
    pats, rows = _filler_patterns(charwise, L, T, seed)
    sym = 3 if charwise else 1
    rng = np.random.default_rng(92000 + seed)
    pick = rng.choice(FILLER_K, size=24, replace=False)
    pick[:4] = [0, FILLER_SUFFIX_EVERY, FILLER_K - 1, FILLER_K - FILLER_SUFFIX_EVERY]  # with and without a suffix pattern
    if not charwise:  # the fillers the builder placed last: their paths end in the highest slots
        pick[4:8] = FILLER_TOP[L]

    def filler(i, k=None):
        return rows[i, : (L if k is None else k) * sym].tobytes()

    def ascii_(n):
        return bytes(rng.integers(97, 102, size=n).tolist())

    hays = [filler(int(i)) for i in pick[:8]]
    hays += [filler(int(i), int(rng.integers(1, L))) for i in pick[8:14]]
    hays += [filler(int(pick[14]), L - 1), filler(int(pick[15]), 3), b"", ascii_(3000), ascii_(17), b""]
    hays += [ascii_(40) + filler(int(pick[16])) + ascii_(40),
             filler(int(pick[17])) + filler(int(pick[18])) + filler(int(pick[19]), int(rng.integers(1, L))),
             filler(int(pick[20]))[-9 * sym:] + ascii_(30) + filler(int(pick[21]), 50),
             ascii_(200) + filler(int(pick[22]), L // 2), filler(int(pick[23])) + ascii_(5)]
    offs = np.zeros(len(hays) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(h) for h in hays])
    return pats, np.frombuffer(b"".join(hays), dtype=np.uint8).copy(), offs


def damage_standard_wire(wire, edits):
    """Overwrite fields of a serialized bytewise Standard automaton: edits = [(slot, column, value)], columns
    0 = base, 1 = fail, 2 = output_pos << 8 | check (src/bytewise.rs:801-820)."""
    w = bytearray(wire)
    n = int(np.frombuffer(w, dtype="<u4", count=1)[0])
    a = np.frombuffer(w, dtype="<u4", count=n * 3, offset=4).reshape(n, 3)
    for slot, col, val in edits:
        a[slot, col] = val
    return bytes(w), a.copy()


def hand_made_case(hay_len=60000, n_hay=3):
    """A serialized Standard automaton whose failure links were rewired by hand (every inner state of depth > 2
    fails to ROOT): valid for the crate's deserialize, not Aho-Corasick's automaton -- the state after a text
    depends on more than its last bytes.  Long haystacks, so that a scan which cuts them into segments shows it."""
    import oracle_api as O
    rng = np.random.default_rng(77)
    pats = sorted(set(bytes(rng.integers(97, 100, size=int(rng.integers(2, 9))).tolist()) for _ in range(300)))
    wire = O.OraclePma.build(pats).serialize()
    _, a = damage_standard_wire(wire, [])
    edits = [(s, 1, 0) for s in range(2, len(a)) if a[s, 0] != 0 and a[s, 1] != 0][::2]
    wire, _ = damage_standard_wire(wire, edits)
    offs = np.arange(n_hay + 1, dtype=np.uint64) * np.uint64(hay_len)
    text = rng.integers(97, 100, size=int(offs[-1])).astype(np.uint8)
    return wire, text, offs
