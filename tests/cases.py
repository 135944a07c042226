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
