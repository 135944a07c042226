"""The surface of the crate's Python wrapper, daac-tools/python-daachorse (the only other consumer the
reference names: README.md:19, 223-229), on top of the GPU scan path.

python-daachorse is a separate repository and is not part of the reference snapshot, so this mirror follows
its published interface as far as it can be stated from the crate side (SURVEY.md section 8(f) rank 4): one
``Automaton`` class built from a list of ``str`` patterns and a match kind, wrapping the crate's
``CharwiseDoubleArrayAhoCorasick`` with pattern indices as values; ``find`` / ``find_overlapping`` /
``find_overlapping_no_suffix`` / ``leftmost_find`` return ``[(start, end, pattern_index), ...]`` with positions
counted in *characters* of the Python ``str`` (the wrapper converts the crate's byte positions), the
``*_as_strings`` variants return the matched substrings.  What cannot be checked offline is flagged as such in
DESIGN.md; the semantics of every method are those of the crate iterator it names, and those are tested.

    >>> pma = Automaton(['bcd', 'ab', 'a'])
    >>> pma.find_overlapping('abcd')
    [(0, 1, 2), (0, 2, 1), (1, 4, 0)]
"""
import numpy as np

from .automaton import (FIND, FIND_OVERLAPPING, FIND_OVERLAPPING_NO_SUFFIX, LEFTMOST_FIND,
                        CharwiseDoubleArrayAhoCorasickBuilder, MatchKind)

MATCH_KIND_STANDARD = int(MatchKind.Standard)
MATCH_KIND_LEFTMOST_LONGEST = int(MatchKind.LeftmostLongest)
MATCH_KIND_LEFTMOST_FIRST = int(MatchKind.LeftmostFirst)


def _char_index(data):
    """byte offset -> character offset table of a UTF-8 buffer (offsets at char boundaries only are used)."""
    b = np.frombuffer(data, dtype=np.uint8)
    starts = (b & 0xC0) != 0x80
    idx = np.zeros(len(b) + 1, dtype=np.int64)
    np.cumsum(starts, out=idx[1:])
    return idx


class Automaton:
    """``Automaton(patterns, match_kind=MATCH_KIND_STANDARD)``: pattern i is reported as value i."""

    def __init__(self, patterns, match_kind=MATCH_KIND_STANDARD):
        self._patterns = [str(p) for p in patterns]
        self._pma = CharwiseDoubleArrayAhoCorasickBuilder.new().match_kind(MatchKind(match_kind)).build(self._patterns)

    def _scan(self, mode, haystacks):
        enc = [h.encode("utf-8") for h in haystacks]
        offs = np.zeros(len(enc) + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(e) for e in enc])
        blob = np.frombuffer(b"".join(enc), dtype=np.uint8) if offs[-1] else np.zeros(0, dtype=np.uint8)
        r = self._pma.scan_batch_host(mode, blob, offs)
        out = []
        for i, e in enumerate(enc):
            m = r.matches[int(r.offsets[i]): int(r.offsets[i + 1])]
            ci = _char_index(e)
            out.append([(int(ci[s]), int(ci[t]), int(v)) for s, t, v in zip(m["start"], m["end"], m["value"])])
        return out

    # -- one haystack: the crate iterator named, collected into a list ------------------------------------
    def find(self, haystack):
        """find_iter (src/charwise.rs:184)"""
        return self._scan(FIND, [haystack])[0]

    def find_overlapping(self, haystack):
        """find_overlapping_iter (src/charwise.rs:290)"""
        return self._scan(FIND_OVERLAPPING, [haystack])[0]

    def find_overlapping_no_suffix(self, haystack):
        """find_overlapping_no_suffix_iter (src/charwise.rs:412)"""
        return self._scan(FIND_OVERLAPPING_NO_SUFFIX, [haystack])[0]

    def leftmost_find(self, haystack):
        """leftmost_find_iter (src/charwise.rs:553)"""
        return self._scan(LEFTMOST_FIND, [haystack])[0]

    def find_as_strings(self, haystack):
        return [haystack[s:e] for s, e, _ in self.find(haystack)]

    def find_overlapping_as_strings(self, haystack):
        return [haystack[s:e] for s, e, _ in self.find_overlapping(haystack)]

    def find_overlapping_no_suffix_as_strings(self, haystack):
        return [haystack[s:e] for s, e, _ in self.find_overlapping_no_suffix(haystack)]

    def leftmost_find_as_strings(self, haystack):
        return [haystack[s:e] for s, e, _ in self.leftmost_find(haystack)]

    # -- many haystacks per call: what the GPU is for ----------------------------------------------------------
    def find_batch(self, haystacks):
        return self._scan(FIND, list(haystacks))

    def find_overlapping_batch(self, haystacks):
        return self._scan(FIND_OVERLAPPING, list(haystacks))

    def find_overlapping_no_suffix_batch(self, haystacks):
        return self._scan(FIND_OVERLAPPING_NO_SUFFIX, list(haystacks))

    def leftmost_find_batch(self, haystacks):
        return self._scan(LEFTMOST_FIND, list(haystacks))
