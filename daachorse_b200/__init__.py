"""daachorse_b200 -- an H100-native (sm_90a) double-array Aho-Corasick scan path that is a
drop-in for the scan path of the Rust crate daac-tools/daachorse 4.0.0.

The package holds only what that path needs: ``csrc/`` (CUDA kernels + the C ABI of
include/daachorse_b200.h, built in-tree as libdaachorse_b200.so) and this host-side mirror of
the crate's public interface.
"""
from .automaton import (FIND, FIND_OVERLAPPING, FIND_OVERLAPPING_NO_SUFFIX, LEFTMOST_FIND, MATCH_DTYPE,
                        BatchResult, CharwiseDoubleArrayAhoCorasick,
                        CharwiseDoubleArrayAhoCorasickBuilder, DaachorseError, DoubleArrayAhoCorasick,
                        DoubleArrayAhoCorasickBuilder, Job, Match, MatchKind)

__all__ = [
    "DoubleArrayAhoCorasick", "DoubleArrayAhoCorasickBuilder", "CharwiseDoubleArrayAhoCorasick",
    "CharwiseDoubleArrayAhoCorasickBuilder", "MatchKind", "Match", "DaachorseError", "BatchResult", "Job",
    "FIND", "FIND_OVERLAPPING", "FIND_OVERLAPPING_NO_SUFFIX", "LEFTMOST_FIND", "MATCH_DTYPE",
]
