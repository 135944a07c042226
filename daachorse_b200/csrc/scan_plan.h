// Which kernel runs a scan, and whether and how its batch is cut into segments: decided here once, for every result
// kind, by enqueue_scan / enqueue_rk in dev_scan.cu and by the CPU emulators under tests/ (so that they test the choice
// the device makes).  Plain C++17 on plain values: modes are dach_scan_mode (== scan_lane.cuh's M_*).
#pragma once

#include <algorithm>
#include <cstdint>

#include "../../include/daachorse_b200.h"

namespace dach {

enum class Machine {
    Lane,        // k_scan / k_scan_rk: one haystack per lane, the reference-shaped loops
    Std,         // StdMachine (option kernel = 1; matches only)
    Std2,        // StdMachine2 (option kernel = 2; matches only)
    Std3,        // StdMachine3 with the per-lane event queue (k_scan_machine, k_scan_machine_rk)
    Std3Direct,  // StdMachine3, events stored at their landing (k_scan_direct; matches only)
    Duo,         // StdMachine3 with two haystacks per lane (k_scan_duo, option kernel = 4; matches only)
    Lm,          // LmMachine: bytewise leftmost
    Cw,          // CwMachine: charwise, every iterator
};

struct ScanInputs {
    int64_t opt_kernel = 3;
    bool compact = false;      // the automaton has a compact image (bytewise Standard, at most 2^24 states)
    bool charwise = false;
    bool root_opos = false;    // root_opos != 0: an empty pattern (find_iter keeps the lane-per-haystack loop)
    bool root_base = false;    // BASE(ROOT) != 0 in the compact image
    bool segmentable = false;  // HostImage::segmentable
    int64_t opt_seg_len = 0;   // < 0: no segments
    int ctas_per_sm = 1;
    int64_t opt_event_queue = 0;
    bool stream = false;       // a chunk of a stream: it resumes in a given state
    bool matches = true;       // the result kind: the match list (RK_MATCHES), or a reduction
    bool first = false;        // ... FIRST (RK_FIRST)
    int mode = DACH_FIND;
};

struct ScanPlan {
    Machine machine = Machine::Lane;
    int mode = DACH_FIND;  // the iterator the kernel runs: FIRST folds the Standard ones into find_overlapping
    bool refused = false;  // a stream chunk without a Standard lane machine
    bool seg = false;      // haystacks may be cut into segments

    bool lane_machine() const { return machine != Machine::Lane; }
    bool std3() const { return machine == Machine::Std3 || machine == Machine::Std3Direct || machine == Machine::Duo; }
    // StdMachine3's matches path stores events (k_scan_machine / k_scan_direct), expanded by k_expand
    bool events() const { return machine == Machine::Std3 || machine == Machine::Std3Direct; }
};

inline ScanPlan plan_scan(const ScanInputs& in) {
    ScanPlan p;
    // the first event of a haystack is the same for all three Standard iterators: FIRST runs find_overlapping (not on
    // a stream: the state carried after a find match is not the find_overlapping one)
    p.mode = (in.first && in.mode != DACH_LEFTMOST_FIND && !in.stream) ? DACH_FIND_OVERLAPPING : in.mode;
    // the lane machines serve every iterator of both automata except find_iter with an empty pattern (it only reports
    // zero-length matches, src/bytewise/iter.rs:60-85), which keeps the simple kernel
    const bool v1 = in.opt_kernel >= 1 && in.compact && !(p.mode == DACH_FIND && in.root_opos);
    if (!v1)
        p.machine = Machine::Lane;
    else if (in.charwise)
        p.machine = Machine::Cw;
    else if (p.mode == DACH_LEFTMOST_FIND)
        p.machine = Machine::Lm;
    else if (!in.matches)
        // StdMachine3 keeps ROOT's record in registers and probes it like any state: needs BASE(ROOT) != 0.  Options
        // kernel = 1, 2, 4 run it too: the other machines exist for the matches only.
        p.machine = in.root_base ? Machine::Std3 : Machine::Lane;
    else if (in.opt_kernel < 2 || !in.root_base)
        p.machine = Machine::Std;
    else if (in.opt_kernel < 3)
        p.machine = Machine::Std2;
    else if (in.opt_kernel >= 4 && in.ctas_per_sm == 1)
        p.machine = Machine::Duo;
    else if (in.ctas_per_sm == 1 && in.opt_event_queue == 0)
        p.machine = Machine::Std3Direct;  // one CTA per SM, whose shared memory the staged records fill
    else
        p.machine = Machine::Std3;
    p.refused = in.stream && (p.machine == Machine::Lane || p.machine == Machine::Std || p.machine == Machine::Lm);
    // find_overlapping / no_suffix on the bytewise Standard machines may cut haystacks into segments (exact with an
    // (L-1)-byte warm-up, SURVEY.md Appendix C.1) so that small batches and long haystacks still fill the machine;
    // everything else works on whole haystacks, and so does a chunk of a stream
    const bool std_machine = p.machine != Machine::Lane && p.machine != Machine::Lm && p.machine != Machine::Cw;
    const bool cut_mode = p.mode == DACH_FIND_OVERLAPPING || p.mode == DACH_FIND_OVERLAPPING_NO_SUFFIX;
    p.seg = std_machine && !in.stream && cut_mode && in.opt_seg_len >= 0 && in.segmentable;
    return p;
}

// The shortest segment: the warm-up (max_pattern_len - 1 bytes) costs at most 1/8
inline uint64_t seg_floor(uint64_t warm) { return std::max<uint64_t>(256, 8 * warm); }

// The segment length a batch of text_bytes bytes on `lanes` lanes asks for: option seg_len if > 0, else ~2 items per lane
inline uint64_t seg_want(int64_t opt_seg_len, uint64_t text_bytes, uint64_t lanes, uint64_t warm) {
    return opt_seg_len > 0 ? (uint64_t)opt_seg_len : std::max(text_bytes / (2 * lanes) + 1, seg_floor(warm));
}

// `want` rounded up to 256 as the segment length of a batch of n haystacks and text_bytes bytes, cut_bytes of which are
// cut; and the most items that makes.  False (whole haystacks, n items) when every haystack fits one segment, the
// length reaches 2^31 or the items would pass 2^32-16.
inline bool seg_cut(uint64_t want, uint64_t text_bytes, uint64_t cut_bytes, uint64_t n, uint32_t* seg_len, uint64_t* n_items_max) {
    want = (want + 255) & ~uint64_t(255);
    *seg_len = 0;
    *n_items_max = n;
    if (want >= text_bytes || want >= (1ull << 31)) return false;
    const uint64_t items = n + cut_bytes / want + 1;
    if (items > 0xfffffff0ull) return false;
    *seg_len = (uint32_t)want;
    *n_items_max = items;
    return true;
}

}  // namespace dach
