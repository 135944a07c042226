// Host-side builder of the device scan image (see scan_lane.cuh for the layouts).
#pragma once

#include <cstdint>
#include <vector>

#include "host.h"

namespace dach {

// Two-entry output lists (HostImage::pairs, read by k_expand_desc): per output record {value, length, parent's value,
// parent's length | class << 30}, class = the length of the list that starts at the record, saturated at 3.  Class 1
// leaves the parent's fields 0; class 3 lists are walked through the outputs from the head.
constexpr uint32_t PAIR_CLASS_SHIFT = 30;
constexpr uint32_t PAIR_LEN_MASK = (1u << PAIR_CLASS_SHIFT) - 1u;

struct HostImage {
    bool charwise = false;
    uint8_t match_kind = 0;
    uint32_t n_slots = 0;
    uint32_t root_opos = 0;
    uint32_t max_pattern_len = 0;
    std::vector<uint32_t> rec;         // 4 words per slot
    std::vector<uint32_t> outputs;     // 4 words per output
    std::vector<uint32_t> pairs;       // 4 words per output (PAIR_* in scan_lane.cuh), empty if a pattern length is >= 2^30
    std::vector<uint32_t> root_table;  // 256 words (bytewise)
    std::vector<uint32_t> crec;        // compact records, 4 words per slot (bytewise Standard, <= 2^24 slots)
    std::vector<uint32_t> opos_tab;    // output_pos per slot (with crec)
    uint32_t root_base = 0;            // BASE of ROOT in the compact image
    // hot-first relayout of the compact bytewise image (dev_image.cpp): the children of the hottest states
    // occupy slots [0, hot_slots), every other slot s of the crate's numbering sits at s + hot_slots
    uint32_t want_hot_slots = 65536;   // in: size of the hot region to build (rounded to 256; 0 = keep the crate's numbering)
    uint32_t hot_slots = 0;            // out
    uint32_t n_cslots = 0;             // slots of the compact image (n_slots + hot_slots)
    std::vector<uint32_t> new_of_old;  // crate slot -> compact slot (stream chunks take and return crate state ids)
    std::vector<uint32_t> old_of_new;  // compact slot -> crate slot
    std::vector<uint32_t> mapper;      // charwise code table
    // bytewise Standard, compact image: the automaton is Aho-Corasick's in the textbook sense (a trie whose failure
    // links lead to the longest proper suffix, no state deeper than the longest pattern), as everything the
    // builders make is.  Only then may a long haystack be cut into segments with a warm-up of max_pattern_len - 1
    // bytes; a hand-made blob that merely passes validation is scanned whole.
    bool segmentable = false;
};

// Returns DACH_OK or DACH_INVALID_AUTOMATON (a failure chain that never reaches ROOT would
// spin a kernel forever; the crate documents the same hazard at src/bytewise.rs:824-830).
int build_image(const dach_pma* p, HostImage* img);

}  // namespace dach
