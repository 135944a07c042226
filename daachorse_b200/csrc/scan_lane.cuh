// Per-lane scan logic of libdaachorse_b200 (sm_90a).
//
// Everything here is __host__ __device__ so that tests/emu can compile the SAME lane logic
// with g++ (-DDACH_EMU) and step it on the CPU against the oracle while no GPU is attached.
// That harness is test infrastructure; the product only ever runs this code inside the
// CUDA kernels of dev_scan.cu.
//
// Contents, in file order:
//   - wide records + the lane-per-haystack loops (scan_standard / scan_leftmost): the reference's control
//     flow as written; used by k_scan for automata above 2^24 slots, find_iter with an empty pattern, kernel=0
//   - StdMachine   bytewise Standard lane machine, first cut (kernel=1)
//   - LmMachine    bytewise leftmost_find_iter on the lane machine
//   - CwMachine    the four charwise iterators on the lane machine; also the charwise stream chunks
//   - StdMachine2  bytewise Standard lane machine, round 1's default (kernel=2: three phases, ROOT in registers,
//                  text shift register)
//   - StdMachine3  the default (kernel=3): no probe-state flags, one stop bit, cursor = address word, records from
//                  the hot-first image (optionally its front from shared memory); probe / resolve are separate so
//                  that k_scan_duo can keep two fetches in flight; serves stream chunks
//   - SinkOps      COUNT / FIRST / HIST on StdMachine3, LmMachine, CwMachine: their drain() / begin_item() for
//                  the other result kinds (sinks: Emitter, CountSink, FirstSink, HistSink)
//   - EventOps     the matches path of StdMachine3: events stored into event blocks (EventSink), expanded after
//                  the scan by k_expand
//
// Device image (built by dev_image.cpp from the validated host automaton):
//   wide bytewise record  uint4 {base, efail, fbase, opos<<8 | check}      16 B / slot
//       base    BASE of the slot (0 = no children)            src/bytewise.rs:1131-1137
//       efail   failure target with child-less states skipped (a state without children can
//               never satisfy a probe, src/bytewise.rs:1075-1083); kRoot ends the chase in the
//               dense root table, kDead (leftmost only) ends it at ROOT without a probe
//               (src/bytewise.rs:1120-1123)
//       fbase   BASE of efail, so a missed probe is followed by the next probe without first
//               loading the failure state's record; bit 31 (F2ROOT_BIT) says efail(efail) == ROOT,
//               so a second miss goes straight to the dense root row (slots are < 2^31)
//   wide charwise record  uint4 {base, check(parent), fail, output_pos}    src/charwise.rs:1096-1101
//   compact records (lane machines, at most 2^24 slots): described above each machine
//   output           uint4 {value, length, parent, chain}                  src/lib.rs:213-218
//       chain   length of the list that starts at this record (1 + chain of the parent): COUNT adds it per
//               find_overlapping event instead of walking the list
//   root table       256 x u32                                             src/bytewise.rs:1040-1056
#pragma once

#include <stdint.h>

#include <type_traits>

#if defined(__CUDACC__)
#define DACH_HD __host__ __device__ __forceinline__
#else
#define DACH_HD inline
#ifndef DACH_EMU_TYPES
#define DACH_EMU_TYPES
struct uint4 {
    uint32_t x, y, z, w;
};
struct uint2 {
    uint32_t x, y;
};
#endif
#endif

#if defined(__CUDA_ARCH__)
#define DACH_SYNCWARP() __syncwarp()
#else
#define DACH_SYNCWARP()
#endif

#if defined(DACH_WATCHDOG) && defined(__CUDA_ARCH__)
#include <cstdio>
#define DACH_WD_DECL(name) unsigned long long name = 0
#define DACH_WD_TICK(name, limit, ...)                 \
    if (++name > (limit)) {                            \
        printf(__VA_ARGS__);                           \
        return;                                        \
    }
#else
#define DACH_WD_DECL(name)
#define DACH_WD_TICK(name, limit, ...)
#endif

namespace dach {

constexpr uint32_t D_ROOT = 0;
constexpr uint32_t D_DEAD = 1;
constexpr uint32_t D_INVALID_CODE = 0xffffffffu;

// scan modes == dach_scan_mode
constexpr int M_FIND = 0, M_OVERLAPPING = 1, M_NO_SUFFIX = 2, M_LEFTMOST = 3;

// Match staging: every lane appends its matches to 256-byte blocks taken from one pool with an
// atomic bump allocator.  Block layout: sixteen 16-byte slots -- slot 0 = {item id, sequence number of
// the block inside the item, -, -}, slots 1..15 = one match each {start, end, value, -}: a match is ONE
// 16-byte store (three 4-byte stores cost three L1 wavefronts each time: VERDICT r1 item 8); k_gather
// packs them to the 12-byte tuples of the result.
constexpr uint32_t BLK_WORDS = 64;
constexpr uint32_t BLK_MATCHES = 15;
constexpr uint32_t BLK_SLOT_WORDS = 4;
// Event blocks (matches path of StdMachine3): the same 256 bytes, header {item, seq, first, -} -- `first` is the
// item-relative index of the block's first match -- then 30 events {end, packed slot} of 8 bytes.  k_expand turns
// them into tuples; the per-item event count (ScanParams::ev_counts) says how many events a block holds.
constexpr uint32_t BLK_EVENTS = 30;
constexpr uint32_t BLK_HDR_WORDS = 4;
// Queue entries of StdMachine3 carry the state's output-list length in the slot's high byte (compact slots are
// < 2^24), saturated at QLEN_ESCAPE: that value means "255 or more, read the head record's chain word".
constexpr uint32_t QSLOT_MASK = 0xffffffu;
constexpr uint32_t QLEN_ESCAPE = 255u;

struct ScanCtrl {
    unsigned long long next_item;  // dynamic work counter
    unsigned int blk_cursor;       // bump allocator
    unsigned int overflow;         // pool exhausted
    unsigned int bad_offsets;      // the haystack offsets are not ascending, exceed text_bytes, or a haystack is >= 4 GiB
    unsigned int carries;          // matches path: times a per-item u32 match count wrapped past 2^32 (count_carry)
};

struct ScanParams {
    // automaton image
    const uint4* rec;
    const uint4* outputs;
    const uint32_t* root_table;  // global copy (kernels stage it in shared memory)
    const uint4* crec;           // compact records (lane-machine kernels), nullptr if > 2^24 slots
    const uint32_t* opos_tab;    // output_pos per slot (lane-machine kernels)
    uint32_t root_base;          // BASE of ROOT
    uint32_t hot_entries;        // leading compact records staged in shared memory (StdMachine3), 0 = none
    const uint32_t* id_in;       // stream chunks: crate state id -> compact slot (nullptr: identity)
    const uint32_t* id_out;      // stream chunks: compact slot -> crate state id
    const uint32_t* mapper;
    uint32_t mapper_len;
    uint32_t n_slots;    // slots in the crate's numbering
    uint32_t root_opos;  // output_pos of ROOT (empty pattern), 0 = none
    uint32_t hot_n;      // leading records staged in shared memory
    // batch
    const uint8_t* text;
    const uint8_t* text_lo;   // first text byte of the batch: nothing below it is read
    const uint8_t* text_end;  // one past the last text byte: nothing at or past it is read
    const uint64_t* offs;
    uint64_t n_items;  // number of work items (== haystacks unless a segment table is given)
    // Optional segment table (find_overlapping / no_suffix only): item i covers bytes
    // [item_beg[i], item_beg[i] + seg_len) of haystack item_hay[i]; the lane warms up on the `warm`
    // bytes before its segment (max pattern length - 1) and reports only matches that end inside it
    // (SURVEY.md Appendix C.1).  n_items_dev, if set, holds the item count on the device.
    const uint32_t* item_hay;
    const uint32_t* item_beg;
    const unsigned long long* n_items_dev;
    uint32_t seg_len, warm;
    uint32_t* state_io;  // stream chunks (dach_dev_scan_stream): state id per haystack, read at its start and
                         // written at its end; nullptr for ordinary scans (every haystack starts in ROOT)
    uint32_t seg_from;  // haystacks below this index stay whole (one item each): only the tail of a batch is cut
    // results
    uint32_t* counts;     // matches per item
    uint32_t* ev_counts;  // event blocks: events stored per item
    uint32_t* pool;
    uint32_t pool_blocks;
    ScanCtrl* ctrl;
    // results of the other result kinds (CountSink / FirstSink), per item
    unsigned long long* item_count;
    uint4* item_first;  // {start, end, value, found}
    // HIST (HistSink): events per compact slot (lane machines) / reported matches per output record (lane per
    // haystack), and how many leading compact slots count in shared memory first
    unsigned long long* slot_hist;
    unsigned long long* rec_hist;
    uint32_t hist_smem;
};

// What a scan produces (compile time): every match (Emitter), the number of matches (CountSink), the first
// match and whether there is one (FirstSink), or the matches per output record of the whole batch (HistSink).
// The lane machines and the lane-per-haystack loops are the same for all four; the sink and, for FIRST, the
// stop rule differ.
constexpr int RK_MATCHES = 0, RK_COUNT = 1, RK_FIRST = 2, RK_HIST = 3;

// L2 eviction policies (64-bit descriptors made once per device by k_make_policies, dev_scan.cu):
//   [0] automaton image (records, output_pos, outputs, mapper): evict_last -- the scan is latency-bound on
//       these dependent random fetches, and a fetch that misses L2 stalls all 32 lanes of its warp;
//   [1] haystack text: a lane returns to its 32-byte sector for the next 8 bytes a few microseconds later;
//   [2] match blocks: written once here, read once by k_gather: evict_first.
// Without them the streaming text and match blocks push record sectors out of L2 (50 MB on H100, about
// the size of a UniDic-scale image).  Option l2_hints: 0 = evict_normal everywhere, 1 = text evict_first,
// 2 = text evict_normal.
#if defined(__CUDACC__)
__constant__ unsigned long long c_l2pol[3];
#endif

DACH_HD uint4 ld_u4(const uint4* p) {
#if defined(__CUDA_ARCH__)
    uint4 v;
    asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p), "l"(c_l2pol[0]));
    return v;
#else
    return *p;
#endif
}
DACH_HD uint32_t ld_u32(const uint32_t* p) {
#if defined(__CUDA_ARCH__)
    uint32_t v;
    asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(c_l2pol[0]));
    return v;
#else
    return *p;
#endif
}
// match blocks: written once here, read once by k_gather
DACH_HD void st_stream_u4(uint32_t* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
#if defined(__CUDA_ARCH__)
    asm volatile("st.global.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d), "l"(c_l2pol[2])
                 : "memory");
#else
    p[0] = a, p[1] = b, p[2] = c, p[3] = d;
#endif
}
DACH_HD void st_stream_u2(uint32_t* p, uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    asm volatile("st.global.L2::cache_hint.v2.u32 [%0], {%1,%2}, %3;" ::"l"(p), "r"(a), "r"(b), "l"(c_l2pol[2]) : "memory");
#else
    p[0] = a, p[1] = b;
#endif
}

// Per-lane atomic increments, written as inline PTX on the device: lanes of one warp reach
// these at unrelated times (each lane walks its own haystack), and the explicit instruction keeps
// the compiler from fusing them into a vote + leader-atomic + shuffle sequence that needs the
// warp to be converged at that point.
DACH_HD uint32_t bump_u32(unsigned int* p) {
#if defined(__CUDA_ARCH__)
    unsigned int old;
    asm volatile("atom.global.add.u32 %0, [%1], 1;" : "=r"(old) : "l"(p) : "memory");
    return old;
#else
    return (*p)++;
#endif
}
DACH_HD unsigned long long bump_u64(unsigned long long* p) {
#if defined(__CUDA_ARCH__)
    unsigned long long old;
    asm volatile("atom.global.add.u64 %0, [%1], 1;" : "=l"(old) : "l"(p) : "memory");
    return old;
#else
    return (*p)++;
#endif
}

// ---- haystack bytes through a 16-byte register window ---------------------------------
// Text is read with aligned 16-byte vector loads; an aligned 16-byte load never crosses a
// page, so the window may cover a few bytes outside the haystack but never faults.
struct TextWin {
    const uint8_t* hay;  // first byte of the haystack
    uint64_t cur;        // address>>4 of the cached window
    uint4 w;

    DACH_HD void open(const uint8_t* h) {
        hay = h;
        cur = ~0ull;
    }
    DACH_HD uint32_t at(uint32_t pos) {
        const uint64_t a = (uint64_t)(uintptr_t)hay + pos;
        const uint64_t blk = a >> 4;
        if (blk != cur) {
            cur = blk;
#if defined(__CUDA_ARCH__)
            const uint4* q = reinterpret_cast<const uint4*>((uintptr_t)(blk << 4));
            asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                         : "=r"(w.x), "=r"(w.y), "=r"(w.z), "=r"(w.w)
                         : "l"(q), "l"(c_l2pol[1]));
#elif defined(DACH_EMU)
            // CPU emulation (tests/emu): gather only bytes inside [emu_lo, emu_hi)
            const uint8_t* q = reinterpret_cast<const uint8_t*>((uintptr_t)(blk << 4));
            uint32_t v[4] = {0, 0, 0, 0};
            for (int i = 0; i < 16; ++i) {
                const uint8_t* qi = q + i;
                uint32_t b = (qi >= emu_lo && qi < emu_hi) ? *qi : 0;
                v[i >> 2] |= b << ((i & 3) * 8);
            }
            w.x = v[0], w.y = v[1], w.z = v[2], w.w = v[3];
#else
            w.x = w.y = w.z = w.w = 0;  // host pass of nvcc: never executed
#endif
        }
        const uint32_t o = (uint32_t)a & 15u;
        const uint32_t lo = (o & 8u) ? w.z : w.x;
        const uint32_t hi = (o & 8u) ? w.w : w.y;
        const uint32_t word = (o & 4u) ? hi : lo;
        return (word >> ((o & 3u) * 8u)) & 0xffu;
    }
#if defined(DACH_EMU)
    const uint8_t* emu_lo = nullptr;
    const uint8_t* emu_hi = nullptr;
#endif
};

// ---- match emission --------------------------------------------------------------------
// The matches path counts matches per item in 32 bits (counts, block headers and the item-relative indices k_gather /
// k_expand place by).  A find_overlapping item that is not cut into segments can pass 2^32 matches; where its count
// wraps, count_carry() records the carry -- finish_scan (dev_scan.cu) then reports the exact total, item_offs[n] +
// carries * 2^32, and refuses the scan -- and raises `overflow`, so that no placement kernel writes by the wrapped
// offsets.  The check sits where a count grows (emit, the event drain), never in a machine's step().
DACH_HD void count_carry(const ScanParams& P) {
#if defined(__CUDA_ARCH__)
    asm volatile("red.global.add.u32 [%0], 1;" ::"l"(&P.ctrl->carries) : "memory");
#else
    ++P.ctrl->carries;
#endif
    P.ctrl->overflow = 1u;
}

struct Emitter {
    static constexpr int KIND = RK_MATCHES;
    uint32_t* blk;   // current block (nullptr when the pool is exhausted or nothing emitted yet)
    uint32_t fill;   // matches in the current block
    uint32_t count;  // matches of the current item
    uint32_t item;

    DACH_HD void begin(uint32_t item_id) {
        blk = nullptr;
        fill = 0;
        count = 0;
        item = item_id;
    }
    DACH_HD void emit(const ScanParams& P, uint32_t start, uint32_t end, uint32_t value) {
        if (fill == 0) {
            const uint32_t b = bump_u32(&P.ctrl->blk_cursor);
            if (b < P.pool_blocks) {
                blk = P.pool + (size_t)b * BLK_WORDS;
                st_stream_u4(blk, item, count / BLK_MATCHES, 0u, 0u);
            } else {
                blk = nullptr;
                P.ctrl->overflow = 1u;
            }
        }
        if (blk) {
            st_stream_u4(blk + BLK_SLOT_WORDS * (1 + fill), start, end, value, 0u);
        }
        fill = (fill + 1 == BLK_MATCHES) ? 0 : fill + 1;
        if (++count == 0) count_carry(P);
    }
    DACH_HD void finish(const ScanParams& P) { P.counts[item] = count; }
    DACH_HD bool stopped() const { return false; }
};

// COUNT: matches of the current item, 64-bit (overlapping lists make more than 2^32 matches on one haystack reachable)
struct CountSink {
    static constexpr int KIND = RK_COUNT;
    unsigned long long count;
    uint32_t item;
    DACH_HD void begin(uint32_t item_id) {
        count = 0;
        item = item_id;
    }
    DACH_HD void emit(const ScanParams&, uint32_t, uint32_t, uint32_t) { ++count; }
    DACH_HD void finish(const ScanParams& P) { P.item_count[item] = count; }
    DACH_HD bool stopped() const { return false; }
};

// FIRST: the first match of the current item; the scan of the item stops once it has one
struct FirstSink {
    static constexpr int KIND = RK_FIRST;
    uint32_t start, end, value, found, item;
    DACH_HD void begin(uint32_t item_id) {
        start = end = value = 0xffffffffu;
        found = 0;
        item = item_id;
    }
    DACH_HD void emit(const ScanParams&, uint32_t s, uint32_t e, uint32_t v) {
        if (!found) start = s, end = e, value = v, found = 1;
    }
    DACH_HD void finish(const ScanParams& P) {
        uint4 r;
        r.x = start, r.y = end, r.z = value, r.w = found;
        P.item_first[item] = r;
    }
    DACH_HD bool stopped() const { return found != 0; }
};

// the chain word of output record `opos` (1-based): how many patterns the list from there holds
DACH_HD uint32_t chain_len(const ScanParams& P, uint32_t opos) {
    return ld_u32(reinterpret_cast<const uint32_t*>(P.outputs + (opos - 1)) + 3);
}
// the list length a StdMachine3 queue entry carries; the escape value costs the two loads it saves otherwise
DACH_HD uint32_t qentry_len(const ScanParams& P, const uint32_t* opos_tab, uint32_t packed) {
    const uint32_t b = packed >> 24;
    return b != QLEN_ESCAPE ? b : chain_len(P, ld_u32(opos_tab + (packed & QSLOT_MASK)));
}

// Matches path of StdMachine3: events go to event blocks as they are, k_expand expands them after the scan.
// Blocks are taken in the warp-converged service phase with one warp-aggregated atomic (EventOps::drain).
struct EventSink {
    static constexpr int KIND = RK_MATCHES;
    uint32_t* blk;   // current block (nullptr: none yet, or the pool is exhausted)
    uint32_t fill;   // events in the current block; BLK_EVENTS when the next event needs a new block
    uint32_t nev;    // events of the current item
    uint32_t count;  // matches of the current item
    uint32_t item;
    DACH_HD void begin(uint32_t item_id) {
        blk = nullptr;
        fill = BLK_EVENTS;
        nev = 0;
        count = 0;
        item = item_id;
    }
    // block `b` of the pool becomes current; its first event is match `count` of the item
    DACH_HD void open(const ScanParams& P, uint32_t b) {
        if (b < P.pool_blocks) {
            blk = P.pool + (size_t)b * BLK_WORDS;
            st_stream_u4(blk, item, nev / BLK_EVENTS, count, 0u);
        } else {
            blk = nullptr;
            P.ctrl->overflow = 1u;
        }
        fill = 0;
    }
    DACH_HD void finish(const ScanParams& P) {
        P.counts[item] = count;
        P.ev_counts[item] = nev;
    }
    DACH_HD bool stopped() const { return false; }
};

// Walk a merged output list from `opos` (1-based, 0 = end), emitting every pattern ending
// at `end` (src/bytewise/iter.rs:134-148).
DACH_HD void emit_chain(const ScanParams& P, Emitter& E, uint32_t opos, uint32_t end) {
    while (opos != 0) {
        const uint4 o = ld_u4(P.outputs + (opos - 1));
        E.emit(P, end - o.y, end, o.x);
        opos = o.z;
    }
}
DACH_HD void emit_head(const ScanParams& P, Emitter& E, uint32_t opos, uint32_t end) {
    const uint4 o = ld_u4(P.outputs + (opos - 1));
    E.emit(P, end - o.y, end, o.x);
}
// COUNT: one loaded word per list, no walk; a head is one match
DACH_HD void emit_chain(const ScanParams& P, CountSink& E, uint32_t opos, uint32_t) {
    if (opos != 0) E.count += chain_len(P, opos);
}
DACH_HD void emit_head(const ScanParams&, CountSink& E, uint32_t, uint32_t) { ++E.count; }
// FIRST: a list's first match is its head
DACH_HD void emit_head(const ScanParams& P, FirstSink& E, uint32_t opos, uint32_t end) {
    const uint4 o = ld_u4(P.outputs + (opos - 1));
    E.emit(P, end - o.y, end, o.x);
}
DACH_HD void emit_chain(const ScanParams& P, FirstSink& E, uint32_t opos, uint32_t end) {
    if (opos != 0) emit_head(P, E, opos, end);
}

// *p += v with no return value (red.global.add.u64)
DACH_HD void red_add_u64(unsigned long long* p, unsigned long long v) {
#if defined(__CUDA_ARCH__)
    asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
#else
    *p += v;
#endif
}

// HIST: occurrences per output record over the whole batch, nothing per item.
//   lane machines: event(slot) counts the event's state -- for find_overlapping the event stands for the
//       state's whole list, for the other iterators for its head -- in P.slot_hist; the post-passes of
//       dev_scan.cu (k_hist_heads, k_hist_fold) give every record its count.  Slots below `k` count in
//       CTA-private u32 counters in shared memory first (`s_cnt`, flushed once when the CTA ends): the
//       hot-first layout puts the shallowest states, where most events land, at the front.  A counter that
//       reaches 2^31 hands 2^31 on to global memory at once (the one thread whose increment crossed it), so
//       it would take 2^31 more increments of the same counter before that thread's next instruction to
//       overflow it.
//   lane per haystack: emit_head / emit_chain add 1 per reported match to its record in P.rec_hist.
struct HistSink {
    static constexpr int KIND = RK_HIST;
    unsigned int* s_cnt = nullptr;
    uint32_t k = 0;
    uint32_t item = 0;
    DACH_HD void begin(uint32_t item_id) { item = item_id; }
    DACH_HD void finish(const ScanParams&) {}
    DACH_HD bool stopped() const { return false; }
    // a match known by its value alone cannot be counted per record: scan_standard routes ROOT's matches
    // through emit_head for HIST, so this is never reached
    DACH_HD void emit(const ScanParams&, uint32_t, uint32_t, uint32_t) {}
    DACH_HD void event(const ScanParams& P, uint32_t slot) {
        if (slot < k) {
#if defined(__CUDA_ARCH__)
            const unsigned int old = atomicAdd(s_cnt + slot, 1u);
            if (old == 0x7fffffffu) {
                atomicSub(s_cnt + slot, 0x80000000u);
                red_add_u64(P.slot_hist + slot, 0x80000000ull);
            }
#else
            if (++s_cnt[slot] == 0x80000000u) {
                s_cnt[slot] = 0;
                red_add_u64(P.slot_hist + slot, 0x80000000ull);
            }
#endif
        } else {
            red_add_u64(P.slot_hist + slot, 1);
        }
    }
};
DACH_HD void emit_head(const ScanParams& P, HistSink&, uint32_t opos, uint32_t) { red_add_u64(P.rec_hist + (opos - 1), 1); }
DACH_HD void emit_chain(const ScanParams& P, HistSink&, uint32_t opos, uint32_t) {
    while (opos != 0) {
        red_add_u64(P.rec_hist + (opos - 1), 1);
        opos = ld_u4(P.outputs + (opos - 1)).z;
    }
}

// ---- record access: leading `hot_n` records come from shared memory --------------------
struct RecView {
    const uint4* glob;
    const uint4* hot;  // shared-memory copy of glob[0 .. hot_n)
    uint32_t hot_n;
    const uint32_t* root;  // root table (shared memory on the device)
    DACH_HD uint4 get(uint32_t i) const { return i < hot_n ? hot[i] : ld_u4(glob + i); }
};

// ---- bytewise transitions ---------------------------------------------------------------
// delta(s, c) for the Standard automaton (src/bytewise.rs:1063-1088) on the device image.
// `r` is the record of the current state s (unused when s == ROOT); returns the new state
// and leaves its record in `r`.
DACH_HD uint32_t bw_step(const RecView& V, uint32_t s, uint4& r, uint32_t c) {
    if (s != D_ROOT) {
        if (r.x != 0) {  // own children
            const uint32_t ci = r.x ^ c;
            const uint4 x = V.get(ci);
            if ((x.w & 0xffu) == c) {
                r = x;
                return ci;
            }
        }
        uint32_t f = r.y, fb = r.z & 0x7fffffffu;  // bit 31 of word z is a flag (F2ROOT_BIT)
        while (f != D_ROOT) {  // failure chase; every visited state has children
            const uint32_t ci = fb ^ c;
            const uint4 x = V.get(ci);
            if ((x.w & 0xffu) == c) {
                r = x;
                return ci;
            }
            const uint4 fr = V.get(f);
            f = fr.y;
            fb = fr.z & 0x7fffffffu;
        }
    }
    const uint32_t n = V.root[c];
    if (n != D_ROOT) r = V.get(n);
    return n;
}

// delta for the leftmost automaton (src/bytewise.rs:1094-1128): as above, but a failure
// link to DEAD ends at ROOT without probing ROOT's children.
DACH_HD uint32_t bw_step_leftmost(const RecView& V, uint32_t s, uint4& r, uint32_t c) {
    if (s != D_ROOT) {
        if (r.x != 0) {
            const uint32_t ci = r.x ^ c;
            const uint4 x = V.get(ci);
            if ((x.w & 0xffu) == c) {
                r = x;
                return ci;
            }
        }
        uint32_t f = r.y, fb = r.z & 0x7fffffffu;
        while (f != D_ROOT) {
            if (f == D_DEAD) return D_ROOT;
            const uint32_t ci = fb ^ c;
            const uint4 x = V.get(ci);
            if ((x.w & 0xffu) == c) {
                r = x;
                return ci;
            }
            const uint4 fr = V.get(f);
            f = fr.y;
            fb = fr.z & 0x7fffffffu;
        }
    }
    const uint32_t n = V.root[c];
    if (n != D_ROOT) r = V.get(n);
    return n;
}

// ---- charwise ----------------------------------------------------------------------------
// UTF-8 decode of one char at `pos` (src/charwise/iter.rs:71-97); input is valid UTF-8.
DACH_HD uint32_t utf8_at(TextWin& T, uint32_t& pos) {
    const uint32_t first = T.at(pos++);
    if (first < 0x80u) return first;
    uint32_t c = T.at(pos++) & 0x3fu;
    if (first < 0xe0u) return ((first & 0x1fu) << 6) | c;
    c = (c << 6) | (T.at(pos++) & 0x3fu);
    if (first < 0xf0u) return ((first & 0x0fu) << 12) | c;
    c = (c << 6) | (T.at(pos++) & 0x3fu);
    return ((first & 0x07u) << 18) | c;
}

DACH_HD uint32_t map_code(const ScanParams& P, uint32_t cp) {  // src/charwise/mapper.rs:36-42
    return cp < P.mapper_len ? ld_u32(P.mapper + cp) : D_INVALID_CODE;
}

// src/charwise.rs:1022-1051 (leftmost == false) and :1057-1092 (leftmost == true)
template <bool LEFTMOST>
DACH_HD uint32_t cw_step(const ScanParams& P, const RecView& V, uint32_t s, uint4& r, uint32_t cp) {
    const uint32_t mc = map_code(P, cp);
    if (mc == D_INVALID_CODE) return D_ROOT;
    for (;;) {
        if (r.x != 0) {
            const uint32_t ci = r.x ^ mc;
            const uint4 x = V.get(ci);
            if (x.y == s) {
                r = x;
                return ci;
            }
        }
        if (s == D_ROOT) return D_ROOT;
        const uint32_t f = r.z;
        // DEAD ends the chase (src/charwise.rs:1081-1084).  A valid Standard automaton never links a
        // live state to DEAD; stopping there too keeps a malformed one from spinning the kernel.
        if (f == D_DEAD) return D_ROOT;
        s = f;
        r = V.get(s);
    }
}

// ---- one haystack, Standard modes --------------------------------------------------------
// FindIterator / FindOverlappingIterator / FindOverlappingNoSuffixIterator
// (src/bytewise/iter.rs:58-113, 133-176, 195-243; src/charwise/iter.rs:115-170, 190-235, 254-302)
template <bool CHARWISE, int MODE, class SINK>
DACH_HD void scan_standard(const ScanParams& P, const RecView& V, TextWin& T, SINK& E, uint32_t len) {
    const uint32_t root_opos = P.root_opos;
    uint4 root_rec = {0, 0, 0, 0};
    if (CHARWISE) root_rec = V.get(D_ROOT);
    if (MODE == M_OVERLAPPING) emit_chain(P, E, root_opos, 0);
    if (MODE == M_NO_SUFFIX && root_opos) {
        if constexpr (SINK::KIND == RK_HIST) {
            emit_head(P, E, root_opos, 0);
        } else {
            const uint4 o = ld_u4(P.outputs + (root_opos - 1));
            E.emit(P, 0, 0, o.x);  // length 0, end 0 (iter.rs:210-214)
        }
    }
    if constexpr (SINK::KIND == RK_HIST) {
        if (MODE == M_FIND && root_opos) {  // one match of ROOT's record per boundary
            unsigned long long k = 1;
            for (uint32_t pos = 0; pos < len; ++k) {
                if (CHARWISE)
                    (void)utf8_at(T, pos);
                else
                    ++pos;
            }
            red_add_u64(P.rec_hist + (root_opos - 1), k);
            return;
        }
    }
    if (MODE == M_FIND && root_opos) {
        // an empty pattern exists: only zero-length matches, one per boundary (iter.rs:60-85)
        const uint32_t v = ld_u4(P.outputs + (root_opos - 1)).x;
        E.emit(P, 0, 0, v);
        uint32_t pos = 0;
        while (pos < len) {
            if constexpr (SINK::KIND == RK_FIRST) return;  // the first match is (0, 0)
            if (CHARWISE)
                (void)utf8_at(T, pos);
            else
                ++pos;
            E.emit(P, pos, pos, v);
        }
        return;
    }
    uint32_t s = D_ROOT;
    uint4 r = root_rec;
    uint32_t pos = 0;
    while (pos < len) {
        if constexpr (SINK::KIND == RK_FIRST) {
            if (E.stopped()) return;
        }
        if (CHARWISE) {
            const uint32_t cp = utf8_at(T, pos);
            if (s == D_ROOT) r = root_rec;
            s = cw_step<false>(P, V, s, r, cp);
        } else {
            const uint32_t c = T.at(pos++);
            s = bw_step(V, s, r, c);
        }
        if (s != D_ROOT) {
            const uint32_t op = CHARWISE ? r.w : (r.w >> 8);
            if (op != 0) {
                if (MODE == M_OVERLAPPING) {
                    emit_chain(P, E, op, pos);
                } else {
                    emit_head(P, E, op, pos);
                    if (MODE == M_FIND) s = D_ROOT;  // every next() restarts at ROOT (iter.rs:87)
                }
            }
        } else if (MODE == M_OVERLAPPING && root_opos) {
            // ROOT carries the empty pattern: it ends at every position the scan is in ROOT
            emit_chain(P, E, root_opos, pos);
        } else if (MODE == M_NO_SUFFIX && root_opos) {
            emit_head(P, E, root_opos, pos);
        }
    }
}

// ---- one haystack, leftmost --------------------------------------------------------------
// LeftmostFindIterator (src/bytewise/iter.rs:272-340; src/charwise/iter.rs:328-399).  The
// iterator fields (pos, init_output_pos, skip_empty) persist across next() calls; one turn of
// the outer loop is one next().
template <bool CHARWISE, class SINK>
DACH_HD void scan_leftmost(const ScanParams& P, const RecView& V, TextWin& T, SINK& E, uint32_t len) {
    uint32_t self_pos = 0;
    uint32_t init_opos = P.root_opos;
    bool skip_empty = false;
    uint4 root_rec = {0, 0, 0, 0};
    if (CHARWISE) root_rec = V.get(D_ROOT);
    DACH_WD_DECL(wd_outer);
    DACH_WD_DECL(wd_inner);
    for (;;) {
        if constexpr (SINK::KIND == RK_FIRST) {
            if (E.stopped()) return;
        }
        uint32_t s = D_ROOT;
        uint4 r = root_rec;
        uint32_t last = init_opos;
        bool yielded = false;
        uint32_t i = self_pos;
        DACH_WD_TICK(wd_outer, 1000000ull, "WD outer item=%u len=%u self_pos=%u init=%u skip=%d count=%u\n", E.item, len,
                     self_pos, init_opos, (int)skip_empty, E.count)
        while (i < len) {
            DACH_WD_TICK(wd_inner, 100000000ull, "WD inner item=%u len=%u i=%u self_pos=%u s=%u last=%u init=%u\n", E.item,
                         len, i, self_pos, s, last, init_opos)
            const uint32_t unit_start = i;
            if (CHARWISE) {
                const uint32_t cp = utf8_at(T, i);
                if (s == D_ROOT) r = root_rec;
                s = cw_step<true>(P, V, s, r, cp);
            } else {
                const uint32_t c = T.at(i++);
                s = bw_step_leftmost(V, s, r, c);
            }
            if (s == D_ROOT) {
                if (last != 0) {
                    const uint32_t end = self_pos;
                    if (last == init_opos) {
                        self_pos += i - unit_start;  // one byte / one char
                        if (CHARWISE) {  // never stop inside a char (DESIGN.md, "Reference divergences")
                            for (int k = 0; k < 3 && self_pos < len && (T.at(self_pos) & 0xC0u) == 0x80u; ++k) ++self_pos;
                        }
                        if (skip_empty) {
                            skip_empty = false;
                            i = self_pos;  // continue 'a: rescan from the new self.pos
                            continue;
                        }
                    } else {
                        skip_empty = true;
                    }
                    emit_head(P, E, last, end);
                    yielded = true;
                    break;
                }
            } else {
                const uint32_t op = CHARWISE ? r.w : (r.w >> 8);
                if (op != 0) {
                    last = op;
                    self_pos = i;
                }
            }
        }
        if (yielded) continue;
        if (self_pos >= len) init_opos = 0;
        if (last != 0) {
            if (self_pos < len && last == init_opos) {
                // The input ended inside a partial match with only the empty pattern pending.  The
                // crate's iterator returns that empty match without advancing (iter.rs:320-335) and
                // therefore never terminates on such input; a kernel must.  End-of-input is treated
                // like the fall-back-to-ROOT branch (iter.rs:283-293): consume one unit at self.pos
                // and honour skip_empty (DESIGN.md, "Reference divergences").
                const uint32_t end = self_pos;
                if (CHARWISE) {
                    uint32_t t = self_pos;
                    (void)utf8_at(T, t);
                    self_pos = t;
                } else {
                    self_pos += 1;
                }
                if (skip_empty) {
                    skip_empty = false;
                    continue;
                }
                emit_head(P, E, last, end);
                continue;
            }
            emit_head(P, E, last, self_pos);
            continue;
        }
        return;
    }
}


// =============================================================================================
// Lane machine for the bytewise Standard modes (find_overlapping / no_suffix / find without an
// empty pattern).
//
// The per-byte loop of src/bytewise.rs:1063-1088 is re-cut so that every lane of a warp does the
// same thing in every iteration: at most ONE 16-byte record fetch, then a short decision.  Lanes
// walk unrelated haystacks, so a loop shaped like the reference's ("for each byte: while miss:
// follow fail") leaves only a few of 32 lanes active per issued instruction;
// here a lane that misses simply spends its next iteration on the next probe of the same byte.
//
// Compact record (automata with at most 2^24 slots), 16 bytes:
//     w0 = BASE << 8 | CHECK                      src/bytewise.rs:1131-1137
//     w1 = efail << 8 | flags                     flags: CF_OUT (state has an output list),
//                                                        CF_F2ROOT (efail(efail) == ROOT)
//     w2 = fbase << 8 | min(list length, 255)     BASE of efail; the length of the state's output list (0: none),
//                                                 queued with StdMachine3's find_overlapping events.  Readers shift.
//     w3 = child signature: bit (c & 31) is set iff the state has a child labelled c
// The signature answers "no child for this byte" without touching the child slot: on the C3
// workload 0.31 of the 1.28 probes per byte were misses of the state's own children; with it
// almost every fetch is a successful probe (1.03 iterations, 0.99 fetches per byte).
// output_pos lives in a side table (opos[slot]) that is only read when an event is queued.
//
// ROOT is not special-cased by a dense row: a lane that falls to ROOT probes rec[BASE(ROOT) ^ c]
// like any other state (those ~40 records live in L1) and a miss there means "stay in ROOT".
//
// Matches are not expanded in the loop: a lane that lands on a state with an output list stores
// (end, output_pos) in its shared-memory queue -- output_pos arrives by cp.async.  The warp drains
// all queues together (service phase), so the output walk -- a divergent pointer chase -- runs
// with many lanes at once.
//
// Text: two 16-byte register windows per lane (current, next).  Crossing into the next window is
// four predicated moves; the load that re-arms `next` is issued on a warp-uniform schedule (every
// TEXT_TOPUP iterations), early enough because a lane consumes at most one byte per iteration.
// =============================================================================================

#ifndef DACH_LANE_Q
#define DACH_LANE_Q 10
#endif
constexpr int LANE_Q = DACH_LANE_Q;  // queued output events per lane (shared memory)
constexpr int TEXT_TOPUP = 8;  // iterations between window top-ups (must be < 16)
constexpr uint32_t CF_OUT = 1u, CF_F2ROOT = 2u;  // flags in record word 1
constexpr uint32_t COMPACT_MAX_SLOTS = 1u << 24;

// lane flags
constexpr uint32_t F_ACTIVE = 1u, F_DONE = 2u, F_NEED_NW = 4u, F_OWN = 8u, F_ROOTP = 16u, F_PROBE = 32u, F_LEARN = 64u,
                   F_FALL = 128u, F_LAND = 256u;

struct QEntry {
    uint32_t end, opos;  // StdMachine: opos = output_pos, filled asynchronously by cp.async when the event is queued;
                         // StdMachine2 / LmMachine / CwMachine: opos = the slot, output_pos is looked up at drain
};

struct LaneStd {
    const uint8_t* hay;
    uint32_t len, pos, item;
    uint4 cw, nw;  // text windows
    uint32_t c;    // byte being matched
    // the state the lane sits in, as the fields of its compact record
    uint32_t cb;   // BASE (0: no children)
    uint32_t sig;  // child signature
    uint32_t nf;   // raw word 1: efail << 8 | CF_* flags
    uint32_t nfb;  // raw word 2: fbase << 8 | list length
    uint32_t addr; // slot being fetched; after a landing: the slot landed on
    uint32_t qn;   // queued events
    uint32_t fl;   // F_* flags
    uint32_t from; // only matches ending after this position are reported (segment start)
};

struct StdEnv {
    const uint4* glob;     // compact records in global memory (hot-first layout, dev_image.cpp)
    const uint4* hot;      // shared-memory copy of glob[0 .. hot_n): the hot region's leading records
    uint32_t hot_s;        // ... its shared-window address (device code addresses it directly)
    uint32_t hot_n;        // records staged in shared memory (StdMachine3), 0 = none
    const uint32_t* opos;  // output_pos per slot (global)
    const uint8_t* text_end;
    const uint8_t* text_lo;
    uint32_t root_base;    // BASE of ROOT: the child for byte c sits in slot root_base ^ c
    uint32_t root_flags;   // CF_OUT if ROOT has an output list (an empty pattern)
    QEntry* q;             // this lane's queue: entry j at q[j * q_stride]
    uint32_t q_stride;
    uint32_t dbg;
    const uint32_t* mapper;  // charwise: code point -> mapped code (D_INVALID_CODE = unmapped)
    uint32_t mapper_len;
    uint4 root_rec;          // StdMachine2: ROOT's compact record
};

DACH_HD uint4 ld_text16(const uint8_t* q, const uint8_t* text_end, const uint8_t* emu_lo, uint32_t dbg = 0) {
    uint4 w;
    w.x = w.y = w.z = w.w = 0;
    (void)emu_lo;
    (void)dbg;
    if (q >= text_end) return w;  // never touch a block that starts past the text
#if defined(__CUDA_ARCH__)
    // Default: read-only path WITH L1 allocation.  A lane comes back to the same 32-byte sector for
    // its next 16 bytes; with L1::no_allocate every one of those loads goes to L2 or DRAM again.
    asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(w.x), "=r"(w.y), "=r"(w.z), "=r"(w.w)
                 : "l"(q), "l"(c_l2pol[1]));
#elif defined(DACH_EMU)
    uint32_t v[4] = {0, 0, 0, 0};
    for (int i = 0; i < 16; ++i) {
        const uint8_t* qi = q + i;
        uint32_t b = (qi >= emu_lo && qi < text_end) ? *qi : 0;
        v[i >> 2] |= b << ((i & 3) * 8);
    }
    w.x = v[0], w.y = v[1], w.z = v[2], w.w = v[3];
#endif
    return w;
}

#if defined(DACH_EMU)
struct EmuStats {
    unsigned long long steps, probes, hits, miss_known, miss_f2root, learns, root_falls, root_stay, sig_skips, pushes,
        cache_hits;
};
extern EmuStats g_emu_stats;
#define DACH_STAT(f) (++g_emu_stats.f)
#else
#define DACH_STAT(f)
#endif

template <int MODE>
struct StdMachine {
    static constexpr int TOPUP = TEXT_TOPUP;
    static constexpr bool LAZY = false;
    static constexpr bool LEAN = false;
    static constexpr uint32_t IDLE = 0;
    static constexpr bool QLEN = false;
    static DACH_HD void finish_item(const LaneStd&, const ScanParams&) {}
    static DACH_HD const uint8_t* block_of(const LaneStd& L) {
        return reinterpret_cast<const uint8_t*>(((uintptr_t)L.hay + L.pos) & ~(uintptr_t)15);
    }

    // warp-uniform schedule: re-arm the prefetched window of the lanes that crossed since last time
    static DACH_HD void text_topup(LaneStd& L, const StdEnv& Ev, const uint8_t* emu_lo) {
        if ((L.fl & (F_ACTIVE | F_NEED_NW)) == (F_ACTIVE | F_NEED_NW)) {
            L.nw = ld_text16(block_of(L) + 16, Ev.text_end, emu_lo, Ev.dbg);
            L.fl &= ~F_NEED_NW;
        }
    }

    // One iteration, called by all 32 lanes of the warp together.  Returns false if the lane did
    // not step (inactive, finished, or queue full).
    //
    //   phase 1  next byte; the signature decides: probe own children (F_PROBE|F_OWN) or fall (F_FALL)
    //   phase 2  F_FALL: the next probe uses the failure state's BASE, or ROOT's BASE if the failure
    //            state is ROOT (ROOT is probed like any other state; a miss there means "stay in ROOT")
    //   phase 3  the one fetch; a hit adopts the record (F_LAND); a miss of a failure-state probe goes to
    //            ROOT (CF_F2ROOT) or learns the failure state's record first (F_LEARN, rare)
    //   phase 4  F_LAND: consume the byte, move the text window, queue an output event
    //
    // A lane that misses keeps its byte and retries in the next iteration; lanes never wait for each
    // other except in the service phase.  On the C3 workload: 1.03 iterations and 1.0 fetches per byte.
    static DACH_HD bool step(LaneStd& L, const StdEnv& Ev, const uint8_t* emu_lo = nullptr) {
        (void)emu_lo;
        uint32_t fl = L.fl;
        const bool run = (fl & (F_ACTIVE | F_DONE)) == F_ACTIVE && L.qn != (uint32_t)LANE_Q;
        if (run) DACH_STAT(steps);
        // ---- phase 1: next byte ------------------------------------------------------------------
        if (run && (fl & (F_PROBE | F_LEARN | F_FALL)) == 0) {
            if (L.pos >= L.len) {
                fl |= F_DONE;
            } else {
                const uint32_t o = ((uint32_t)(uintptr_t)L.hay + L.pos) & 15u;
                const uint32_t lo = (o & 8u) ? L.cw.z : L.cw.x;
                const uint32_t hi = (o & 8u) ? L.cw.w : L.cw.y;
#if defined(__CUDA_ARCH__)
                const uint32_t c = __byte_perm(lo, hi, o & 7u) & 0xffu;  // byte (o & 7) of the 8-byte half
#else
                const uint32_t c = (((o & 4u) ? hi : lo) >> ((o & 3u) * 8u)) & 0xffu;
#endif
                L.c = c;
                L.addr = L.cb ^ c;
                if ((L.sig >> (c & 31u)) & 1u) {
                    fl |= F_PROBE | F_OWN;
                } else {
                    DACH_STAT(sig_skips);
                    fl |= F_FALL;  // certainly no child for this byte
                }
            }
        }
        DACH_SYNCWARP();
        // ---- phase 2: failure link ------------------------------------------------------------------
        if (fl & F_FALL) {
            const uint32_t f = L.nf >> 8;
            const bool to_root = f == D_ROOT;
            if (to_root) DACH_STAT(root_falls);
            L.addr = (to_root ? Ev.root_base : (L.nfb >> 8)) ^ L.c;
            fl = (fl & ~(F_FALL | F_OWN | F_ROOTP)) | F_PROBE | (to_root ? F_ROOTP : 0u);
        }
        DACH_SYNCWARP();
        // ---- phase 3: the one record fetch ---------------------------------------------------------
        if (run && (fl & (F_PROBE | F_LEARN)) != 0) {
            const uint32_t a = L.addr;
            const uint4 x = ld_u4(Ev.glob + a);
            if (fl & F_PROBE) {
                DACH_STAT(probes);
                // BASE 0 means "no children" (src/bytewise.rs:1075): a ROOT without children is never entered
                if ((x.x & 0xffu) == L.c && !((fl & F_ROOTP) && Ev.root_base == 0)) {  // hit: adopt the record
                    DACH_STAT(hits);
                    L.cb = x.x >> 8;
                    L.nf = x.y;
                    L.nfb = x.z;
                    L.sig = x.w;
                    fl = (fl & ~(F_PROBE | F_OWN | F_ROOTP)) | F_LAND;
                } else if (fl & F_ROOTP) {  // ROOT has no child for this byte: stay in ROOT
                    DACH_STAT(root_stay);
                    L.cb = 0;
                    L.sig = 0;
                    L.nf = Ev.root_flags;  // efail = ROOT
                    L.nfb = 0;
                    L.addr = D_ROOT;
                    fl = (fl & ~(F_PROBE | F_ROOTP)) | F_LAND;
                } else if (fl & F_OWN) {  // signature false positive: take the failure link next
                    DACH_STAT(miss_known);
                    fl = (fl & ~(F_PROBE | F_OWN)) | F_FALL;
                } else if (L.nf & CF_F2ROOT) {  // the failure state's own failure target is ROOT
                    DACH_STAT(miss_f2root);
                    L.nf = 0;  // efail = ROOT
                    fl = (fl & ~F_PROBE) | F_FALL;
                } else {  // need the failure state's record to go on
                    fl = (fl & ~F_PROBE) | F_LEARN;
                    L.addr = L.nf >> 8;
                }
            } else {  // F_LEARN: x is the failure state's record
                DACH_STAT(learns);
                L.nf = x.y;
                L.nfb = x.z;
                fl = (fl & ~F_LEARN) | F_FALL;
            }
        }
        DACH_SYNCWARP();
        // ---- phase 4: land (the byte is consumed; the lane sits in the adopted state) ------------------
        if (fl & F_LAND) {
            fl &= ~F_LAND;
            ++L.pos;
            if ((((uint32_t)(uintptr_t)L.hay + L.pos) & 15u) == 0) {  // crossed into the next window
                L.cw = L.nw;
                fl |= F_NEED_NW;
            }
            if ((L.nf & CF_OUT) && L.pos > L.from) {
                DACH_STAT(pushes);
                QEntry* qe = Ev.q + L.qn * Ev.q_stride;
                qe->end = L.pos;
                // output_pos of the slot goes from the side table straight into the queue entry, off the
                // critical path; the service phase waits for these copies before it reads the entries
#if defined(__CUDA_ARCH__)
                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(&qe->opos)),
                             "l"(Ev.opos + L.addr)
                             : "memory");
#else
                qe->opos = Ev.opos[L.addr];
#endif
                ++L.qn;
                if (MODE == M_FIND) {  // every next() restarts at ROOT (src/bytewise/iter.rs:87)
                    L.cb = 0;
                    L.sig = 0;
                    L.nf = 0;
                    L.nfb = 0;
                }
            }
        }
        L.fl = fl;
        return run;
    }

    // ---- service pieces ---------------------------------------------------------------------------
    static DACH_HD void drain(LaneStd& L, const StdEnv& Ev, const ScanParams& P, Emitter& E) {
#if defined(__CUDA_ARCH__)
        asm volatile("cp.async.wait_all;" ::: "memory");
#endif
        for (uint32_t j = 0; j < (uint32_t)LANE_Q; ++j) {
            if (j < L.qn) {
                const QEntry e = Ev.q[j * Ev.q_stride];
                if (MODE == M_OVERLAPPING)
                    emit_chain(P, E, e.opos, e.end);
                else
                    emit_head(P, E, e.opos, e.end);
            }
        }
        L.qn = 0;
    }

    static DACH_HD void begin_item(LaneStd& L, const ScanParams& P, const StdEnv& Ev, Emitter& E, uint64_t item,
                                   const uint8_t* emu_lo) {
        uint64_t hay = item;
        uint32_t beg = 0;
        if (P.item_hay) {
            hay = P.item_hay[item];
            beg = P.item_beg[item];
        }
        const uint64_t o0 = P.offs[hay], o1 = P.offs[hay + 1];
        const uint32_t hay_len = (uint32_t)(o1 - o0);
        L.hay = P.text + o0;
        L.len = hay_len;
        uint32_t start = 0;
        if (P.item_hay && hay >= P.seg_from) {
            const uint32_t end = beg + P.seg_len;
            L.len = end < hay_len ? end : hay_len;
            start = beg > P.warm ? beg - P.warm : 0;  // warm-up: the state at `beg` only depends on these bytes
        }
        L.pos = start;
        L.from = beg;
        L.item = (uint32_t)item;
        L.qn = 0;
        E.begin((uint32_t)item);
        const uint8_t* b0 = block_of(L);
        L.cw = ld_text16(b0, Ev.text_end, emu_lo, Ev.dbg);
        L.nw = ld_text16(b0 + 16, Ev.text_end, emu_lo, Ev.dbg);
        // the iterator starts in ROOT with ROOT's output list pending at position 0
        // (src/bytewise.rs:303-313; no-suffix variant: src/bytewise/iter.rs:196-216)
        L.cb = 0;
        L.sig = 0;
        L.nf = 0;  // efail = ROOT
        L.nfb = 0;
        L.fl = F_ACTIVE;
        if (MODE != M_FIND && (Ev.root_flags & CF_OUT) && beg == 0) {
            QEntry e;
            e.end = 0;
            e.opos = ld_u32(Ev.opos + D_ROOT);
            Ev.q[0] = e;
            L.qn = 1;
        }
    }
};


// =============================================================================================
// Lane machine for the bytewise leftmost iterator (LeftmostFindIterator,
// src/bytewise/iter.rs:272-340, transitions src/bytewise.rs:1094-1128).
//
// Same four phases and the same compact records as StdMachine; what differs:
//   * a failure link to DEAD ends the chase at ROOT without probing ROOT's children
//     (flags CF_FDEAD-style information travels as efail == DEAD and CF_F2DEAD);
//   * the landing phase runs the iterator's bookkeeping: remember the last state with an output
//     (`last`, `self_pos`), and when the automaton falls back to ROOT report that match (its list
//     head only) and re-scan from the end of the match -- the cursor can move backwards, the text
//     windows are then simply reloaded (those sectors are still in L1);
//   * the empty-pattern rules (`init`, `skip_empty`) and the end-of-input rules of the reference,
//     including the terminating extension documented in DESIGN.md section 1.
// =============================================================================================

constexpr uint32_t CF_F2DEAD = 4u;  // leftmost records: efail(efail) == DEAD
// leftmost iterator flags (LaneLm::it)
constexpr uint32_t F_REPORT = 0x200u, F_FLUSH = 0x400u;  // lane flags of the leftmost machines (phase 5)
constexpr uint32_t IT_INIT = 1u;          // init_output_pos is Some (an empty pattern exists and is still reportable)
constexpr uint32_t IT_HAVE_LAST = 2u;     // last_output_pos is Some
constexpr uint32_t IT_LAST_IS_INIT = 4u;  // ... and it is the empty pattern's
constexpr uint32_t IT_SKIP_EMPTY = 8u;

struct LaneLm : LaneStd {
    uint32_t self_pos;  // self.pos of the iterator
    uint32_t last;      // slot of the last state seen with an output (D_ROOT for the empty pattern)
    uint32_t it;        // IT_* flags
};

struct LmMachine {
    static constexpr int TOPUP = TEXT_TOPUP;
    static constexpr bool LAZY = true;
    static constexpr bool LEAN = false;
    static constexpr uint32_t IDLE = 0;
    static constexpr bool QLEN = false;
    static DACH_HD void finish_item(const LaneLm&, const ScanParams&) {}
    using Std = StdMachine<M_LEFTMOST>;

    static DACH_HD void seek_full(LaneLm& L, const StdEnv& Ev, uint32_t pos, const uint8_t* emu_lo) {
        L.pos = pos;
        const uint8_t* b0 = Std::block_of(L);
        L.cw = ld_text16(b0, Ev.text_end, emu_lo, Ev.dbg);
        L.nw = ld_text16(b0 + 16, Ev.text_end, emu_lo, Ev.dbg);
        L.fl &= ~F_NEED_NW;
    }
    // The cursor goes back to `pos` (the end of the reported match): usually a few bytes, so the windows
    // are kept when `pos` is in the block they hold, and only one block is loaded when it is the one before.
    static DACH_HD void seek(LaneLm& L, const StdEnv& Ev, uint32_t pos, const uint8_t* emu_lo) {
        const uint8_t* cur = Std::block_of(L);
        L.pos = pos;
        const uint8_t* nb = Std::block_of(L);
        if (nb == cur) return;
        if (nb + 16 == cur) {
            L.nw = L.cw;
            L.cw = ld_text16(nb, Ev.text_end, emu_lo, Ev.dbg);
            L.fl &= ~F_NEED_NW;
            return;
        }
        seek_full(L, Ev, pos, emu_lo);
    }

    // start of one next() call: ROOT, last = init, scan from self.pos
    static DACH_HD void restart(LaneLm& L, const StdEnv& Ev, const uint8_t* emu_lo, bool full = false) {
        L.cb = 0;
        L.sig = 0;
        L.nf = 0;
        L.nfb = 0;
        L.last = D_ROOT;
        L.it = (L.it & (IT_INIT | IT_SKIP_EMPTY)) | ((L.it & IT_INIT) ? (IT_HAVE_LAST | IT_LAST_IS_INIT) : 0u);
        if (full)
            seek_full(L, Ev, L.self_pos, emu_lo);
        else
            seek(L, Ev, L.self_pos, emu_lo);
    }

    static DACH_HD void push(LaneLm& L, const StdEnv& Ev, uint32_t end, uint32_t slot) {
        QEntry e;  // (end, slot): output_pos is looked up when the queue is drained
        e.end = end;
        e.opos = slot;
        Ev.q[L.qn * Ev.q_stride] = e;
        ++L.qn;
    }

    // End of one next() call, the only place a match is queued.  F_REPORT: the automaton fell back to ROOT
    // (or the input ended inside a partial match, see DESIGN.md) with a match pending -- the rules of
    // iter.rs:283-306.  F_FLUSH: the input ended (iter.rs:320-339).  Then the next call starts at self.pos.
    static DACH_HD void finish_next(LaneLm& L, const StdEnv& Ev, uint32_t& fl, const uint8_t* emu_lo) {
        const uint32_t end = L.self_pos;
        bool emit = true;
        if (fl & F_REPORT) {
            if (L.it & IT_LAST_IS_INIT) {
                L.self_pos += 1;
                if (L.it & IT_SKIP_EMPTY) {
                    L.it &= ~IT_SKIP_EMPTY;
                    emit = false;  // continue 'a: re-scan from the new self.pos without yielding
                }
            } else {
                L.it |= IT_SKIP_EMPTY;
            }
        }
        if (emit) push(L, Ev, end, L.last);
        L.fl = fl & ~(F_REPORT | F_FLUSH);
        restart(L, Ev, emu_lo);
        fl = L.fl;
    }

    // failure link of the state in L: the next probe, or ROOT at once if the link is DEAD
    // (src/bytewise.rs:1120-1123)
    static DACH_HD void fall(LaneLm& L, const StdEnv& Ev, uint32_t& fl) {
        const uint32_t f = L.nf >> 8;
        if (f == D_DEAD) {
            L.cb = 0;
            L.sig = 0;
            L.nf = 0;
            L.nfb = 0;
            L.addr = D_ROOT;
            fl = (fl & ~(F_PROBE | F_LEARN | F_OWN | F_ROOTP)) | F_LAND;
        } else {
            const bool to_root = f == D_ROOT;
            L.addr = (to_root ? Ev.root_base : (L.nfb >> 8)) ^ L.c;
            fl = (fl & ~(F_LEARN | F_OWN | F_ROOTP)) | F_PROBE | (to_root ? F_ROOTP : 0u);
        }
    }

    static DACH_HD bool step(LaneLm& L, const StdEnv& Ev, const uint8_t* emu_lo) {
        uint32_t fl = L.fl;
        const bool run = (fl & (F_ACTIVE | F_DONE)) == F_ACTIVE && L.qn != (uint32_t)LANE_Q;
        // ---- phase 1: next byte, or the end-of-input rules (iter.rs:320-339) -----------------------
        if (run && (fl & (F_PROBE | F_LEARN | F_FALL)) == 0) {
            if (L.pos >= L.len) {
                if (L.self_pos == L.len) L.it &= ~IT_INIT;
                if (L.it & IT_HAVE_LAST) {
                    // input ended inside a partial match with only the empty pattern pending: the reference
                    // never terminates here; treated like the fall-back-to-ROOT branch (F_REPORT)
                    fl |= (L.self_pos < L.len && (L.it & IT_LAST_IS_INIT)) ? F_REPORT : F_FLUSH;
                } else {
                    fl |= F_DONE;
                }
            } else {
                const uint32_t o = ((uint32_t)(uintptr_t)L.hay + L.pos) & 15u;
                const uint32_t lo = (o & 8u) ? L.cw.z : L.cw.x;
                const uint32_t hi = (o & 8u) ? L.cw.w : L.cw.y;
#if defined(__CUDA_ARCH__)
                const uint32_t c = __byte_perm(lo, hi, o & 7u) & 0xffu;
#else
                const uint32_t c = (((o & 4u) ? hi : lo) >> ((o & 3u) * 8u)) & 0xffu;
#endif
                L.c = c;
                if ((L.sig >> (c & 31u)) & 1u) {
                    L.addr = L.cb ^ c;
                    fl |= F_PROBE | F_OWN;
                } else {
                    fall(L, Ev, fl);  // certainly no child for this byte
                }
            }
        }
        DACH_SYNCWARP();
        // ---- phase 3: the one record fetch ---------------------------------------------------------
        if (run && (fl & (F_PROBE | F_LEARN)) != 0) {
            const uint4 x = ld_u4(Ev.glob + L.addr);
            if (fl & F_PROBE) {
                if ((x.x & 0xffu) == L.c && !((fl & F_ROOTP) && Ev.root_base == 0)) {
                    L.cb = x.x >> 8;
                    L.nf = x.y;
                    L.nfb = x.z;
                    L.sig = x.w;
                    fl = (fl & ~(F_PROBE | F_OWN | F_ROOTP)) | F_LAND;
                } else if ((fl & F_ROOTP) || (!(fl & F_OWN) && (L.nf & CF_F2DEAD))) {
                    // ROOT has no such child, or the failure state's own failure link is DEAD: ROOT
                    L.cb = 0;
                    L.sig = 0;
                    L.nf = 0;
                    L.nfb = 0;
                    L.addr = D_ROOT;
                    fl = (fl & ~(F_PROBE | F_ROOTP)) | F_LAND;
                } else if (fl & F_OWN) {
                    fall(L, Ev, fl);
                } else if (L.nf & CF_F2ROOT) {
                    L.nf = 0;
                    fall(L, Ev, fl);
                } else {
                    fl = (fl & ~F_PROBE) | F_LEARN;
                    L.addr = L.nf >> 8;
                }
            } else {  // F_LEARN
                L.nf = x.y;
                L.nfb = x.z;
                fall(L, Ev, fl);
            }
        }
        DACH_SYNCWARP();
        // ---- phase 4: land and run the iterator's bookkeeping (iter.rs:282-315) -----------------------
        if (fl & F_LAND) {
            fl &= ~F_LAND;
            ++L.pos;
            if ((((uint32_t)(uintptr_t)L.hay + L.pos) & 15u) == 0) {
                L.cw = L.nw;
                fl |= F_NEED_NW;
            }
            if (L.addr == D_ROOT) {
                if (L.it & IT_HAVE_LAST) fl |= F_REPORT;
            } else if (L.nf & CF_OUT) {
                L.last = L.addr;
                L.it = (L.it | IT_HAVE_LAST) & ~IT_LAST_IS_INIT;
                L.self_pos = L.pos;
            }
        }
        // ---- phase 5: a next() call ends ---------------------------------------------------------------
        if (fl & (F_REPORT | F_FLUSH)) finish_next(L, Ev, fl, emu_lo);
        L.fl = fl;
        return run;
    }

    static DACH_HD void drain(LaneLm& L, const StdEnv& Ev, const ScanParams& P, Emitter& E) {
        for (uint32_t j = 0; j < (uint32_t)LANE_Q; ++j) {
            if (j < L.qn) {
                const QEntry e = Ev.q[j * Ev.q_stride];
                emit_head(P, E, ld_u32(Ev.opos + e.opos), e.end);
            }
        }
        L.qn = 0;
    }

    static DACH_HD void text_topup(LaneLm& L, const StdEnv& Ev, const uint8_t* emu_lo) { Std::text_topup(L, Ev, emu_lo); }

    static DACH_HD void begin_item(LaneLm& L, const ScanParams& P, const StdEnv& Ev, Emitter& E, uint64_t item,
                                   const uint8_t* emu_lo) {
        const uint64_t o0 = P.offs[item], o1 = P.offs[item + 1];
        L.hay = P.text + o0;
        L.len = (uint32_t)(o1 - o0);
        L.from = 0;
        L.item = (uint32_t)item;
        L.qn = 0;
        L.fl = F_ACTIVE;
        L.self_pos = 0;
        L.it = (Ev.root_flags & CF_OUT) ? IT_INIT : 0u;
        E.begin((uint32_t)item);
        restart(L, Ev, emu_lo, true);
    }
};

// =============================================================================================
// Lane machine for the charwise automaton, all four iterators (src/charwise/iter.rs:115-399,
// transitions src/charwise.rs:1022-1092).
//
// One iteration consumes one char.  Phase 1 decodes it from the register windows (up to four bytes,
// src/charwise/iter.rs:71-97) and maps the code point (src/charwise/mapper.rs:36-42; an unmapped
// char sends the automaton straight to ROOT); phases 2-4 are those of the bytewise machines.
// CHECK of a charwise state is its parent's id, so a probe hits when the fetched record names the
// state the probe was made from (the lane's own state, the failure state, or ROOT).
//
// Compact record (at most 2^24 - 1 slots), 16 bytes:
//     w0 = BASE << 8  | signature bits 0..7        src/charwise.rs:1132-1160
//     w1 = efail << 8 | flags (CF_OUT, CF_F2ROOT, CF_F2DEAD)
//     w2 = fbase << 8 | signature bits 8..15
//     w3 = CHECK << 8
// signature: bit (mapped code & 15) is set iff the state has a child with that code.
//
// The windows are re-armed every TOPUP = 4 iterations: a lane consumes at most 16 bytes in between,
// i.e. crosses at most one 16-byte block, and after the crossing the next three decodes stay inside
// the block that became current.
// =============================================================================================

struct LaneCw : LaneLm {
    uint32_t cur;   // slot of the state the lane sits in
    uint32_t ulen;  // bytes of the char being matched
};

template <int MODE>
struct CwMachine {
    static constexpr int TOPUP = 4;
    static constexpr bool LAZY = true;
    static constexpr bool LEAN = false;
    static constexpr uint32_t IDLE = 0;
    static constexpr bool QLEN = false;
    // the item is complete: hand the state on to the next chunk of the stream (the charwise steppers,
    // src/charwise/iter.rs:403-534; the charwise image keeps the crate's state ids)
    static DACH_HD void finish_item(const LaneCw& L, const ScanParams& P) {
        if (P.state_io) P.state_io[L.item] = L.cur;
    }
    static constexpr bool LM = MODE == M_LEFTMOST;
    using Std = StdMachine<M_OVERLAPPING>;

    // the four bytes at L.pos, little endian (bytes past the windows' 32 are never needed)
    static DACH_HD uint32_t peek4(const LaneCw& L) {
        const uint32_t o = ((uint32_t)(uintptr_t)L.hay + L.pos) & 15u;
        const uint32_t a = (o & 8u) ? L.cw.z : L.cw.x;
        const uint32_t b = (o & 8u) ? L.cw.w : L.cw.y;
        const uint32_t d = (o & 8u) ? L.nw.x : L.cw.z;
        const uint32_t lo = (o & 4u) ? b : a;
        const uint32_t hi = (o & 4u) ? d : b;
        const uint32_t sh = (o & 3u) * 8u;
#if defined(__CUDA_ARCH__)
        return __funnelshift_r(lo, hi, sh);
#else
        return sh ? (lo >> sh) | (hi << (32u - sh)) : lo;
#endif
    }
    static DACH_HD uint32_t utf8_len(uint32_t first) { return first < 0x80u ? 1u : first < 0xe0u ? 2u : first < 0xf0u ? 3u : 4u; }
    static DACH_HD uint32_t utf8_cp(uint32_t u, uint32_t n) {
        const uint32_t first = u & 0xffu, b1 = (u >> 8) & 0x3fu, b2 = (u >> 16) & 0x3fu, b3 = (u >> 24) & 0x3fu;
        const uint32_t c2 = ((first & 0x1fu) << 6) | b1;
        const uint32_t c3 = ((first & 0x0fu) << 12) | (b1 << 6) | b2;
        const uint32_t c4 = ((first & 0x07u) << 18) | (b1 << 12) | (b2 << 6) | b3;
        return n == 1u ? first : n == 2u ? c2 : n == 3u ? c3 : c4;
    }

    static DACH_HD void set_root(LaneCw& L, const StdEnv& Ev) {
        L.cb = 0;
        L.sig = 0;
        L.nf = LM ? 0u : Ev.root_flags;  // efail = ROOT
        L.nfb = 0;
        L.addr = D_ROOT;
    }

    static DACH_HD void seek_full(LaneCw& L, const StdEnv& Ev, uint32_t pos, const uint8_t* emu_lo) {
        L.pos = pos;
        const uint8_t* b0 = Std::block_of(L);
        L.cw = ld_text16(b0, Ev.text_end, emu_lo, Ev.dbg);
        L.nw = ld_text16(b0 + 16, Ev.text_end, emu_lo, Ev.dbg);
        L.fl &= ~F_NEED_NW;
    }
    // the cursor goes back a few bytes: keep the windows when they still hold `pos` (see LmMachine::seek)
    static DACH_HD void seek(LaneCw& L, const StdEnv& Ev, uint32_t pos, const uint8_t* emu_lo) {
        const uint8_t* cur = Std::block_of(L);
        const bool nw_stale = (L.fl & F_NEED_NW) != 0;
        L.pos = pos;
        const uint8_t* nb = Std::block_of(L);
        if (nb == cur && !nw_stale) return;
        if (nb + 16 == cur) {
            L.nw = L.cw;
            L.cw = ld_text16(nb, Ev.text_end, emu_lo, Ev.dbg);
            L.fl &= ~F_NEED_NW;
            return;
        }
        seek_full(L, Ev, pos, emu_lo);
    }

    static DACH_HD void restart(LaneCw& L, const StdEnv& Ev, const uint8_t* emu_lo, bool full = false) {
        L.cb = 0;
        L.sig = 0;
        L.nf = 0;
        L.nfb = 0;
        L.cur = D_ROOT;
        L.last = D_ROOT;
        L.it = (L.it & (IT_INIT | IT_SKIP_EMPTY)) | ((L.it & IT_INIT) ? (IT_HAVE_LAST | IT_LAST_IS_INIT) : 0u);
        if (full)
            seek_full(L, Ev, L.self_pos, emu_lo);
        else
            seek(L, Ev, L.self_pos, emu_lo);
    }

    static DACH_HD void push(LaneCw& L, const StdEnv& Ev, uint32_t end, uint32_t slot) {
        QEntry e;  // (end, slot): output_pos is looked up when the queue is drained
        e.end = end;
        e.opos = slot;
        Ev.q[L.qn * Ev.q_stride] = e;
        ++L.qn;
    }

    // End of one next() call, the only place a leftmost match is queued (see LmMachine::finish_next).
    // F_REPORT: src/charwise/iter.rs:345-366 with adv = L.ulen, the bytes of the char that led back to ROOT.
    static DACH_HD void finish_next(LaneCw& L, const StdEnv& Ev, uint32_t& fl, const uint8_t* emu_lo) {
        const uint32_t end = L.self_pos;
        bool emit = true;
        bool snap = false;
        if (fl & F_REPORT) {
            if (L.it & IT_LAST_IS_INIT) {
                L.self_pos += L.ulen;
                snap = true;
                if (L.it & IT_SKIP_EMPTY) {
                    L.it &= ~IT_SKIP_EMPTY;
                    emit = false;
                }
            } else {
                L.it |= IT_SKIP_EMPTY;
            }
        }
        if (emit) push(L, Ev, end, L.last);
        L.fl = fl & ~(F_REPORT | F_FLUSH);
        restart(L, Ev, emu_lo);
        if (snap && L.self_pos < L.len) {
            // the advance belongs to the char that fell back to ROOT, not to the one at self_pos: never stop
            // inside a char (DESIGN.md, "Reference divergences") -- skip at most 3 continuation bytes
            const uint32_t u = peek4(L);
            uint32_t k = 0;
            while (k < 3u && L.self_pos + k < L.len && ((u >> (8u * k)) & 0xC0u) == 0x80u) ++k;
            if (k) {
                L.self_pos += k;
                seek(L, Ev, L.self_pos, emu_lo);
            }
        }
        fl = L.fl;
    }

    // failure link of the state in L: the next probe, or ROOT at once if the link is DEAD
    static DACH_HD void fall(LaneCw& L, const StdEnv& Ev, uint32_t& fl) {
        const uint32_t f = L.nf >> 8;
        if (f == D_DEAD) {
            set_root(L, Ev);
            fl = (fl & ~(F_PROBE | F_LEARN | F_OWN | F_ROOTP)) | F_LAND;
        } else {
            const bool to_root = f == D_ROOT;
            L.addr = (to_root ? Ev.root_base : (L.nfb >> 8)) ^ L.c;
            fl = (fl & ~(F_LEARN | F_OWN | F_ROOTP)) | F_PROBE | (to_root ? F_ROOTP : 0u);
        }
    }

    static DACH_HD bool step(LaneCw& L, const StdEnv& Ev, const uint8_t* emu_lo) {
        (void)emu_lo;
        uint32_t fl = L.fl;
        const bool run = (fl & (F_ACTIVE | F_DONE)) == F_ACTIVE && L.qn != (uint32_t)LANE_Q;
        // ---- phase 1: next char ----------------------------------------------------------------------
        if (run && (fl & (F_PROBE | F_LEARN | F_FALL)) == 0) {
            if (L.pos >= L.len) {
                if (!LM) {
                    fl |= F_DONE;
                } else {  // end-of-input rules (src/charwise/iter.rs:381-398), as in LmMachine
                    if (L.self_pos >= L.len) L.it &= ~IT_INIT;
                    if (L.it & IT_HAVE_LAST) {
                        if (L.self_pos < L.len && (L.it & IT_LAST_IS_INIT)) {
                            L.fl = fl;  // the unit consumed is the char at self_pos
                            seek(L, Ev, L.self_pos, emu_lo);
                            fl = L.fl;
                            L.ulen = utf8_len(peek4(L) & 0xffu);
                            fl |= F_REPORT;
                        } else {
                            fl |= F_FLUSH;
                        }
                    } else {
                        fl |= F_DONE;
                    }
                }
            } else {
                const uint32_t u = peek4(L);
                const uint32_t n = utf8_len(u & 0xffu);
                const uint32_t cp = utf8_cp(u, n);
                L.ulen = n;
                const uint32_t mc = cp < Ev.mapper_len ? ld_u32(Ev.mapper + cp) : D_INVALID_CODE;
                if (mc == D_INVALID_CODE) {  // unmapped char: ROOT (src/charwise.rs:1030-1032)
                    set_root(L, Ev);
                    fl |= F_LAND;
                } else {
                    L.c = mc;
                    if ((L.sig >> (mc & 15u)) & 1u) {
                        L.addr = L.cb ^ mc;
                        fl |= F_PROBE | F_OWN;
                    } else {
                        fall(L, Ev, fl);  // certainly no child for this code
                    }
                }
            }
        }
        DACH_SYNCWARP();
        // ---- phase 3: the one record fetch ---------------------------------------------------------
        if (run && (fl & (F_PROBE | F_LEARN)) != 0) {
            const uint4 x = ld_u4(Ev.glob + L.addr);
            if (fl & F_PROBE) {
                const uint32_t expect = (fl & F_OWN) ? L.cur : (fl & F_ROOTP) ? D_ROOT : (L.nf >> 8);
                if ((x.w >> 8) == expect && !((fl & F_ROOTP) && Ev.root_base == 0)) {
                    L.cb = x.x >> 8;
                    L.sig = (x.x & 0xffu) | ((x.z & 0xffu) << 8);
                    L.nf = x.y;
                    L.nfb = x.z;
                    fl = (fl & ~(F_PROBE | F_OWN | F_ROOTP)) | F_LAND;
                } else if ((fl & F_ROOTP) || (!(fl & F_OWN) && (L.nf & CF_F2DEAD))) {
                    set_root(L, Ev);
                    fl = (fl & ~(F_PROBE | F_ROOTP)) | F_LAND;
                } else if (fl & F_OWN) {
                    fall(L, Ev, fl);
                } else if (L.nf & CF_F2ROOT) {
                    L.nf = 0;
                    fall(L, Ev, fl);
                } else {
                    fl = (fl & ~F_PROBE) | F_LEARN;
                    L.addr = L.nf >> 8;
                }
            } else {  // F_LEARN
                L.nf = x.y;
                L.nfb = x.z;
                fall(L, Ev, fl);
            }
        }
        DACH_SYNCWARP();
        // ---- phase 4: land ------------------------------------------------------------------------------
        if (fl & F_LAND) {
            fl &= ~F_LAND;
            const uint32_t a0 = (uint32_t)(uintptr_t)L.hay + L.pos;
            L.pos += L.ulen;
            if ((a0 ^ (a0 + L.ulen)) & 16u) {  // crossed into the next window
                L.cw = L.nw;
                fl |= F_NEED_NW;
            }
            L.cur = L.addr;
            if (LM) {
                if (L.addr == D_ROOT) {
                    if (L.it & IT_HAVE_LAST) fl |= F_REPORT;
                } else if (L.nf & CF_OUT) {
                    L.last = L.addr;
                    L.it = (L.it | IT_HAVE_LAST) & ~IT_LAST_IS_INIT;
                    L.self_pos = L.pos;
                }
            } else if (L.nf & CF_OUT) {
                push(L, Ev, L.pos, L.addr);
                if (MODE == M_FIND) {  // every next() restarts at ROOT (src/charwise/iter.rs:150)
                    L.cb = 0;
                    L.sig = 0;
                    L.nf = 0;
                    L.nfb = 0;
                    L.cur = D_ROOT;
                }
            }
        }
        // ---- phase 5 (leftmost): a next() call ends --------------------------------------------------------
        if (LM && (fl & (F_REPORT | F_FLUSH))) finish_next(L, Ev, fl, emu_lo);
        L.fl = fl;
        return run;
    }

    static DACH_HD void drain(LaneCw& L, const StdEnv& Ev, const ScanParams& P, Emitter& E) {
        for (uint32_t j = 0; j < (uint32_t)LANE_Q; ++j) {
            if (j < L.qn) {
                const QEntry e = Ev.q[j * Ev.q_stride];
                const uint32_t opos = ld_u32(Ev.opos + e.opos);
                if (MODE == M_OVERLAPPING)
                    emit_chain(P, E, opos, e.end);
                else
                    emit_head(P, E, opos, e.end);
            }
        }
        L.qn = 0;
    }

    static DACH_HD void text_topup(LaneCw& L, const StdEnv& Ev, const uint8_t* emu_lo) { Std::text_topup(L, Ev, emu_lo); }

    static DACH_HD void begin_item(LaneCw& L, const ScanParams& P, const StdEnv& Ev, Emitter& E, uint64_t item,
                                   const uint8_t* emu_lo) {
        const uint64_t o0 = P.offs[item], o1 = P.offs[item + 1];
        L.hay = P.text + o0;
        L.len = (uint32_t)(o1 - o0);
        L.from = 0;
        L.item = (uint32_t)item;
        L.qn = 0;
        L.fl = F_ACTIVE;
        L.ulen = 0;
        L.self_pos = 0;
        L.it = (LM && (Ev.root_flags & CF_OUT)) ? IT_INIT : 0u;
        E.begin((uint32_t)item);
        restart(L, Ev, emu_lo, true);
        if (!LM && P.state_io) {
            // a chunk of a stream (whole chars): resume in the state the previous chunk ended in; the outputs of
            // that state were reported with the previous chunk
            const uint32_t st = P.state_io[item];
            if (st != D_ROOT && st < P.n_slots) {
                const uint4 x = ld_u4(Ev.glob + st);
                L.cb = x.x >> 8;
                L.sig = (x.x & 0xffu) | ((x.z & 0xffu) << 8);
                L.nf = x.y;
                L.nfb = x.z;
                L.cur = st;
                L.addr = st;
            }
            return;
        }
        if (!LM && MODE != M_FIND && (Ev.root_flags & CF_OUT)) {  // ROOT's output list is pending at position 0
            QEntry e;
            e.end = 0;
            e.opos = D_ROOT;
            Ev.q[0] = e;
            L.qn = 1;
        }
    }
};

// =============================================================================================
// StdMachine2: the bytewise Standard machine again, cut for instruction count (the kernel is
// issue-bound as much as latency-bound).
//
//   * three phases instead of four: a miss computes the address of its next probe on the spot;
//     fbase of a state whose failure target is ROOT is ROOT's BASE (pre-resolved in the image,
//     flag CF_FROOT), so "sig says no child" is one select: probe (own ? BASE : fbase) ^ c;
//   * ROOT is an ordinary state: its compact record is kept in registers and adopted when the
//     chase ends there (needs BASE(ROOT) != 0; otherwise the launcher keeps StdMachine);
//   * text: a 64-bit shift register (current 8 bytes, low byte = the byte being matched -- it feeds
//     the signature shift, the address XOR and the CHECK compare without being extracted) plus the
//     next 8 bytes, re-armed on the same warp-uniform schedule.
// =============================================================================================

constexpr uint32_t CF_FROOT = 8u;  // efail == ROOT (Standard records)
constexpr uint32_t S2_OWN = 0x10u, S2_FAIL = 0x20u, S2_ROOT = 0x40u, S2_LEARN = 0x80u, S2_BUSY = 0xf0u, S2_LAND = 0x100u,
                   S2_FULL = 0x200u;

struct Lane2 {
    const uint8_t* hay;
    uint32_t len, pos, item;
    uint32_t w0, w1, n0, n1;  // text: current 8 bytes (shifted), next 8 bytes
    uint32_t r0, nf, r2, sig; // the state the lane sits in: raw words of its compact record
    uint32_t addr, qn, fl, from;
};

DACH_HD uint2 ld_text8(const uint8_t* q, const uint8_t* text_end, const uint8_t* emu_lo) {
    uint2 w;
    w.x = w.y = 0;
    (void)emu_lo;
    if (q >= text_end) return w;
#if defined(__CUDA_ARCH__)
    asm volatile("ld.global.nc.L2::cache_hint.v2.u32 {%0,%1}, [%2], %3;" : "=r"(w.x), "=r"(w.y) : "l"(q), "l"(c_l2pol[1]));
#elif defined(DACH_EMU)
    uint32_t v[2] = {0, 0};
    for (int i = 0; i < 8; ++i) {
        const uint8_t* qi = q + i;
        uint32_t b = (qi >= emu_lo && qi < text_end) ? *qi : 0;
        v[i >> 2] |= b << ((i & 3) * 8);
    }
    w.x = v[0], w.y = v[1];
#endif
    return w;
}

template <int MODE>
struct StdMachine2 {
    static constexpr int TOPUP = 8;
    static constexpr bool LAZY = true;
    static constexpr bool LEAN = false;
    static constexpr uint32_t IDLE = 0;
    static constexpr bool QLEN = false;

    static DACH_HD const uint8_t* block_of(const Lane2& L) {
        return reinterpret_cast<const uint8_t*>(((uintptr_t)L.hay + L.pos) & ~(uintptr_t)7);
    }
    static DACH_HD void text_topup(Lane2& L, const StdEnv& Ev, const uint8_t* emu_lo) {
        if ((L.fl & (F_ACTIVE | F_NEED_NW)) == (F_ACTIVE | F_NEED_NW)) {
            const uint2 n = ld_text8(block_of(L) + 8, Ev.text_end, emu_lo);
            L.n0 = n.x;
            L.n1 = n.y;
            L.fl &= ~F_NEED_NW;
        }
    }
    static DACH_HD void to_root(Lane2& L, const StdEnv& Ev) {
        L.r0 = Ev.root_rec.x;
        L.nf = Ev.root_rec.y;
        L.r2 = Ev.root_rec.z;
        L.sig = Ev.root_rec.w;
    }

    // the byte is consumed; the lane sits in the state whose record it just adopted
    static DACH_HD void land(Lane2& L, const StdEnv& Ev, uint32_t& fl) {
        ++L.pos;
        L.w0 = (L.w0 >> 8) | (L.w1 << 24);
        L.w1 >>= 8;
        if ((((uint32_t)(uintptr_t)L.hay + L.pos) & 7u) == 0) {  // the next 8 bytes become current
            L.w0 = L.n0;
            L.w1 = L.n1;
            fl |= F_NEED_NW;
        }
        if ((L.nf & CF_OUT) && L.pos > L.from) {
            // one 8-byte store: (end, slot).  output_pos is looked up when the queue is drained -- this block
            // runs with ~1.5 of 32 lanes active in three of four iterations, so it has to be short
            QEntry e;
            e.end = L.pos;
            e.opos = L.addr;
            Ev.q[L.qn * Ev.q_stride] = e;
            ++L.qn;
            if (L.qn == (uint32_t)LANE_Q) fl |= S2_FULL;
            if (MODE == M_FIND) {  // every next() restarts at ROOT (src/bytewise/iter.rs:87)
                to_root(L, Ev);
                L.addr = D_ROOT;
            }
        }
    }

    static DACH_HD bool step(Lane2& L, const StdEnv& Ev, const uint8_t* emu_lo = nullptr) {
        (void)emu_lo;
        uint32_t fl = L.fl;
        const bool run = (fl & (F_ACTIVE | F_DONE | S2_FULL)) == F_ACTIVE;
        // ---- phase A: next byte, first probe address ---------------------------------------------------
        if (run && (fl & S2_BUSY) == 0) {
            if (L.pos >= L.len) {
                fl |= F_DONE;
            } else {
                const uint32_t own = (L.sig >> (L.w0 & 31u)) & 1u;
                L.addr = ((own ? L.r0 : L.r2) >> 8) ^ (L.w0 & 0xffu);
                fl |= S2_FAIL >> own;  // S2_OWN == S2_FAIL >> 1
            }
        }
        DACH_SYNCWARP();
        // ---- phase B: the one record fetch; a hit lands at once ----------------------------------------
        if (run && (fl & S2_BUSY) != 0) {
            const uint4 x = ld_u4(Ev.glob + L.addr);
            if ((((x.x ^ L.w0) & 0xffu) | (fl & S2_LEARN)) == 0) {  // CHECK == c: adopt the record
                L.r0 = x.x;
                L.nf = x.y;
                L.r2 = x.z;
                L.sig = x.w;
                fl &= ~S2_BUSY;
                land(L, Ev, fl);
            } else {
                const uint32_t c = L.w0 & 0xffu;
                if (fl & S2_OWN) {  // signature false positive (the common miss): probe the failure state's children
                    L.addr = (L.r2 >> 8) ^ c;
                    fl ^= S2_OWN | S2_FAIL;
                } else if (fl & S2_LEARN) {  // x is the failure state's record
                    L.nf = x.y;
                    L.r2 = x.z;
                    L.addr = (x.z >> 8) ^ c;
                    fl ^= S2_LEARN | S2_FAIL;
                } else if ((fl & S2_ROOT) || (L.nf & CF_FROOT)) {  // ROOT has no such child: stay in ROOT
                    to_root(L, Ev);
                    L.addr = D_ROOT;
                    fl &= ~S2_BUSY;
                    land(L, Ev, fl);
                } else if (L.nf & CF_F2ROOT) {  // the failure state's own failure target is ROOT
                    L.addr = Ev.root_base ^ c;
                    fl ^= S2_FAIL | S2_ROOT;
                } else {  // need the failure state's record to go on
                    L.addr = L.nf >> 8;
                    fl ^= S2_FAIL | S2_LEARN;
                }
            }
        }
        L.fl = fl;
        return run;
    }

    static DACH_HD void drain(Lane2& L, const StdEnv& Ev, const ScanParams& P, Emitter& E) {
        for (uint32_t j = 0; j < (uint32_t)LANE_Q; ++j) {
            if (j < L.qn) {
                const QEntry e = Ev.q[j * Ev.q_stride];
                const uint32_t opos = ld_u32(Ev.opos + e.opos);  // the entry holds the slot
                if (MODE == M_OVERLAPPING)
                    emit_chain(P, E, opos, e.end);
                else
                    emit_head(P, E, opos, e.end);
            }
        }
        L.qn = 0;
        L.fl &= ~S2_FULL;
    }

    // the item is complete (its last byte landed): hand the state on to the next chunk of the stream
    static DACH_HD void finish_item(const Lane2& L, const ScanParams& P) {
        if (P.state_io) P.state_io[L.item] = P.id_out ? P.id_out[L.addr] : L.addr;
    }

    static DACH_HD void begin_item(Lane2& L, const ScanParams& P, const StdEnv& Ev, Emitter& E, uint64_t item,
                                   const uint8_t* emu_lo) {
        uint64_t hay = item;
        uint32_t beg = 0;
        if (P.item_hay) {
            hay = P.item_hay[item];
            beg = P.item_beg[item];
        }
        const uint64_t o0 = P.offs[hay], o1 = P.offs[hay + 1];
        const uint32_t hay_len = (uint32_t)(o1 - o0);
        L.hay = P.text + o0;
        L.len = hay_len;
        uint32_t start = 0;
        if (P.item_hay && hay >= P.seg_from) {
            const uint32_t end = beg + P.seg_len;
            L.len = end < hay_len ? end : hay_len;
            start = beg > P.warm ? beg - P.warm : 0;
        }
        L.pos = start;
        L.from = beg;
        L.item = (uint32_t)item;
        L.qn = 0;
        E.begin((uint32_t)item);
        const uint8_t* b0 = block_of(L);
        const uint2 a = ld_text8(b0, Ev.text_end, emu_lo);
        const uint2 n = ld_text8(b0 + 8, Ev.text_end, emu_lo);
        const uint32_t sh = (((uint32_t)(uintptr_t)L.hay + L.pos) & 7u) * 8u;  // the byte at pos goes to bit 0
        const uint64_t cur = (((uint64_t)a.y << 32) | a.x) >> sh;
        L.w0 = (uint32_t)cur;
        L.w1 = (uint32_t)(cur >> 32);
        L.n0 = n.x;
        L.n1 = n.y;
        to_root(L, Ev);
        L.addr = D_ROOT;
        L.fl = F_ACTIVE;
        if (P.state_io) {
            // a chunk of a stream: resume in the state the previous chunk ended in (the stepper contract,
            // src/bytewise/iter.rs:344-475); the outputs of that state were reported with the previous chunk
            uint32_t st = P.state_io[item];
            if (st != D_ROOT && st < P.n_slots) {
                if (P.id_in) st = P.id_in[st];
                const uint4 x = ld_u4(Ev.glob + st);
                L.r0 = x.x;
                L.nf = x.y;
                L.r2 = x.z;
                L.sig = x.w;
                L.addr = st;
            }
            return;
        }
        if (MODE != M_FIND && (Ev.root_flags & CF_OUT) && beg == 0) {
            QEntry e;
            e.end = 0;
            e.opos = D_ROOT;
            Ev.q[0] = e;
            L.qn = 1;
        }
    }
};

// =============================================================================================
// StdMachine3: the bytewise Standard machine, third cut -- the default.
//
// StdMachine2 sits on two ceilings at once: the L1 data pipe (every lane's record
// fetch is its own wavefront) and the issue slots (98 warp instructions per lock-step iteration).
// This cut attacks both:
//   * records come from the hot-first image (dev_image.cpp): the leading Ev.hot_n slots are staged
//     in shared memory and served from there by a plain prefix compare -- no tag, no dependent
//     lookup; a warp's 32 random 16-byte reads cost ~10 shared-memory wavefronts instead of 32 L1 ones;
//   * no probe-state flags: a missed own-child probe (signature false positive) clears the
//     signature bit of that byte, a missed failure probe rewrites (nf, r2) in place, so every
//     iteration is the same "probe, compare, adopt" and the rare paths leave no trace in the loop;
//   * one stop bit (haystack finished or queue full) replaces the per-iteration bookkeeping; the
//     service vote reads it once per period;
//   * the cursor is the low address word of the byte being matched: the same register answers
//     "window boundary?", "end of haystack?" and, minus the haystack's low address word, the match end;
//   * the segment filter (only matches ending inside the segment) moved out of the loop to the drain.
// Semantics are StdMachine2's (src/bytewise.rs:1063-1088, src/bytewise/iter.rs:58-243, 344-475).
// =============================================================================================

constexpr uint32_t F3_STOP = 0x10u;   // the lane does not step: idle, finished, or its queue is full
constexpr uint32_t F3_LEARN = 0x20u;  // the record being fetched is the failure state's: take its (efail, fbase) and go on

struct Lane3 {
    uint32_t hay_lo, hay_hi;  // address of the haystack's first byte
    uint32_t ap, ap_end;      // low address word of the byte being matched / of one past the item's last byte
    uint32_t w0, w1, n0, n1;  // text: current 8 bytes (shifted: the low byte is the one being matched), next 8 bytes
    uint32_t r0, nf, r2, sig; // the state the lane sits in: raw words of its compact record
    uint32_t addr;            // the slot landed on
    uint32_t qn, fl, item;
    uint32_t from;            // drain: only events with end >= from are reported (segment start + 1, or 0)
};

// 8 text bytes at the 8-aligned address q; bytes outside [text_lo, text_end) read as 0 and are never touched
DACH_HD uint2 ld_text8_safe(const uint8_t* q, const uint8_t* text_lo, const uint8_t* text_end) {
    uint2 w;
    w.x = w.y = 0;
    if (q >= text_end || q + 8 <= text_lo) return w;
    if (q >= text_lo && q + 8 <= text_end) {
#if defined(__CUDA_ARCH__)
        asm volatile("ld.global.nc.L2::cache_hint.v2.u32 {%0,%1}, [%2], %3;" : "=r"(w.x), "=r"(w.y) : "l"(q), "l"(c_l2pol[1]));
#else
        for (int i = 0; i < 8; ++i) (i < 4 ? w.x : w.y) |= (uint32_t)q[i] << ((i & 3) * 8);
#endif
        return w;
    }
    for (int i = 0; i < 8; ++i) {  // first or last block of the batch: byte by byte
        const uint8_t* qi = q + i;
        if (qi >= text_lo && qi < text_end) {
#if defined(__CUDA_ARCH__)
            const uint32_t b = __ldg(qi);
#else
            const uint32_t b = *qi;
#endif
            (i < 4 ? w.x : w.y) |= b << ((i & 3) * 8);
        }
    }
    return w;
}

template <int MODE>
struct StdMachine3 {
    static constexpr int TOPUP = 8;
    static constexpr bool LAZY = true;
    static constexpr bool LEAN = true;
    static constexpr uint32_t IDLE = F3_STOP;
    static constexpr bool QLEN = true;  // find_overlapping entries carry the list length (QSLOT_MASK)
    static constexpr int ITER = MODE;

    // one record: the hot region's leading slots from shared memory, everything else through L1 / L2
    static DACH_HD uint4 fetch(const StdEnv& Ev, uint32_t a) {
#if defined(__CUDA_ARCH__) && defined(DACH_FETCH_GENERIC)
        // experiment build: one generic load, the address space is resolved per lane by the hardware
        const uint4* q = a < Ev.hot_n ? Ev.hot + a : Ev.glob + a;
        return *q;
#else
        if (a < Ev.hot_n) {
            DACH_STAT(cache_hits);
#if defined(__CUDA_ARCH__)
            uint4 v;
            asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(Ev.hot_s + a * 16u));
            return v;
#else
            return Ev.hot[a];
#endif
        }
        return ld_u4(Ev.glob + a);
#endif
    }
    static DACH_HD const uint8_t* block_of(const Lane3& L) {  // the 8-byte block the cursor is in
        const uint64_t hi = (uint64_t)(L.hay_hi + (L.ap < L.hay_lo ? 1u : 0u));  // the cursor wrapped past 2^32
        return reinterpret_cast<const uint8_t*>((uintptr_t)((hi << 32) | (L.ap & ~7u)));
    }
    static DACH_HD void text_topup(Lane3& L, const StdEnv& Ev, const uint8_t* emu_lo) {
        (void)emu_lo;
        if (L.fl & F_NEED_NW) {
            const uint2 n = ld_text8_safe(block_of(L) + 8, Ev.text_lo, Ev.text_end);
            L.n0 = n.x;
            L.n1 = n.y;
            L.fl &= ~F_NEED_NW;
        }
    }
    static DACH_HD void to_root(Lane3& L, const StdEnv& Ev) {
        L.r0 = Ev.root_rec.x;
        L.nf = Ev.root_rec.y;
        L.r2 = Ev.root_rec.z;
        L.sig = Ev.root_rec.w;
        L.addr = D_ROOT;
    }

    // the byte is consumed; the lane sits in the state whose record it just adopted
    static DACH_HD void land(Lane3& L, const StdEnv& Ev) {
        ++L.ap;
        L.w0 = (L.w0 >> 8) | (L.w1 << 24);
        L.w1 >>= 8;
        if ((L.ap & 7u) == 0) {  // the next 8 bytes become current
            L.w0 = L.n0;
            L.w1 = L.n1;
            L.fl |= F_NEED_NW;
        }
        if (L.ap == L.ap_end) L.fl |= F_DONE | F3_STOP;
        if (L.nf & CF_OUT) {
            DACH_STAT(pushes);
            QEntry e;  // one 8-byte store: (end, slot | list length << 24); output_pos is looked up after the scan
            e.end = L.ap - L.hay_lo;
            e.opos = MODE == M_OVERLAPPING ? L.addr | (L.r2 << 24) : L.addr;  // the length: low byte of record word 2
            Ev.q[L.qn * Ev.q_stride] = e;
            if (++L.qn == (uint32_t)LANE_Q) L.fl |= F3_STOP;
            if (MODE == M_FIND) to_root(L, Ev);  // every next() restarts at ROOT (src/bytewise/iter.rs:87)
        }
    }

    // One iteration = probe() -> the fetch -> resolve().  They are separate so that a lane walking two haystacks
    // (k_scan_duo) can put both fetches in flight before it looks at either result.
    // probe: the slot to fetch for the byte under the cursor; `own` = it is a child slot of the lane's own state
    // (else of its failure state).  A stopped lane probes slot 0 (ROOT's record: always there) and ignores it.
    static DACH_HD uint32_t probe(const Lane3& L, uint32_t& own) {
        const uint32_t c = L.w0 & 0xffu;
        own = (L.sig >> (L.w0 & 31u)) & 1u;  // may this state have a child labelled c?
        const uint32_t a = ((own ? L.r0 : L.r2) >> 8) ^ c;  // its child, or the failure state's
        return (L.fl & F3_STOP) ? 0u : a;
    }
    static DACH_HD void resolve(Lane3& L, const StdEnv& Ev, const uint4& x, uint32_t a, uint32_t own) {
        if (L.fl & (F3_STOP | F3_LEARN)) {  // one test keeps both rare cases out of the common path
            if (L.fl & F3_STOP) return;
            // x is the failure state's record (fetched through the own-child path: r0 held its slot ^ c and the
            // signature bit of c was set, so probe() needed no extra case): go on from its failure link
            DACH_STAT(steps);
            DACH_STAT(learns);
            L.nf = x.y;
            L.r2 = x.z;
            L.sig &= ~(1u << (L.w0 & 31u));
            L.fl &= ~F3_LEARN;
            return;
        }
        DACH_STAT(steps);
        DACH_STAT(probes);
        if (((x.x ^ L.w0) & 0xffu) == 0) {  // CHECK == c: adopt the record
            DACH_STAT(hits);
            L.r0 = x.x;
            L.nf = x.y;
            L.r2 = x.z;
            L.sig = x.w;
            L.addr = a;
            land(L, Ev);
        } else if (own) {  // signature false positive: this state has no child for c after all
            DACH_STAT(miss_known);
            L.sig &= ~(1u << (L.w0 & 31u));
        } else if (L.nf & CF_FROOT) {  // that was ROOT's row: stay in ROOT
            DACH_STAT(root_stay);
            to_root(L, Ev);
            land(L, Ev);
        } else if (L.nf & CF_F2ROOT) {  // the failure state's own failure target is ROOT: probe ROOT's row next
            DACH_STAT(miss_f2root);
            L.r2 = Ev.root_base << 8;
            L.nf |= CF_FROOT;
        } else {
            // The failure state's record is needed to go on (0.003 per byte on the C3 text, 0.21 on C2's): it is
            // the NEXT iteration's fetch -- a second dependent fetch inside this one would hold the whole warp.
            // r0 := (its slot ^ c) << 8 with c's signature bit set makes probe() address exactly that slot.
            L.r0 = ((L.nf >> 8) ^ (L.w0 & 0xffu)) << 8;
            L.sig |= 1u << (L.w0 & 31u);
            L.fl |= F3_LEARN;
        }
    }
    static DACH_HD bool step(Lane3& L, const StdEnv& Ev, const uint8_t* emu_lo = nullptr) {
        (void)emu_lo;
        if (L.fl & F3_STOP) return false;
        uint32_t own;
        const uint32_t a = probe(L, own);
        const uint4 x = fetch(Ev, a);
        resolve(L, Ev, x, a, own);
        return true;
    }

    static DACH_HD void drain(Lane3& L, const StdEnv& Ev, const ScanParams& P, Emitter& E) {
        for (uint32_t j = 0; j < (uint32_t)LANE_Q; ++j) {
            if (j < L.qn) {
                const QEntry e = Ev.q[j * Ev.q_stride];
                if (e.end >= L.from) {  // a segment reports only what ends inside it
                    const uint32_t opos = ld_u32(Ev.opos + (e.opos & QSLOT_MASK));  // the entry holds the slot
                    if (MODE == M_OVERLAPPING)
                        emit_chain(P, E, opos, e.end);
                    else
                        emit_head(P, E, opos, e.end);
                }
            }
        }
        L.qn = 0;
        if (!(L.fl & F_DONE)) L.fl &= ~F3_STOP;
    }

    // the item is complete (its last byte landed): hand the state on to the next chunk of the stream
    static DACH_HD void finish_item(const Lane3& L, const ScanParams& P) {
        if (P.state_io) P.state_io[L.item] = P.id_out ? P.id_out[L.addr] : L.addr;
    }

    static DACH_HD void begin_item(Lane3& L, const ScanParams& P, const StdEnv& Ev, Emitter& E, uint64_t item,
                                   const uint8_t* emu_lo) {
        (void)emu_lo;
        uint64_t hay = item;
        uint32_t beg = 0;
        if (P.item_hay) {
            hay = P.item_hay[item];
            beg = P.item_beg[item];
        }
        const uint64_t o0 = P.offs[hay], o1 = P.offs[hay + 1];
        const uint32_t hay_len = (uint32_t)(o1 - o0);
        const uintptr_t h = (uintptr_t)(P.text + o0);
        L.hay_lo = (uint32_t)h;
        L.hay_hi = (uint32_t)((uint64_t)h >> 32);
        uint32_t start = 0, end = hay_len;
        if (P.item_hay && hay >= P.seg_from) {
            const uint64_t e64 = (uint64_t)beg + P.seg_len;
            if (e64 < hay_len) end = (uint32_t)e64;
            start = beg > P.warm ? beg - P.warm : 0;  // warm-up: the state at `beg` only depends on these bytes
        }
        L.ap = L.hay_lo + start;
        L.ap_end = L.hay_lo + end;
        L.from = beg ? beg + 1 : 0;
        L.item = (uint32_t)item;
        L.qn = 0;
        E.begin((uint32_t)item);
        const uint8_t* b0 = block_of(L);
        const uint2 a = ld_text8_safe(b0, Ev.text_lo, Ev.text_end);
        const uint2 n = ld_text8_safe(b0 + 8, Ev.text_lo, Ev.text_end);
        const uint32_t sh = (L.ap & 7u) * 8u;  // the byte at the cursor goes to bit 0
        const uint64_t cur = (((uint64_t)a.y << 32) | a.x) >> sh;
        L.w0 = (uint32_t)cur;
        L.w1 = (uint32_t)(cur >> 32);
        L.n0 = n.x;
        L.n1 = n.y;
        to_root(L, Ev);
        L.fl = F_ACTIVE | (start >= end ? (F_DONE | F3_STOP) : 0u);
        if (P.state_io) {
            // a chunk of a stream: resume in the state the previous chunk ended in (the stepper contract,
            // src/bytewise/iter.rs:344-475); the outputs of that state were reported with the previous chunk
            uint32_t st = P.state_io[item];
            if (st != D_ROOT && st < P.n_slots) {
                if (P.id_in) st = P.id_in[st];
                const uint4 x = fetch(Ev, st);
                L.r0 = x.x;
                L.nf = x.y;
                L.r2 = x.z;
                L.sig = x.w;
                L.addr = st;
            }
            return;
        }
        if (MODE != M_FIND && (Ev.root_flags & CF_OUT) && beg == 0) {
            QEntry e;  // the iterator starts in ROOT with ROOT's output list pending at position 0
            e.end = 0;
            e.opos = MODE == M_OVERLAPPING ? D_ROOT | (Ev.root_rec.z << 24) : D_ROOT;
            Ev.q[0] = e;
            L.qn = 1;
        }
    }
};

// =============================================================================================
// COUNT and FIRST on the lane machines (StdMachine3, LmMachine, CwMachine).
//
// The machines queue one (end, slot) entry per output event and stop stepping when the queue is full;
// their drain() turns entries into matches.  SinkOps<M, MODE, RK> replaces drain() and begin_item() for
// the other two result kinds and leaves step() -- the lock-step loop -- exactly as it is:
//   COUNT  adds 1 per event (find / no_suffix / leftmost: the head of the list) or the list's chain
//          word (find_overlapping), without walking the list;
//   FIRST  gives the lane a queue of depth one: begin_item() starts the queue at its last entry, so the
//          first event fills it and the machine stops by its own rule.  If the event is reportable (it
//          ends inside the item's segment; warm-up events do not count) its list head is the item's
//          answer and the item is done; otherwise the queue is emptied and the lane goes on.
//   HIST   adds 1 per reportable event to the event's slot (HistSink::event): no output list is read
//          here; dev_scan.cu's post-passes turn slot counts into output-record counts.
// MODE is the machine's iterator: FIRST of a Standard automaton always runs the find_overlapping
// machine, whose first event is the first event of all three Standard iterators.
// =============================================================================================
template <class M, int MODE, int RK>
struct SinkOps {
    using Sink = typename std::conditional<RK == RK_COUNT, CountSink,
                                           typename std::conditional<RK == RK_FIRST, FirstSink, HistSink>::type>::type;

    template <class LANE>
    static DACH_HD void begin_item(LANE& L, const ScanParams& P, const StdEnv& Ev, Sink& E, uint64_t item, const uint8_t* emu_lo) {
        Emitter unused;  // the machines only name the item to their sink
        M::begin_item(L, P, Ev, unused, item, emu_lo);
        E.begin((uint32_t)item);
        if constexpr (RK == RK_FIRST) {
            if (L.qn) {  // ROOT's list at position 0 (an empty pattern): reportable at once
                E.emit(P, 0, 0, ld_u4(P.outputs + (ld_u32(Ev.opos + (Ev.q[0].opos & QSLOT_MASK)) - 1)).x);
                L.qn = 0;
                L.fl |= F_DONE | M::IDLE;
            } else {
                L.qn = (uint32_t)LANE_Q - 1;
            }
        }
    }

    template <class LANE>
    static DACH_HD void drain(LANE& L, const StdEnv& Ev, const ScanParams& P, Sink& E) {
        if constexpr (RK == RK_COUNT) {
            for (uint32_t j = 0; j < (uint32_t)LANE_Q; ++j) {
                if (j < L.qn) {
                    const QEntry e = Ev.q[j * Ev.q_stride];
                    if (e.end >= L.from)
                        E.count += MODE != M_OVERLAPPING ? 1u
                                   : M::QLEN         ? qentry_len(P, Ev.opos, e.opos)
                                                     : chain_len(P, ld_u32(Ev.opos + e.opos));
                }
            }
            L.qn = 0;
        } else if constexpr (RK == RK_HIST) {
            for (uint32_t j = 0; j < (uint32_t)LANE_Q; ++j) {
                if (j < L.qn) {
                    const QEntry e = Ev.q[j * Ev.q_stride];
                    if (e.end >= L.from) E.event(P, e.opos & QSLOT_MASK);  // the entry holds the slot
                }
            }
            L.qn = 0;
        } else {
            if (L.qn == (uint32_t)LANE_Q) {
                const QEntry e = Ev.q[(LANE_Q - 1) * Ev.q_stride];
                if (e.end >= L.from) {
                    emit_head(P, E, ld_u32(Ev.opos + (e.opos & QSLOT_MASK)), e.end);
                    L.fl |= F_DONE | M::IDLE;
                }
            }
            if (!(L.fl & F_DONE)) L.qn = (uint32_t)LANE_Q - 1;
        }
        if (!(L.fl & F_DONE)) L.fl &= ~M::IDLE;
    }
};

// =============================================================================================
// The matches path of StdMachine3: the drain stores events, k_expand (dev_scan.cu) expands them.
//
// The drain does no dependent load: each reportable entry (end >= L.from) is one 8-byte store into the lane's
// current event block, and the item's match count grows by the list length the entry carries (1 for find /
// no_suffix, whose events report the list's head only).  A lane stores at most LANE_Q < BLK_EVENTS events per
// service phase, so it needs at most one new block per phase; the kernel hands those out with one warp-aggregated
// atomic between need_block() and drain().
// =============================================================================================
template <int MODE>
struct EventOps {
    using M = StdMachine3<MODE>;

    static DACH_HD void begin_item(Lane3& L, const ScanParams& P, const StdEnv& Ev, EventSink& E, uint64_t item,
                                   const uint8_t* emu_lo) {
        Emitter unused;  // the machine only names the item to its sink
        M::begin_item(L, P, Ev, unused, item, emu_lo);
        E.begin((uint32_t)item);
    }

    static DACH_HD uint32_t reportable(const Lane3& L, const StdEnv& Ev) {
        uint32_t n = 0;
        for (uint32_t j = 0; j < (uint32_t)LANE_Q; ++j)
            if (j < L.qn && Ev.q[j * Ev.q_stride].end >= L.from) ++n;
        return n;
    }
    static DACH_HD bool need_block(const Lane3& L, const StdEnv& Ev, const EventSink& E) {
        return reportable(L, Ev) > BLK_EVENTS - E.fill;
    }

    // blk: the pool block this lane was given this phase (used only if need_block() said so)
    static DACH_HD void drain(Lane3& L, const StdEnv& Ev, const ScanParams& P, EventSink& E, uint32_t blk) {
        for (uint32_t j = 0; j < (uint32_t)LANE_Q; ++j) {
            if (j < L.qn) {
                const QEntry e = Ev.q[j * Ev.q_stride];
                if (e.end >= L.from) {  // a segment reports only what ends inside it
                    if (E.fill == BLK_EVENTS) E.open(P, blk);
                    if (E.blk) st_stream_u2(E.blk + BLK_HDR_WORDS + 2 * E.fill, e.end, e.opos);
                    ++E.fill;
                    ++E.nev;
                    const uint32_t c = E.count + (MODE == M_OVERLAPPING ? qentry_len(P, Ev.opos, e.opos) : 1u);
                    if (c < E.count) count_carry(P);
                    E.count = c;
                }
            }
        }
        L.qn = 0;
        if (!(L.fl & F_DONE)) L.fl &= ~F3_STOP;
    }
};

}  // namespace dach
