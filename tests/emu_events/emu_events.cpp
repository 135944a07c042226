// CPU emulation of StdMachine3's matches path with event blocks (TEST INFRASTRUCTURE ONLY).
//
// Compiles daachorse_b200/csrc/scan_lane.cuh with g++ (-DDACH_EMU) and drives it the way dev_scan.cu does for the
// bytewise Standard iterators: warps of 32 lanes in lock step, the service phase of scan_machine (event blocks handed
// out to the lanes that need one with one "atomic" per warp, EventOps::drain), the per-item offsets and a restatement
// of k_expand that walks the output lists on its own (parent links, not the chain word the kernel uses).  It is never
// loaded by the product.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../daachorse_b200/csrc/dev_image.h"
#include "../../daachorse_b200/csrc/host.h"
#include "../../daachorse_b200/csrc/scan_lane.cuh"

using namespace dach;

namespace dach {
EmuStats g_emu_stats;
}

// scan_machine<StdMachine3<MODE>, EventOps<MODE>, Lane3, EventSink> with the warp collectives written out as loops
template <int MODE>
static void run_warps(const ScanParams& P, const StdEnv& Ev0, const uint8_t* lo, int n_warps) {
    using M = StdMachine3<MODE>;
    using OPS = EventOps<MODE>;
    struct Warp {
        Lane3 L[32];
        EventSink E[32];
        StdEnv Ev[32];
        std::vector<QEntry> queue;
        bool exhausted[32];
        bool finished;
    };
    std::vector<Warp> warps(n_warps);
    for (auto& w : warps) {
        w.queue.assign((size_t)LANE_Q * 32, QEntry{0, 0});
        for (int l = 0; l < 32; ++l) {
            w.L[l].fl = M::IDLE;
            w.L[l].qn = 0;
            w.E[l].begin(0);
            w.exhausted[l] = false;
            w.Ev[l] = Ev0;
            w.Ev[l].q = w.queue.data() + l;
            w.Ev[l].q_stride = 32;
        }
        w.finished = false;
    }
    bool any_left = true;
    while (any_left) {  // round-robin over warps, one "service + run" turn each, to interleave block allocation
        any_left = false;
        for (auto& w : warps) {
            if (w.finished) continue;
            unsigned mb = 0;
            for (int l = 0; l < 32; ++l)
                if ((w.L[l].fl & F_ACTIVE) && OPS::need_block(w.L[l], w.Ev[l], w.E[l])) mb |= 1u << l;
            const uint32_t b0 = P.ctrl->blk_cursor;
            P.ctrl->blk_cursor += __builtin_popcount(mb);
            for (int l = 0; l < 32; ++l)
                if (w.L[l].fl & F_ACTIVE) OPS::drain(w.L[l], w.Ev[l], P, w.E[l], b0 + __builtin_popcount(mb & ((1u << l) - 1u)));
            for (int l = 0; l < 32; ++l)
                if ((w.L[l].fl & (F_ACTIVE | F_DONE)) == (F_ACTIVE | F_DONE)) {
                    w.E[l].finish(P);
                    M::finish_item(w.L[l], P);
                    w.L[l].fl = M::IDLE;
                }
            unsigned m = 0;
            for (int l = 0; l < 32; ++l)
                if (!(w.L[l].fl & F_ACTIVE) && !w.exhausted[l]) m |= 1u << l;
            if (m) {
                const unsigned long long base = P.ctrl->next_item;
                P.ctrl->next_item += __builtin_popcount(m);
                for (int l = 0; l < 32; ++l)
                    if (m & (1u << l)) {
                        const unsigned long long item = base + __builtin_popcount(m & ((1u << l) - 1u));
                        if (item < P.n_items)
                            OPS::begin_item(w.L[l], P, w.Ev[l], w.E[l], item, lo);
                        else
                            w.exhausted[l] = true;
                    }
            }
            bool any_active = false;
            for (int l = 0; l < 32; ++l) any_active |= (w.L[l].fl & F_ACTIVE) != 0;
            if (!any_active) {
                w.finished = true;
                continue;
            }
            any_left = true;
            bool stop = false;
            while (!stop) {
                for (int l = 0; l < 32; ++l) M::text_topup(w.L[l], w.Ev[l], lo);
                for (int k = 0; k < M::TOPUP; ++k)
                    for (int l = 0; l < 32; ++l) (void)M::step(w.L[l], w.Ev[l], lo);
                for (int l = 0; l < 32; ++l)
                    if ((w.L[l].fl & (F_ACTIVE | M::IDLE)) == (F_ACTIVE | M::IDLE)) stop = true;
            }
        }
    }
}

// dach_dev_scan_batch / dach_dev_scan_stream (state_io, pos_in) of a bytewise Standard automaton on StdMachine3.
// Returns a dach_status, or -1 if the automaton / mode does not run on StdMachine3 (dev_scan.cu: enqueue_scan).
// blocks_used: the event blocks the scan took from the pool.
extern "C" int emu_events_scan_wire(const uint8_t* wire, size_t wire_len, int mode, const uint8_t* text, const uint64_t* offs,
                                    uint64_t n, uint32_t hot_n, uint32_t seg_len, uint32_t seg_from, uint32_t pool_blocks,
                                    uint32_t* state_io, const uint32_t* pos_in, dach_match* out, uint64_t out_cap,
                                    uint64_t* out_offs, uint64_t* needed, uint32_t* blocks_used) {
    dach_pma* pma = nullptr;
    size_t used = 0;
    int rc = wire_read(wire, wire_len, false, &pma, &used);
    if (rc) return rc;
    HostImage img;
    rc = build_image(pma, &img);
    const bool lm = is_leftmost(pma->match_kind);
    delete pma;
    if (rc) return rc;
    if (lm || mode == M_LEFTMOST) return DACH_MATCH_KIND_MISMATCH;
    if (img.crec.empty() || img.root_base == 0 || (mode == M_FIND && img.root_opos != 0)) return -1;

    // segment table (k_seg_count / k_seg_fill)
    const bool seg = !state_io && seg_len > 0 && (mode == M_OVERLAPPING || mode == M_NO_SUFFIX);
    std::vector<uint32_t> item_hay, item_beg;
    std::vector<uint64_t> seg_first(n + 1, 0);
    uint64_t n_items = n;
    if (seg) {
        for (uint64_t h = 0; h < n; ++h) {
            const uint64_t len = offs[h + 1] - offs[h];
            uint64_t k = h < seg_from ? 1 : (len + seg_len - 1) / seg_len;
            if (k == 0) k = 1;
            seg_first[h + 1] = seg_first[h] + k;
            for (uint64_t j = 0; j < k; ++j) {
                item_hay.push_back((uint32_t)h);
                item_beg.push_back((uint32_t)(j * seg_len));
            }
        }
        n_items = seg_first[n];
    }
    std::vector<uint32_t> counts(n_items ? n_items : 1, 0), ev_counts(n_items ? n_items : 1, 0);
    std::vector<uint32_t> pool((size_t)pool_blocks * BLK_WORDS + 1, 0xdeadbeefu);
    ScanCtrl ctrl;
    memset(&ctrl, 0, sizeof(ctrl));
    ScanParams P;
    memset(&P, 0, sizeof(P));
    P.outputs = reinterpret_cast<const uint4*>(img.outputs.data());
    P.n_slots = img.n_slots;
    P.root_opos = img.root_opos;
    P.text = text;
    P.text_lo = text + (n ? offs[0] : 0);
    P.text_end = text + (n ? offs[n] : 0);
    if (img.hot_slots) {
        P.id_in = img.new_of_old.data();
        P.id_out = img.old_of_new.data();
    }
    P.offs = offs;
    P.n_items = n_items;
    if (seg) {
        P.item_hay = item_hay.data();
        P.item_beg = item_beg.data();
        P.seg_len = seg_len;
        P.seg_from = seg_from;
        P.warm = img.max_pattern_len ? img.max_pattern_len - 1 : 0;
    }
    P.counts = counts.data();
    P.ev_counts = ev_counts.data();
    P.pool = pool.data();
    P.pool_blocks = pool_blocks;
    P.ctrl = &ctrl;
    P.state_io = state_io;
    // the leading hot_n compact records come from a "shared memory" copy; everything past them there is poison
    uint32_t entries = hot_n < img.hot_slots ? hot_n : img.hot_slots;
    std::vector<uint32_t> tab(img.crec.size(), 0xdeadbeefu);
    memcpy(tab.data(), img.crec.data(), (size_t)entries * 16);
    const StdEnv Ev{reinterpret_cast<const uint4*>(img.crec.data()), reinterpret_cast<const uint4*>(tab.data()), 0u, entries,
                    img.opos_tab.data(), P.text_end, P.text_lo, img.root_base, P.root_opos ? CF_OUT : 0u, nullptr, 0, 0, nullptr, 0,
                    reinterpret_cast<const uint4*>(img.crec.data())[D_ROOT]};
    const int n_warps = 3;
    if (mode == M_FIND) run_warps<M_FIND>(P, Ev, P.text_lo, n_warps);
    if (mode == M_OVERLAPPING) run_warps<M_OVERLAPPING>(P, Ev, P.text_lo, n_warps);
    if (mode == M_NO_SUFFIX) run_warps<M_NO_SUFFIX>(P, Ev, P.text_lo, n_warps);
    if (blocks_used) *blocks_used = ctrl.blk_cursor;

    // offsets (k_offsets_*), per-haystack offsets (k_final_offsets)
    std::vector<uint64_t> item_offs(n_items + 1, 0);
    for (uint64_t i = 0; i < n_items; ++i) item_offs[i + 1] = item_offs[i] + counts[i];
    const uint64_t total = item_offs[n_items] + ((uint64_t)ctrl.carries << 32);  // finish_scan: exact past 2^32
    for (uint64_t h = 0; h <= n; ++h) out_offs[h] = seg ? item_offs[seg_first[h]] : item_offs[h];
    if (needed) *needed = total;
    if (ctrl.carries) return DACH_INVALID_ARGUMENT;  // a haystack with 2^32 or more matches cannot be placed
    if (ctrl.overflow || total > out_cap) return DACH_OUTPUT_OVERFLOW;
    // k_expand: every event of every block, its list from output_pos of its slot along the parent links
    const uint32_t n_blocks = ctrl.blk_cursor < pool_blocks ? ctrl.blk_cursor : pool_blocks;
    uint32_t* out_words = reinterpret_cast<uint32_t*>(out);
    for (uint32_t b = 0; b < n_blocks; ++b) {
        const uint32_t* blk = pool.data() + (size_t)b * BLK_WORDS;
        const uint32_t item = blk[0], seq = blk[1], first = blk[2];
        uint32_t nev = ev_counts[item] - seq * BLK_EVENTS;
        if (nev > BLK_EVENTS) nev = BLK_EVENTS;
        uint32_t* dst = out_words + (item_offs[item] + first) * 3ull;
        for (uint32_t j = 0; j < nev; ++j) {
            const uint32_t end = blk[BLK_HDR_WORDS + 2 * j], slot = blk[BLK_HDR_WORDS + 2 * j + 1] & QSLOT_MASK;
            for (uint32_t op = img.opos_tab[slot]; op != 0; op = mode == M_OVERLAPPING ? img.outputs[(op - 1) * 4 + 2] : 0) {
                *dst++ = end - img.outputs[(op - 1) * 4 + 1];
                *dst++ = end;
                *dst++ = img.outputs[(op - 1) * 4];
            }
        }
    }
    if (pos_in)  // k_add_base
        for (uint64_t h = 0; h < n; ++h)
            for (uint64_t m = out_offs[h]; m < out_offs[h + 1]; ++m) {
                out_words[m * 3 + 0] += pos_in[h];
                out_words[m * 3 + 1] += pos_in[h];
            }
    return DACH_OK;
}
