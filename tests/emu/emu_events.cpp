// CPU emulation of StdMachine3's event paths of the matches scan (TEST INFRASTRUCTURE ONLY): the lanes store (end,
// state) events into pool blocks -- through the per-lane queue (scan_machine with EventOps) or at the landing that makes
// them (k_scan_direct) -- and placement expands them: k_expand, restated to walk the output lists on its own (parent
// links, not the chain word the kernel uses), or k_blk_desc + k_expand_desc, the ordered placement from block
// descriptors and two-entry output lists.  The drivers are emu_driver.h's.
#include "emu_driver.h"

using namespace emu;

// The kernel's view of an event list: the tuples of its block descriptors' events, U blocks at a time as one warp takes
// them, into a buffer whose first tuple sits `pad` words past a 16-byte boundary (as a staged shard-group copy or a base
// does).  Returns -2 if the image has no pairs table.
static int place_desc(const HostImage& img, int mode, const std::vector<uint32_t>& pool, uint32_t n_blocks, const Segments& S,
                      const std::vector<uint32_t>& ev_counts, const std::vector<uint64_t>& item_offs, uint64_t total, uint32_t u,
                      uint32_t pad, dach_match* out) {
    // blocks per item and their first block in output order (k_offsets_* <BLK_EVENTS>), k_blk_desc
    std::vector<uint64_t> blk_first(S.n_items + 1, 0);
    for (uint64_t i = 0; i < S.n_items; ++i) blk_first[i + 1] = blk_first[i] + (ev_counts[i] + BLK_EVENTS - 1) / BLK_EVENTS;
    std::vector<uint32_t> desc((size_t)n_blocks * 4 + 4, 0xdeadbeefu);
    for (uint32_t b = 0; b < n_blocks; ++b) {
        const uint32_t* h = pool.data() + (size_t)b * BLK_WORDS;  // {item, seq, first, -}
        const uint64_t j = blk_first[h[0]] + h[1];
        if (j < n_blocks) {
            const uint64_t at = item_offs[h[0]] + h[2];
            uint32_t nev = ev_counts[h[0]] - h[1] * BLK_EVENTS;
            desc[j * 4 + 0] = b;
            desc[j * 4 + 1] = nev < BLK_EVENTS ? nev : BLK_EVENTS;
            desc[j * 4 + 2] = (uint32_t)at;
            desc[j * 4 + 3] = (uint32_t)(at >> 32);
        }
    }
    // k_expand_desc
    if (img.pairs.empty() && !img.outputs.empty()) return -2;
    std::vector<uint32_t> words((size_t)total * 3 + 8, 0);
    uint32_t* out_words = words.data() + (pad & 3u);
    const uint32_t* pairs = img.pairs.data();
    const uint32_t* outs = img.outputs.data();
    for (uint32_t b0 = 0; b0 < n_blocks; b0 += u) {
        for (uint32_t k = 0; k < u && b0 + k < n_blocks; ++k) {
            const uint32_t* d = desc.data() + (size_t)(b0 + k) * 4;
            const uint32_t* ev = pool.data() + (size_t)d[0] * BLK_WORDS + BLK_HDR_WORDS;
            uint32_t cls[32], len[32], op[32];
            for (uint32_t l = 0; l < 32; ++l) {
                op[l] = l < d[1] ? img.opos_tab[ev[2 * l + 1] & QSLOT_MASK] : 0u;
                cls[l] = !op[l] ? 0u : mode == M_OVERLAPPING ? pairs[(op[l] - 1) * 4 + 3] >> PAIR_CLASS_SHIFT : 1u;
                len[l] = cls[l] == 3u ? outs[(op[l] - 1) * 4 + 3] : cls[l];
            }
            uint32_t* w = out_words + ((uint64_t)d[3] << 32 | d[2]) * 3ull;
            for (uint32_t l = 0; l < 32; ++l) {
                const uint32_t end = ev[2 * l];
                const uint32_t* p = pairs + (size_t)(op[l] ? op[l] - 1 : 0) * 4;
                if (cls[l] == 1u || cls[l] == 2u) {
                    *w++ = end - p[1], *w++ = end, *w++ = p[0];
                    if (cls[l] == 2u) *w++ = end - (p[3] & PAIR_LEN_MASK), *w++ = end, *w++ = p[2];
                } else if (cls[l] == 3u) {
                    for (uint32_t r = op[l]; r != 0; r = outs[(r - 1) * 4 + 2])
                        *w++ = end - outs[(r - 1) * 4 + 1], *w++ = end, *w++ = outs[(r - 1) * 4];
                }
            }
        }
    }
    memcpy(out, out_words, (size_t)total * 12);
    return DACH_OK;
}

// dach_dev_scan_batch / dach_dev_scan_stream (state_io, pos_in) of a bytewise Standard automaton on StdMachine3's event
// paths.  direct = 0: the queue kernel, 1: k_scan_direct; place_u > 0: placed by k_expand_desc with place_u blocks per
// warp and place_pad words of misalignment, else by k_expand.  Returns a dach_status, or -1 if plan_scan would not run
// StdMachine3's event path on this automaton and mode, -2 if placement by descriptors finds no pairs table.
// blocks_used: the event blocks the scan took from the pool.
extern "C" int emu_events_scan_wire(const uint8_t* wire, size_t wire_len, int mode, const uint8_t* text, const uint64_t* offs,
                                    uint64_t n, uint32_t hot_n, uint32_t seg_len, uint32_t seg_from, uint32_t pool_blocks,
                                    uint32_t* state_io, const uint32_t* pos_in, dach_match* out, uint64_t out_cap,
                                    uint64_t* out_offs, uint64_t* needed, uint32_t* blocks_used, int direct, uint32_t place_u,
                                    uint32_t place_pad) {
    HostImage img;
    bool lm = false;
    const int rc = load(wire, wire_len, false, &img, &lm);
    if (rc) return rc;
    if (lm || mode == M_LEFTMOST) return DACH_MATCH_KIND_MISMATCH;
    // one CTA per SM, the queue kernel by option event_queue; seg_len > 0 cuts whatever automaton it is given, as the
    // matches emulator does
    ScanInputs in = plan_inputs(img, false, mode);
    in.segmentable = true;
    in.opt_event_queue = direct ? 0 : 1;
    in.stream = state_io != nullptr;
    const ScanPlan plan = plan_scan(in);
    if (!plan.events()) return -1;
    const Segments S = seg_table(offs, n, plan.seg ? seg_len : 0, seg_from);
    std::vector<uint32_t> counts(S.n_items ? S.n_items : 1, 0), ev_counts(S.n_items ? S.n_items : 1, 0);
    std::vector<uint32_t> pool((size_t)pool_blocks * BLK_WORDS + 1, 0xdeadbeefu);
    ScanCtrl ctrl;
    memset(&ctrl, 0, sizeof(ctrl));
    ScanParams P = scan_params(img, text, offs, n, S, &ctrl);
    P.counts = counts.data();
    P.ev_counts = ev_counts.data();
    P.pool = pool.data();
    P.pool_blocks = pool_blocks;
    P.state_io = state_io;
    const Smem sm(img, plan, hot_n, P.text_lo, P.text_end);
    for_mode(mode, [&](auto M) {
        constexpr int MODE = decltype(M)::value;
        if constexpr (MODE != M_LEFTMOST) {
            if (plan.machine == Machine::Std3Direct)
                run_direct<MODE>(P, sm.Ev, P.text_lo, 3);
            else
                run_machine<StdMachine3<MODE>, EventOps<MODE>, Lane3, EventSink>(P, sm.Ev, P.text_lo, 1, 3);
        }
    });
    if (blocks_used) *blocks_used = ctrl.blk_cursor;
    std::vector<uint64_t> item_offs;
    const int orc = offsets(S, n, counts, ctrl, out_cap, item_offs, out_offs, needed);
    if (orc) return orc;
    const uint32_t n_blocks = ctrl.blk_cursor < pool_blocks ? ctrl.blk_cursor : pool_blocks;
    uint32_t* out_words = reinterpret_cast<uint32_t*>(out);
    if (place_u) {
        const int prc = place_desc(img, mode, pool, n_blocks, S, ev_counts, item_offs, item_offs[S.n_items], place_u, place_pad, out);
        if (prc) return prc;
    } else {
        // k_expand: every event of every block, its list from output_pos of its slot along the parent links
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
    }
    if (pos_in) add_base(out_words, out_offs, n, pos_in);
    return DACH_OK;
}

// outputs and pairs of the device image (4 words per output record each); returns the number of records, -1 if the
// image has no pairs table, or -100 - the image status
extern "C" int64_t emu_place_tables(const uint8_t* wire, size_t wire_len, uint32_t* outputs, uint32_t* pairs, uint64_t cap) {
    HostImage img;
    const int rc = load(wire, wire_len, false, &img);
    if (rc) return -(int64_t)rc - 100;
    const uint64_t n = img.outputs.size() / 4;
    if (img.pairs.empty() && n) return -1;
    if (n <= cap) {
        memcpy(outputs, img.outputs.data(), n * 16);
        memcpy(pairs, img.pairs.data(), n * 16);
    }
    return (int64_t)n;
}
