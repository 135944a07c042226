// CPU restatement of the ordered event placement from block descriptors (TEST INFRASTRUCTURE ONLY).
//
// Scans as tests/emu_direct does (its warps are compiled in from there), then places the event blocks the way
// dev_scan.cu's k_blk_desc and k_expand_desc do: descriptors in output order from the block headers, ev_counts and
// item_offs; per warp U blocks, each event's list from the two-entry table (HostImage::pairs), lists of three or more
// walked from the head; each block's tuples written as one run from its descriptor's first match.
// Also hands out the image's outputs and pairs tables.  It is never loaded by the product.
#include "../emu_direct/emu_direct.cpp"

// outputs and pairs of the device image (4 words per output record each); returns the number of records, or -1 if
// the image has no pairs table, or the image status
extern "C" int64_t emu_place_tables(const uint8_t* wire, size_t wire_len, uint32_t* outputs, uint32_t* pairs, uint64_t cap) {
    dach_pma* pma = nullptr;
    size_t used = 0;
    int rc = wire_read(wire, wire_len, false, &pma, &used);
    if (rc) return -(int64_t)rc - 100;
    HostImage img;
    rc = build_image(pma, &img);
    delete pma;
    if (rc) return -(int64_t)rc - 100;
    const uint64_t n = img.outputs.size() / 4;
    if (img.pairs.empty() && n) return -1;
    if (n <= cap) {
        memcpy(outputs, img.outputs.data(), n * 16);
        memcpy(pairs, img.pairs.data(), n * 16);
    }
    return (int64_t)n;
}

extern "C" int emu_place_scan_wire(const uint8_t* wire, size_t wire_len, int mode, const uint8_t* text, const uint64_t* offs,
                                    uint64_t n, uint32_t hot_n, uint32_t seg_len, uint32_t seg_from, uint32_t pool_blocks,
                                    uint32_t* state_io, const uint32_t* pos_in, dach_match* out, uint64_t out_cap, uint32_t u, uint32_t pad,
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
    // blocks per item and their first block in output order (k_offsets_* <BLK_EVENTS>), k_blk_desc
    const uint32_t n_blocks = ctrl.blk_cursor < pool_blocks ? ctrl.blk_cursor : pool_blocks;
    std::vector<uint64_t> blk_first(n_items + 1, 0);
    for (uint64_t i = 0; i < n_items; ++i) blk_first[i + 1] = blk_first[i] + (ev_counts[i] + BLK_EVENTS - 1) / BLK_EVENTS;
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
    // k_expand_desc into a buffer whose first tuple sits `pad` words past a 16-byte boundary (as a staged shard-group
    // copy or a base does); U blocks at a time, as one warp takes them
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
    if (pos_in)  // k_add_base
        for (uint64_t h = 0; h < n; ++h)
            for (uint64_t m = out_offs[h]; m < out_offs[h + 1]; ++m) {
                reinterpret_cast<uint32_t*>(out)[m * 3 + 0] += pos_in[h];
                reinterpret_cast<uint32_t*>(out)[m * 3 + 1] += pos_in[h];
            }
    return DACH_OK;
}
