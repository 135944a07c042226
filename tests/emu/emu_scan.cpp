// CPU emulation of the matches scans (TEST INFRASTRUCTURE ONLY): dach_dev_scan_batch and dach_dev_scan_stream on
// every machine, with the matches gathered from the pool blocks (k_gather), and checks of the device image against the
// crate's transition function.  The drivers are emu_driver.h's; this file also holds what the whole library shares
// once: the lane machines' counters and the size of the hot region.
#include <cstdio>
#include <cstdlib>

#include "emu_driver.h"

using namespace emu;

namespace dach {
EmuStats g_emu_stats;
}
extern "C" void emu_stats(unsigned long long* out, int reset) {
    memcpy(out, &g_emu_stats, sizeof(g_emu_stats));
    if (reset) memset(&g_emu_stats, 0, sizeof(g_emu_stats));
}
extern "C" void emu_set_hot_slots(uint32_t n) { g_want_hot_slots = n; }

static uint32_t* g_state_io = nullptr;
static const uint32_t* g_pos_in = nullptr;
static int g_stream_kernel = 3;       // which bytewise Standard machine serves emu_scan_stream_wire
static uint32_t g_stream_hot = 4096;  // ... and its shared-memory records
static int g_stream_charwise = 0;
extern "C" void emu_stream_config(int kernel, uint32_t hot_n) {
    g_stream_kernel = kernel;
    g_stream_hot = hot_n;
}
extern "C" void emu_stream_charwise(int cw) { g_stream_charwise = cw; }

extern "C" int emu_scan_batch_wire(const uint8_t* wire, size_t wire_len, int charwise, int mode, const uint8_t* text, const uint64_t* offs,
                                   uint64_t n, uint32_t hot_n, int kernel_version, uint32_t seg_len, uint32_t seg_from, uint32_t pool_blocks,
                                   dach_match* out, uint64_t out_cap, uint64_t* out_offs, uint64_t* needed) {
    HostImage img;
    bool lm = false;
    const int rc = load(wire, wire_len, charwise != 0, &img, &lm);
    if (rc) return rc;
    if ((mode == M_LEFTMOST) != lm) return DACH_MATCH_KIND_MISMATCH;
    if (mode < M_FIND || mode > M_LEFTMOST) return DACH_INVALID_ARGUMENT;
    // kernel choice as enqueue_scan (one CTA per SM).  seg_len > 0 cuts even an automaton the device scans whole (not
    // segmentable): the hand-made case of test_emu_lane.py shows with it why the device does not.
    ScanInputs in = plan_inputs(img, charwise != 0, mode);
    in.opt_kernel = kernel_version;
    in.segmentable = true;
    in.stream = g_state_io != nullptr;
    const ScanPlan plan = plan_scan(in);
    if (plan.refused) return DACH_INVALID_ARGUMENT;
    const Segments S = seg_table(offs, n, plan.seg ? seg_len : 0, seg_from);
    std::vector<uint32_t> counts(S.n_items ? S.n_items : 1, 0);
    std::vector<uint32_t> pool((size_t)pool_blocks * BLK_WORDS, 0xdeadbeefu);
    ScanCtrl ctrl;
    memset(&ctrl, 0, sizeof(ctrl));
    ScanParams P = scan_params(img, text, offs, n, S, &ctrl);
    P.counts = counts.data();
    P.pool = pool.data();
    P.pool_blocks = pool_blocks;
    P.state_io = g_state_io;
    const Smem sm(img, plan, std::min(hot_n, img.n_slots), P.text_lo, P.text_end);
    for_mode(mode, [&](auto M) { run_matches<decltype(M)::value>(plan.machine, charwise != 0, P, sm, 3); });
    std::vector<uint64_t> item_offs;
    const int orc = offsets(S, n, counts, ctrl, out_cap, item_offs, out_offs, needed);
    if (orc) return orc;
    // k_gather
    const uint32_t used_blocks = ctrl.blk_cursor < pool_blocks ? ctrl.blk_cursor : pool_blocks;
    uint32_t* out_words = reinterpret_cast<uint32_t*>(out);
    for (uint32_t b = 0; b < used_blocks; ++b) {
        const uint32_t* blk = pool.data() + (size_t)b * BLK_WORDS;
        const uint32_t item = blk[0], seq = blk[1];
        const uint32_t first = seq * BLK_MATCHES;
        uint32_t nm = counts[item] - first;
        if (nm > BLK_MATCHES) nm = BLK_MATCHES;
        uint32_t* dst = out_words + (item_offs[item] + first) * 3ull;
        for (uint32_t w = 0; w < nm * 3; ++w) dst[w] = blk[BLK_SLOT_WORDS * (1 + w / 3) + w % 3];
    }
    if (g_pos_in) add_base(out_words, out_offs, n, g_pos_in);
    return DACH_OK;
}

// dach_dev_scan_stream: chunks of streams (state in/out per haystack, optional base position)
extern "C" int emu_scan_stream_wire(const uint8_t* wire, size_t wire_len, int mode, const uint8_t* text, const uint64_t* offs,
                                    uint64_t n, uint32_t* state_io, const uint32_t* pos_in, uint32_t pool_blocks, dach_match* out,
                                    uint64_t out_cap, uint64_t* out_offs, uint64_t* needed) {
    if (mode != M_FIND && mode != M_OVERLAPPING) return DACH_INVALID_ARGUMENT;
    g_state_io = state_io;
    g_pos_in = pos_in;
    const int rc = emu_scan_batch_wire(wire, wire_len, g_stream_charwise, mode, text, offs, n, g_stream_hot, g_stream_kernel, 0, 0, pool_blocks, out, out_cap, out_offs, needed);
    g_state_io = nullptr;
    g_pos_in = nullptr;
    return rc;
}

// Exhaustive check of the compact bytewise image against the crate's transition function: for every state s of
// the host automaton and every byte c, following the image's records (signature, BASE ^ c with CHECK, efail /
// fbase chain, the flags CF_FROOT / CF_F2ROOT / CF_F2DEAD) from new_of_old[s] must end in new_of_old[delta(s, c)].
// Returns the number of mismatches (0 = the relayout and every derived field are consistent), -1 on a bad automaton.
extern "C" long long emu_check_image_transitions(const uint8_t* wire, size_t wire_len, uint32_t want_hot_slots,
                                                 uint32_t* hot_slots_out, uint32_t* hot_used_out) {
    dach_pma* pma = nullptr;
    size_t used = 0;
    if (wire_read(wire, wire_len, false, &pma, &used)) return -1;
    HostImage img;
    img.want_hot_slots = want_hot_slots;
    if (build_image(pma, &img) || img.crec.empty()) {
        delete pma;
        return -1;
    }
    const bool lm = is_leftmost(pma->match_kind);
    const size_t n = pma->slots();
    const uint32_t N = img.n_cslots;
    auto rec = [&](uint32_t slot) { return &img.crec[(size_t)slot * 4]; };
    auto nid = [&](uint32_t s) { return img.hot_slots ? img.new_of_old[s] : s; };
    // states a scan can be in: the closure of ROOT under the crate's transition function (for an automaton the
    // builders made that is the trie; a hand-made one may have states only failure links lead to)
    std::vector<uint8_t> live(n, 0);
    std::vector<uint32_t> q{kRoot};
    live[kRoot] = 1;
    long long bad = 0;
    uint32_t hot_used = 0;
    for (size_t h = 0; h < q.size(); ++h) {
        const uint32_t s = q[h];
        if (nid(s) < img.hot_slots) ++hot_used;
        {  // output position and CF_OUT travel with the state; stream state ids map back
            const uint32_t op = pma->opos_ch[s] >> 8;
            if (img.opos_tab[nid(s)] != op || ((rec(nid(s))[1] & 1u) != 0) != (op != 0)) ++bad;
            if (img.hot_slots && img.old_of_new[nid(s)] != s) ++bad;
        }
        for (uint32_t c = 0; c < 256; ++c) {
            // the crate (src/bytewise.rs:1063-1088 / :1094-1128)
            uint32_t t = s;
            for (;;) {
                const uint32_t b = pma->base[t];
                if (b) {
                    const uint32_t ci = b ^ c;
                    if (ci < n && (pma->opos_ch[ci] & 0xffu) == c) {
                        t = ci;
                        break;
                    }
                }
                if (t == kRoot) break;
                const uint32_t f = pma->fail[t];
                if (lm && f == kDead) {
                    t = kRoot;
                    break;
                }
                t = f;
            }
            if (!live[t]) live[t] = 1, q.push_back(t);
            // the image, field by field as the lane machines read it (scan_lane.cuh, StdMachine3 / LmMachine)
            auto child = [&](uint32_t base, uint32_t* out) {
                if (!base) return false;
                const uint32_t a = base ^ c;
                if (a >= N || (rec(a)[0] & 0xffu) != c) return false;
                *out = a;
                return true;
            };
            uint32_t cur = nid(s), got = kRoot;
            bool done = child(rec(cur)[0] >> 8, &got);
            if (done && !((rec(cur)[3] >> (c & 31u)) & 1u)) ++bad;  // the signature must never hide a child
            if (!done && cur != kRoot) {
                for (int guard = 0; guard < 1 << 20 && !done; ++guard) {
                    const uint32_t nf = rec(cur)[1], f = nf >> 8, fbase = rec(cur)[2] >> 8;
                    if (f == kRoot) {
                        if (!lm && (!(nf & 8u) || fbase != img.root_base)) ++bad;  // CF_FROOT, pre-resolved base
                        if (!child(img.root_base, &got)) got = kRoot;
                        break;
                    }
                    if (lm && f == kDead) {
                        got = kRoot;
                        break;
                    }
                    if (fbase != (rec(f)[0] >> 8)) ++bad;  // fbase is the failure state's BASE
                    if (child(fbase, &got)) break;
                    const uint32_t f2 = rec(f)[1] >> 8;
                    if (((nf & 2u) != 0) != (f2 == kRoot)) ++bad;  // CF_F2ROOT
                    if (lm && ((nf & 4u) != 0) != (f2 == kDead)) ++bad;  // CF_F2DEAD
                    if (nf & 2u) {
                        if (!child(img.root_base, &got)) got = kRoot;
                        break;
                    }
                    if (lm && (nf & 4u)) {
                        got = kRoot;
                        break;
                    }
                    cur = f;  // its children were just probed through fbase: go on with ITS failure fields
                }
            }
            if (got != nid(t)) {
                if (getenv("EMU_DBG") && bad < 10) fprintf(stderr, "s=%u(new %u) c=%u crate->%u(new %u) image->%u base=%u\n", s, nid(s), c, t, nid(t), got, rec(nid(s))[0]>>8);
                ++bad;
            }
        }
    }
    if (hot_slots_out) *hot_slots_out = img.hot_slots;
    if (hot_used_out) *hot_used_out = hot_used;
    delete pma;
    return bad;
}

// The same for the charwise compact image (CwMachine): every reachable state x every mapped code.  Records are
// {BASE << 8 | sig lo, efail << 8 | flags, fbase << 8 | sig hi, parent << 8}; a child of `cur` for code k is
// the slot BASE ^ k whose parent field is `cur` (src/charwise.rs:1022-1095, next_state_id(_leftmost)_unchecked).
// Returns the mismatches, -1 for a refused automaton, -2 where the crate's own walk would not terminate.
extern "C" long long emu_check_image_transitions_charwise(const uint8_t* wire, size_t wire_len) {
    dach_pma* pma = nullptr;
    size_t used = 0;
    if (wire_read(wire, wire_len, true, &pma, &used)) return -1;
    HostImage img;
    if (build_image(pma, &img) || img.crec.empty()) {
        delete pma;
        return -1;
    }
    const bool lm = is_leftmost(pma->match_kind);
    const uint32_t n = uint32_t(pma->slots()), A = pma->alphabet_size;
    auto rec = [&](uint32_t slot) { return &img.crec[(size_t)slot * 4]; };
    auto crate_child = [&](uint32_t s, uint32_t k, uint32_t* out) {
        const uint32_t b = pma->base[s];
        if (!b) return false;
        const uint32_t ci = b ^ k;
        if (ci >= n || pma->check[ci] != s) return false;
        *out = ci;
        return true;
    };
    std::vector<uint8_t> live(n, 0);
    std::vector<uint32_t> q{kRoot};
    live[kRoot] = 1;
    long long bad = 0;
    for (size_t h = 0; h < q.size(); ++h) {  // closure of ROOT under the crate's transition function
        const uint32_t s = q[h];
        if (img.opos_tab[s] != pma->output_pos[s] || ((rec(s)[1] & 1u) != 0) != (pma->output_pos[s] != 0)) ++bad;
        for (uint32_t k = 0; k < A; ++k) {
            uint32_t t = s;
            for (;;) {  // the crate
                if (crate_child(t, k, &t)) break;
                if (t == kRoot) break;
                const uint32_t f = pma->fail[t];
                if (f == kDead) {
                    if (!lm) {  // DEAD fails to itself: the crate's standard walk would never return (hand-made
                        delete pma;  // automata only; DESIGN.md section 1 lists it as a deliberate divergence)
                        return -2;
                    }
                    t = kRoot;
                    break;
                }
                t = f;
            }
            if (!live[t]) live[t] = 1, q.push_back(t);
            auto child = [&](uint32_t par, uint32_t base, uint32_t* out) {  // the image
                if (!base) return false;
                const uint32_t a = base ^ k;
                if (a >= n || (rec(a)[3] >> 8) != par) return false;
                *out = a;
                return true;
            };
            uint32_t cur = s, got = kRoot;
            bool done = child(cur, rec(cur)[0] >> 8, &got);
            const uint32_t sig = (rec(cur)[0] & 0xffu) | ((rec(cur)[2] & 0xffu) << 8);
            if (done && !((sig >> (k & 15u)) & 1u)) ++bad;
            if (!done && cur != kRoot) {
                for (int guard = 0; guard < 1 << 20; ++guard) {
                    const uint32_t nf = rec(cur)[1], f = nf >> 8, fbase = rec(cur)[2] >> 8;
                    if (f == kRoot) {
                        if (!child(kRoot, img.root_base, &got)) got = kRoot;
                        break;
                    }
                    if (f == kDead) {
                        got = kRoot;
                        break;
                    }
                    if (fbase != (rec(f)[0] >> 8)) ++bad;
                    if (child(f, fbase, &got)) break;
                    const uint32_t f2 = rec(f)[1] >> 8;
                    if (((nf & 2u) != 0) != (f2 == kRoot) || ((nf & 4u) != 0) != (f2 == kDead)) ++bad;
                    if (nf & 2u) {
                        if (!child(kRoot, img.root_base, &got)) got = kRoot;
                        break;
                    }
                    if (nf & 4u) {
                        got = kRoot;
                        break;
                    }
                    cur = f;
                }
            }
            if (got != t) ++bad;
        }
    }
    delete pma;
    return bad;
}

// HostImage::segmentable of a serialized bytewise automaton: 1 / 0, -1 for a refused one.
extern "C" int emu_image_segmentable(const uint8_t* wire, size_t wire_len) {
    HostImage img;
    return load(wire, wire_len, false, &img) ? -1 : (img.segmentable ? 1 : 0);
}

// the device image's output records {value, length, parent, chain} (dev_image.cpp): up to cap records, returns their number
extern "C" long long emu_image_outputs(const uint8_t* wire, size_t wire_len, int charwise, uint32_t* out, size_t cap) {
    HostImage img;
    if (load(wire, wire_len, charwise != 0, &img)) return -1;
    const size_t k = img.outputs.size() / 4;
    if (out) memcpy(out, img.outputs.data(), std::min(k, cap) * 16);
    return (long long)k;
}
