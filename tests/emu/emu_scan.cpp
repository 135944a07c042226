// CPU emulation harness for the per-lane scan logic (TEST INFRASTRUCTURE ONLY).
//
// Compiles daachorse_b200/csrc/scan_lane.cuh -- the exact code the CUDA kernels run -- with
// g++ (-DDACH_EMU) and drives it the way dev_scan.cu does (items -> lanes, pooled 256-byte
// blocks, exclusive scan of counts, gather), so that lane-logic bugs surface on the CPU box
// before GPU minutes are spent.  It is never loaded by the product.
#include <cstdint>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../daachorse_b200/csrc/dev_image.h"
#include "../../daachorse_b200/csrc/host.h"
#include "../../daachorse_b200/csrc/scan_lane.cuh"
#include "../../daachorse_b200/csrc/scan_plan.h"

using namespace dach;

namespace dach {
EmuStats g_emu_stats;
}
extern "C" void emu_stats(unsigned long long* out, int reset) {
    memcpy(out, &g_emu_stats, sizeof(g_emu_stats));
    if (reset) memset(&g_emu_stats, 0, sizeof(g_emu_stats));
}

template <bool CW, int MODE>
static void run_items(const ScanParams& P, const RecView& V, const uint8_t* lo, const uint8_t* hi) {
    for (uint64_t item = 0; item < P.n_items; ++item) {
        TextWin T;
        T.emu_lo = lo;
        T.emu_hi = hi;
        Emitter E;
        const uint64_t o0 = P.offs[item], o1 = P.offs[item + 1];
        T.open(P.text + o0);
        E.begin((uint32_t)item);
        if (MODE == M_LEFTMOST)
            scan_leftmost<CW>(P, V, T, E, (uint32_t)(o1 - o0));
        else
            scan_standard<CW, MODE>(P, V, T, E, (uint32_t)(o1 - o0));
        E.finish(P);
    }
}

// Warp-level driver of the v1 lane machine, mirroring k_scan_std in dev_scan.cu with the warp
// collectives (ballot / any / shuffle) written out as loops over 32 lane states.
template <class M, class LANE>
static void run_machine(const ScanParams& P, const StdEnv& Ev0, const uint8_t* lo, int n_warps) {
    struct Warp {
        LANE L[32];
        Emitter E[32];
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
    // round-robin over warps, one "service + run" turn each, to interleave allocation order
    bool any_left = true;
    while (any_left) {
        any_left = false;
        for (auto& w : warps) {
            if (w.finished) continue;
            for (int l = 0; l < 32; ++l)
                if (w.L[l].fl & F_ACTIVE) M::drain(w.L[l], w.Ev[l], P, w.E[l]);
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
                unsigned long long base = P.ctrl->next_item;
                P.ctrl->next_item += __builtin_popcount(m);
                for (int l = 0; l < 32; ++l)
                    if (m & (1u << l)) {
                        const unsigned long long item = base + __builtin_popcount(m & ((1u << l) - 1u));
                        if (item < P.n_items)
                            M::begin_item(w.L[l], P, w.Ev[l], w.E[l], item, lo);
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
                bool waiting[32] = {false};
                for (int k = 0; k < M::TOPUP && !stop; ++k) {
                    bool need_service = false;
                    for (int l = 0; l < 32; ++l) {
                        const bool ok = M::step(w.L[l], w.Ev[l], lo);
                        if (!ok) waiting[l] = true;
                        if (!ok && (w.L[l].fl & F_ACTIVE)) need_service = true;
                    }
                    if (!M::LAZY && need_service) stop = true;
                }
                if (M::LEAN) {  // mirrors the votes in k_scan_machine
                    for (int l = 0; l < 32; ++l)
                        if ((w.L[l].fl & (F_ACTIVE | M::IDLE)) == (F_ACTIVE | M::IDLE)) stop = true;
                } else if (M::LAZY) {
                    for (int l = 0; l < 32; ++l)
                        if (waiting[l] && (w.L[l].fl & F_ACTIVE)) stop = true;
                }
            }
        }
    }
}

// k_scan_duo: StdMachine3 with two haystacks per lane (mirrors the kernel in dev_scan.cu)
template <int MODE>
static void run_duo(const ScanParams& P, const StdEnv& Ev0, int n_warps) {
    using M = StdMachine3<MODE>;
    struct Warp {
        Lane3 L[2][32];
        Emitter E[2][32];
        StdEnv Ev[2][32];
        std::vector<QEntry> queue;
        bool exhausted[32];
        bool finished;
    };
    std::vector<Warp> warps(n_warps);
    for (auto& w : warps) {
        w.queue.assign((size_t)LANE_Q * 32 * 2, QEntry{0, 0});
        for (int l = 0; l < 32; ++l) {
            for (int k = 0; k < 2; ++k) {
                w.L[k][l].fl = M::IDLE;
                w.L[k][l].qn = 0;
                w.E[k][l].begin(0);
                w.Ev[k][l] = Ev0;
                w.Ev[k][l].q = w.queue.data() + (size_t)k * LANE_Q * 32 + l;
                w.Ev[k][l].q_stride = 32;
            }
            w.exhausted[l] = false;
        }
        w.finished = false;
    }
    constexpr uint32_t WAIT = F_ACTIVE | F3_STOP;
    bool any_left = true;
    while (any_left) {
        any_left = false;
        for (auto& w : warps) {
            if (w.finished) continue;
            for (int k = 0; k < 2; ++k)
                for (int l = 0; l < 32; ++l)
                    if (w.L[k][l].fl & F_ACTIVE) M::drain(w.L[k][l], w.Ev[k][l], P, w.E[k][l]);
            for (int k = 0; k < 2; ++k)
                for (int l = 0; l < 32; ++l)
                    if ((w.L[k][l].fl & (F_ACTIVE | F_DONE)) == (F_ACTIVE | F_DONE)) {
                        w.E[k][l].finish(P);
                        M::finish_item(w.L[k][l], P);
                        w.L[k][l].fl = M::IDLE;
                    }
            unsigned m[2] = {0, 0};
            for (int k = 0; k < 2; ++k)
                for (int l = 0; l < 32; ++l)
                    if (!(w.L[k][l].fl & F_ACTIVE) && !w.exhausted[l]) m[k] |= 1u << l;
            if (m[0] | m[1]) {
                const unsigned long long base = P.ctrl->next_item;
                P.ctrl->next_item += __builtin_popcount(m[0]) + __builtin_popcount(m[1]);
                for (int l = 0; l < 32; ++l) {
                    const unsigned lt = (1u << l) - 1u;
                    for (int k = 0; k < 2; ++k)
                        if (m[k] & (1u << l)) {
                            const unsigned long long item = base + (k ? __builtin_popcount(m[0]) : 0) + __builtin_popcount(m[k] & lt);
                            if (item < P.n_items)
                                M::begin_item(w.L[k][l], P, w.Ev[k][l], w.E[k][l], item, nullptr);
                            else
                                w.exhausted[l] = true;
                        }
                }
            }
            bool any_active = false;
            for (int l = 0; l < 32; ++l) any_active |= ((w.L[0][l].fl | w.L[1][l].fl) & F_ACTIVE) != 0;
            if (!any_active) {
                w.finished = true;
                continue;
            }
            any_left = true;
            bool stop = false;
            while (!stop) {
                for (int k = 0; k < 2; ++k)
                    for (int l = 0; l < 32; ++l) M::text_topup(w.L[k][l], w.Ev[k][l], nullptr);
                for (int it = 0; it < M::TOPUP; ++it)
                    for (int l = 0; l < 32; ++l) {
                        uint32_t own0, own1;
                        const uint32_t a0 = M::probe(w.L[0][l], own0), a1 = M::probe(w.L[1][l], own1);
                        const uint4 x0 = M::fetch(w.Ev[0][l], a0), x1 = M::fetch(w.Ev[1][l], a1);
                        M::resolve(w.L[0][l], w.Ev[0][l], x0, a0, own0);
                        M::resolve(w.L[1][l], w.Ev[1][l], x1, a1, own1);
                    }
                for (int l = 0; l < 32; ++l)
                    if ((w.L[0][l].fl & WAIT) == WAIT || (w.L[1][l].fl & WAIT) == WAIT) stop = true;
            }
        }
    }
}

template <int MODE>
static void run_items_v1(const ScanParams& P, const StdEnv& Ev0, const uint8_t* lo, int n_warps) {
    run_machine<StdMachine<MODE>, LaneStd>(P, Ev0, lo, n_warps);
}

static uint32_t* g_state_io = nullptr;
static int g_stream_kernel = 3;       // which bytewise Standard machine serves emu_scan_stream_wire
static uint32_t g_stream_hot = 4096;  // ... and its shared-memory records
static uint32_t g_want_hot_slots = 65536;  // size of the hot region build_image() lays out
extern "C" void emu_set_hot_slots(uint32_t n) { g_want_hot_slots = n; }
extern "C" void emu_stream_config(int kernel, uint32_t hot_n) {
    g_stream_kernel = kernel;
    g_stream_hot = hot_n;
}
static const uint32_t* g_pos_in = nullptr;

extern "C" int emu_scan_batch_wire(const uint8_t* wire, size_t wire_len, int charwise, int mode,
                                   const uint8_t* text, const uint64_t* offs, uint64_t n, uint32_t hot_n,
                                   int kernel_version, uint32_t seg_len, uint32_t seg_from, uint32_t pool_blocks, dach_match* out, uint64_t out_cap, uint64_t* out_offs,
                                   uint64_t* needed) {
    dach_pma* pma = nullptr;
    size_t used = 0;
    int rc = wire_read(wire, wire_len, charwise != 0, &pma, &used);
    if (rc) return rc;
    HostImage img;
    img.want_hot_slots = g_want_hot_slots;
    rc = build_image(pma, &img);
    const bool lm = is_leftmost(pma->match_kind);
    delete pma;
    if (rc) return rc;
    if ((mode == M_LEFTMOST) != lm) return DACH_MATCH_KIND_MISMATCH;

    // kernel choice as enqueue_scan (one CTA per SM; StdMachine3's event queue and direct paths run the same lanes here)
    // seg_len > 0 cuts even an automaton the device scans whole (not segmentable): the hand-made case of
    // test_emu_lane.py shows with it why the device does not
    const ScanPlan plan = plan_scan({.opt_kernel = kernel_version, .compact = !img.crec.empty(),
                                     .charwise = charwise != 0, .root_opos = img.root_opos != 0,
                                     .root_base = img.root_base != 0, .segmentable = true, .opt_seg_len = seg_len,
                                     .stream = g_state_io != nullptr, .mode = mode});
    if (plan.refused) return DACH_INVALID_ARGUMENT;
    // segment table (mirrors k_seg_count / k_seg_fill in dev_scan.cu)
    const bool seg = plan.seg && seg_len > 0;
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
    std::vector<uint32_t> counts(n_items ? n_items : 1, 0);
    std::vector<uint32_t> pool((size_t)pool_blocks * BLK_WORDS, 0xdeadbeefu);
    ScanCtrl ctrl;
    memset(&ctrl, 0, sizeof(ctrl));
    ScanParams P;
    memset(&P, 0, sizeof(P));
    P.rec = reinterpret_cast<const uint4*>(img.rec.data());
    P.outputs = reinterpret_cast<const uint4*>(img.outputs.data());
    P.root_table = img.root_table.data();
    P.mapper = img.mapper.data();
    P.mapper_len = (uint32_t)img.mapper.size();
    P.n_slots = img.n_slots;
    P.root_opos = img.root_opos;
    if (hot_n > img.n_slots) hot_n = img.n_slots;
    P.hot_n = hot_n;
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
    P.pool = pool.data();
    P.pool_blocks = pool_blocks;
    P.ctrl = &ctrl;
    P.state_io = g_state_io;
    // "shared memory" copy of the hot records
    std::vector<uint32_t> hot(img.rec.begin(), img.rec.begin() + (size_t)hot_n * 4);
    hot.resize(hot.size() + 4);
    RecView V{P.rec, reinterpret_cast<const uint4*>(hot.data()), hot_n, img.root_table.data()};
    const uint8_t* lo = text + (n ? offs[0] : 0);
    const uint8_t* hi = text + (n ? offs[n] : 0);
    const Machine m = plan.machine;
    if (m != Machine::Lane) {
        // StdMachine3: the leading hot_n compact records are served from a "shared memory" copy; everything past
        // them in that copy is poison, so a wrong prefix compare cannot go unnoticed
        uint32_t entries = plan.std3() ? hot_n : 0;
        if (entries > img.hot_slots) entries = img.hot_slots;
        std::vector<uint32_t> tab(img.crec.size() ? img.crec.size() : 4, 0xdeadbeefu);
        memcpy(tab.data(), img.crec.data(), (size_t)entries * 16);
        StdEnv Ev{reinterpret_cast<const uint4*>(img.crec.data()), reinterpret_cast<const uint4*>(tab.data()), 0u, entries,
                  img.opos_tab.data(), P.text_end, P.text_lo, img.root_base, P.root_opos ? CF_OUT : 0u, nullptr, 0, 0, P.mapper, P.mapper_len,
                  reinterpret_cast<const uint4*>(img.crec.data())[D_ROOT]};
        const int n_warps = 3;
        const bool trace = getenv("DACH_EMU_TRACE") != nullptr;
        switch (m) {
            case Machine::Cw:
                if (trace) fprintf(stderr, "emu: charwise lane machine\n");
                if (mode == M_FIND) run_machine<CwMachine<M_FIND>, LaneCw>(P, Ev, lo, n_warps);
                if (mode == M_OVERLAPPING) run_machine<CwMachine<M_OVERLAPPING>, LaneCw>(P, Ev, lo, n_warps);
                if (mode == M_NO_SUFFIX) run_machine<CwMachine<M_NO_SUFFIX>, LaneCw>(P, Ev, lo, n_warps);
                if (mode == M_LEFTMOST) run_machine<CwMachine<M_LEFTMOST>, LaneCw>(P, Ev, lo, n_warps);
                break;
            case Machine::Duo:
                if (trace) fprintf(stderr, "emu: StdMachine3, two haystacks per lane\n");
                Ev.hot_n = 0;
                if (mode == M_FIND) run_duo<M_FIND>(P, Ev, n_warps);
                if (mode == M_OVERLAPPING) run_duo<M_OVERLAPPING>(P, Ev, n_warps);
                if (mode == M_NO_SUFFIX) run_duo<M_NO_SUFFIX>(P, Ev, n_warps);
                break;
            case Machine::Std3:
            case Machine::Std3Direct:
                if (trace) fprintf(stderr, "emu: StdMachine3, %u hot records\n", entries);
                if (mode == M_FIND) run_machine<StdMachine3<M_FIND>, Lane3>(P, Ev, lo, n_warps);
                if (mode == M_OVERLAPPING) run_machine<StdMachine3<M_OVERLAPPING>, Lane3>(P, Ev, lo, n_warps);
                if (mode == M_NO_SUFFIX) run_machine<StdMachine3<M_NO_SUFFIX>, Lane3>(P, Ev, lo, n_warps);
                break;
            case Machine::Std2:
                if (trace) fprintf(stderr, "emu: StdMachine2\n");
                if (mode == M_FIND) run_machine<StdMachine2<M_FIND>, Lane2>(P, Ev, lo, n_warps);
                if (mode == M_OVERLAPPING) run_machine<StdMachine2<M_OVERLAPPING>, Lane2>(P, Ev, lo, n_warps);
                if (mode == M_NO_SUFFIX) run_machine<StdMachine2<M_NO_SUFFIX>, Lane2>(P, Ev, lo, n_warps);
                break;
            case Machine::Lm:
                if (trace) fprintf(stderr, "emu: leftmost lane machine\n");
                run_machine<LmMachine, LaneLm>(P, Ev, lo, n_warps);
                break;
            default:
                if (mode == M_FIND) run_items_v1<M_FIND>(P, Ev, lo, n_warps);
                if (mode == M_OVERLAPPING) run_items_v1<M_OVERLAPPING>(P, Ev, lo, n_warps);
                if (mode == M_NO_SUFFIX) run_items_v1<M_NO_SUFFIX>(P, Ev, lo, n_warps);
        }
    } else
    switch ((charwise ? 4 : 0) + mode) {
        case 0: run_items<false, M_FIND>(P, V, lo, hi); break;
        case 1: run_items<false, M_OVERLAPPING>(P, V, lo, hi); break;
        case 2: run_items<false, M_NO_SUFFIX>(P, V, lo, hi); break;
        case 3: run_items<false, M_LEFTMOST>(P, V, lo, hi); break;
        case 4: run_items<true, M_FIND>(P, V, lo, hi); break;
        case 5: run_items<true, M_OVERLAPPING>(P, V, lo, hi); break;
        case 6: run_items<true, M_NO_SUFFIX>(P, V, lo, hi); break;
        case 7: run_items<true, M_LEFTMOST>(P, V, lo, hi); break;
        default: return DACH_INVALID_ARGUMENT;
    }
    // offsets (k_offsets_*), per-haystack offsets (k_hay_offsets) and gather (k_gather)
    std::vector<uint64_t> item_offs(n_items + 1, 0);
    for (uint64_t i = 0; i < n_items; ++i) item_offs[i + 1] = item_offs[i] + counts[i];
    const uint64_t run = item_offs[n_items] + ((uint64_t)ctrl.carries << 32);  // finish_scan: exact past 2^32
    for (uint64_t h = 0; h <= n; ++h) out_offs[h] = seg ? item_offs[seg_first[h]] : item_offs[h];
    if (needed) *needed = run;
    if (ctrl.carries) return DACH_INVALID_ARGUMENT;  // a haystack with 2^32 or more matches cannot be placed
    if (ctrl.overflow || run > out_cap) return DACH_OUTPUT_OVERFLOW;
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
    if (g_pos_in)  // k_add_base
        for (uint64_t h = 0; h < n; ++h)
            for (uint64_t m = out_offs[h]; m < out_offs[h + 1]; ++m) {
                out_words[m * 3 + 0] += g_pos_in[h];
                out_words[m * 3 + 1] += g_pos_in[h];
            }
    return DACH_OK;
}

// dach_dev_scan_stream: chunks of streams (state in/out per haystack, optional base position)
static int g_stream_charwise = 0;
extern "C" void emu_stream_charwise(int cw) { g_stream_charwise = cw; }
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
    dach_pma* pma = nullptr;
    size_t used = 0;
    if (wire_read(wire, wire_len, false, &pma, &used)) return -1;
    HostImage img;
    const int rc = build_image(pma, &img);
    delete pma;
    return rc ? -1 : (img.segmentable ? 1 : 0);
}
