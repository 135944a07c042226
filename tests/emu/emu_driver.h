// CPU restatement of the scan kernels' drivers (TEST INFRASTRUCTURE ONLY).
//
// The emulation compiles daachorse_b200/csrc/scan_lane.cuh -- the exact lane logic the CUDA kernels run -- with g++
// (-DDACH_EMU) and drives it the way dev_scan.cu does: items -> lanes of warps of CTAs, the warp collectives (ballot /
// any / shuffle) written out as loops over 32 lane states, several warps interleaved one service phase and run at a
// time.  Every device loop and every piece of per-call setup is written here once; the emu_*.cpp files hold only what
// one result kind does on its own (its checks, its sink's outputs, its post-processing).  It is never loaded by the
// product.
#pragma once

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <type_traits>
#include <vector>

#include "../../daachorse_b200/csrc/dev_image.h"
#include "../../daachorse_b200/csrc/host.h"
#include "../../daachorse_b200/csrc/scan_lane.cuh"
#include "../../daachorse_b200/csrc/scan_plan.h"

namespace emu {
using namespace dach;

inline uint32_t g_want_hot_slots = 65536;  // size of the hot region build_image() lays out (emu_set_hot_slots)

// wire_read + build_image: the device image of a serialized automaton, and whether it is a leftmost one
inline int load(const uint8_t* wire, size_t wire_len, bool charwise, HostImage* img, bool* lm = nullptr) {
    dach_pma* pma = nullptr;
    size_t used = 0;
    int rc = wire_read(wire, wire_len, charwise, &pma, &used);
    if (rc) return rc;
    img->want_hot_slots = g_want_hot_slots;
    rc = build_image(pma, img);
    if (lm) *lm = is_leftmost(pma->match_kind);
    delete pma;
    return rc;
}

// what plan_scan needs to know of the image; the caller adds the options and the result kind
inline ScanInputs plan_inputs(const HostImage& img, bool charwise, int mode) {
    ScanInputs in;
    in.compact = !img.crec.empty();
    in.charwise = charwise;
    in.root_opos = img.root_opos != 0;
    in.root_base = img.root_base != 0;
    in.segmentable = img.segmentable;
    in.mode = mode;
    return in;
}

// k_seg_count / k_seg_fill: haystacks below seg_from stay whole, the others are cut into seg_len-byte items (an empty
// haystack still is one item).  seg_len == 0: one item per haystack.
struct Segments {
    std::vector<uint32_t> item_hay, item_beg;
    std::vector<uint64_t> seg_first;  // haystack h's items are [seg_first[h], seg_first[h + 1])
    uint64_t n_items = 0;
    uint32_t seg_len = 0, seg_from = 0;
    uint64_t first(uint64_t h) const { return seg_len ? seg_first[h] : h; }
};

inline Segments seg_table(const uint64_t* offs, uint64_t n, uint32_t seg_len, uint32_t seg_from) {
    Segments S;
    S.n_items = n;
    S.seg_len = seg_len;
    S.seg_from = seg_from;
    if (!seg_len) return S;
    S.seg_first.assign(n + 1, 0);
    for (uint64_t h = 0; h < n; ++h) {
        uint64_t k = h < seg_from ? 1 : (offs[h + 1] - offs[h] + seg_len - 1) / seg_len;
        if (k == 0) k = 1;
        S.seg_first[h + 1] = S.seg_first[h] + k;
        for (uint64_t j = 0; j < k; ++j) {
            S.item_hay.push_back((uint32_t)h);
            S.item_beg.push_back((uint32_t)(j * seg_len));
        }
    }
    S.n_items = S.seg_first[n];
    return S;
}

// The ScanParams fields every scan sets alike: the image, the batch's text bounds, the items.  The result fields are
// the caller's.
inline ScanParams scan_params(const HostImage& img, const uint8_t* text, const uint64_t* offs, uint64_t n, const Segments& S,
                              ScanCtrl* ctrl) {
    ScanParams P;
    memset(&P, 0, sizeof(P));
    P.rec = reinterpret_cast<const uint4*>(img.rec.data());
    P.outputs = reinterpret_cast<const uint4*>(img.outputs.data());
    P.root_table = img.root_table.data();
    P.opos_tab = img.opos_tab.data();
    P.mapper = img.mapper.data();
    P.mapper_len = (uint32_t)img.mapper.size();
    P.n_slots = img.n_slots;
    P.root_opos = img.root_opos;
    P.text = text;
    P.text_lo = text + (n ? offs[0] : 0);
    P.text_end = text + (n ? offs[n] : 0);
    if (img.hot_slots) {  // the compact image is renumbered: stream state ids are translated at the boundary
        P.id_in = img.new_of_old.data();
        P.id_out = img.old_of_new.data();
    }
    P.offs = offs;
    P.n_items = S.n_items;
    if (S.seg_len) {
        P.item_hay = S.item_hay.data();
        P.item_beg = S.item_beg.data();
        P.seg_len = S.seg_len;
        P.seg_from = S.seg_from;
        P.warm = img.max_pattern_len ? img.max_pattern_len - 1 : 0;
    }
    P.ctrl = ctrl;
    return P;
}

// The kernels' shared memory.  Lane per haystack: the leading min(hot_n, n_slots) wide records behind RecView.
// StdMachine3 (and only it): the leading min(hot_n, hot_slots) compact records, in a copy whose remainder is poison so
// that a wrong prefix compare cannot go unnoticed; the other lane machines get the poisoned copy with no entries.
struct Smem {
    std::vector<uint32_t> hot, tab;
    RecView V{};
    StdEnv Ev{};

    Smem(const HostImage& img, const ScanPlan& plan, uint32_t hot_n, const uint8_t* text_lo, const uint8_t* text_end) {
        const uint32_t hot_w = plan.machine == Machine::Lane ? std::min(hot_n, img.n_slots) : 0u;
        hot.assign(img.rec.begin(), img.rec.begin() + (size_t)hot_w * 4);
        hot.resize(hot.size() + 4);
        V = RecView{reinterpret_cast<const uint4*>(img.rec.data()), reinterpret_cast<const uint4*>(hot.data()), hot_w,
                    img.root_table.data()};
        if (img.crec.empty()) return;
        const uint32_t entries = plan.std3() ? std::min(hot_n, img.hot_slots) : 0u;
        tab.assign(img.crec.size(), 0xdeadbeefu);
        memcpy(tab.data(), img.crec.data(), (size_t)entries * 16);
        const uint4* crec = reinterpret_cast<const uint4*>(img.crec.data());
        Ev = StdEnv{crec, reinterpret_cast<const uint4*>(tab.data()), 0u, entries, img.opos_tab.data(), text_end, text_lo, img.root_base,
                    img.root_opos ? CF_OUT : 0u, nullptr, 0, 0, img.mapper.data(), (uint32_t)img.mapper.size(), crec[D_ROOT]};
    }
};

// scan_items in dev_scan.cu (k_scan / k_scan_rk): one lane per haystack, the reference-shaped loops
template <bool CW, int MODE, class SINK>
void run_items(const ScanParams& P, const RecView& V, const uint8_t* lo, const uint8_t* hi) {
    for (uint64_t item = 0; item < P.n_items; ++item) {
        TextWin T;
        T.emu_lo = lo;
        T.emu_hi = hi;
        SINK E;
        const uint64_t o0 = P.offs[item], o1 = P.offs[item + 1];
        T.open(P.text + o0);
        E.begin((uint32_t)item);
        if constexpr (SINK::KIND == RK_MASK) E.base = P.mask_out + o0;
        if (MODE == M_LEFTMOST)
            scan_leftmost<CW>(P, V, T, E, (uint32_t)(o1 - o0));
        else
            scan_standard<CW, MODE>(P, V, T, E, (uint32_t)(o1 - o0));
        E.finish(P);
    }
}

// scan_machine in dev_scan.cu (k_scan_machine / k_scan_machine_rk): M the lane machine, OPS where drain() and
// begin_item() come from, SINK the result.  n_ctas CTAs of n_warps warps take turns, one service phase and one run of
// lock-step iterations each, so that the order in which they take items, blocks and counters interleaves.
template <class M, class OPS, class LANE, class SINK>
void run_machine(const ScanParams& P, const StdEnv& Ev0, const uint8_t* lo, int n_ctas, int n_warps) {
    struct Warp {
        LANE L[32];
        SINK E[32];
        StdEnv Ev[32];
        std::vector<QEntry> queue;
        bool exhausted[32];
        bool finished;
    };
    // HIST: each CTA's shared-memory counters of the compact slots [0, hist_smem)
    std::vector<std::vector<unsigned int>> cta_cnt(n_ctas, std::vector<unsigned int>(P.hist_smem + 1, 0));
    std::vector<Warp> warps((size_t)n_ctas * n_warps);
    for (size_t wi = 0; wi < warps.size(); ++wi) {
        Warp& w = warps[wi];
        w.queue.assign((size_t)LANE_Q * 32, QEntry{0, 0});
        for (int l = 0; l < 32; ++l) {
            w.L[l].fl = M::IDLE;
            w.L[l].qn = 0;
            w.E[l].begin(0);
            if constexpr (SINK::KIND == RK_HIST) {
                w.E[l].s_cnt = cta_cnt[wi / n_warps].data();
                w.E[l].k = P.hist_smem;
            }
            w.exhausted[l] = false;
            w.Ev[l] = Ev0;
            w.Ev[l].q = w.queue.data() + l;
            w.Ev[l].q_stride = 32;
        }
        w.finished = false;
    }
    bool any_left = true;
    while (any_left) {
        any_left = false;
        for (auto& w : warps) {
            if (w.finished) continue;
            // ---- service phase ----
            if constexpr (std::is_same<SINK, EventSink>::value) {
                // event blocks: the lanes that need one this phase take them with one atomic for the warp
                unsigned mb = 0;
                for (int l = 0; l < 32; ++l)
                    if ((w.L[l].fl & F_ACTIVE) && OPS::need_block(w.L[l], w.Ev[l], w.E[l])) mb |= 1u << l;
                const uint32_t b0 = P.ctrl->blk_cursor;
                P.ctrl->blk_cursor += __builtin_popcount(mb);
                for (int l = 0; l < 32; ++l)
                    if (w.L[l].fl & F_ACTIVE) OPS::drain(w.L[l], w.Ev[l], P, w.E[l], b0 + __builtin_popcount(mb & ((1u << l) - 1u)));
            } else {
                for (int l = 0; l < 32; ++l)
                    if (w.L[l].fl & F_ACTIVE) OPS::drain(w.L[l], w.Ev[l], P, w.E[l]);
            }
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
            // ---- lock-step iterations until some lane needs service: the device's three votes ----
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
                    if (!M::LAZY && need_service) stop = true;  // eager: after the iteration that needs it
                }
                if (M::LEAN) {  // the lane's stop bit, once per top-up period
                    for (int l = 0; l < 32; ++l)
                        if ((w.L[l].fl & (F_ACTIVE | M::IDLE)) == (F_ACTIVE | M::IDLE)) stop = true;
                } else if (M::LAZY) {  // lanes that needed service during the period
                    for (int l = 0; l < 32; ++l)
                        if (waiting[l] && (w.L[l].fl & F_ACTIVE)) stop = true;
                }
            }
        }
    }
    if constexpr (SINK::KIND == RK_HIST)  // the end of every CTA: its counters go to global memory once
        for (auto& c : cta_cnt)
            for (uint32_t i = 0; i < P.hist_smem; ++i) P.slot_hist[i] += c[i];
}

// k_scan_direct: StdMachine3's matches path without the queue, one CTA of n_warps warps
template <int MODE>
void run_direct(const ScanParams& P, const StdEnv& Ev, const uint8_t* lo, int n_warps) {
    using M = StdMachine3<MODE>;
    using OPS = DirectOps<MODE>;
    struct Warp {
        Lane3D L[32];
        bool exhausted[32];
        bool finished;
    };
    std::vector<Warp> warps(n_warps);
    for (auto& w : warps) {
        for (int l = 0; l < 32; ++l) {
            w.L[l].fl = M::IDLE;
            w.L[l].qn = 0;
            w.L[l].E.begin(0);
            w.exhausted[l] = false;
        }
        w.finished = false;
    }
    bool any_left = true;
    while (any_left) {
        any_left = false;
        for (auto& w : warps) {
            if (w.finished) continue;
            unsigned mb = 0;
            for (int l = 0; l < 32; ++l)
                if (OPS::need_block(w.L[l])) mb |= 1u << l;
            const uint32_t b0 = P.ctrl->blk_cursor;
            P.ctrl->blk_cursor += __builtin_popcount(mb);
            for (int l = 0; l < 32; ++l)
                if (w.L[l].fl & F_ACTIVE) OPS::drain(w.L[l], Ev, P, b0 + __builtin_popcount(mb & ((1u << l) - 1u)));
            for (int l = 0; l < 32; ++l)
                if ((w.L[l].fl & (F_ACTIVE | F_DONE)) == (F_ACTIVE | F_DONE)) {
                    w.L[l].E.finish(P);
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
                            OPS::begin_item(w.L[l], P, Ev, item);
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
                for (int l = 0; l < 32; ++l) M::text_topup(w.L[l], Ev, lo);
                for (int k = 0; k < M::TOPUP; ++k)
                    for (int l = 0; l < 32; ++l) (void)M::step(w.L[l], Ev, lo);
                for (int l = 0; l < 32; ++l)
                    if ((w.L[l].fl & (F_ACTIVE | F3_STOP)) == (F_ACTIVE | F3_STOP)) stop = true;
            }
        }
    }
}

// k_scan_duo: StdMachine3 with two haystacks per lane, one CTA of n_warps warps
template <int MODE>
void run_duo(const ScanParams& P, const StdEnv& Ev0, int n_warps) {
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

// f(std::integral_constant<int, MODE>{}) for the run-time iterator `mode`
template <class F>
void for_mode(int mode, F&& f) {
    switch (mode) {
        case M_FIND: return f(std::integral_constant<int, M_FIND>{});
        case M_OVERLAPPING: return f(std::integral_constant<int, M_OVERLAPPING>{});
        case M_NO_SUFFIX: return f(std::integral_constant<int, M_NO_SUFFIX>{});
        case M_LEFTMOST: return f(std::integral_constant<int, M_LEFTMOST>{});
    }
}

// launch_matches in dev_scan.cu, with each machine's own drain storing the tuples: StdMachine3 runs the same lanes
// for the queue and the direct kernel (their event paths are emu_events.cpp's), the duo loop without staged records.
// The lane machines run one CTA of n_warps warps.
template <int MODE>
void run_matches(Machine m, bool cw, const ScanParams& P, const Smem& S, int n_warps) {
    const uint8_t *lo = P.text_lo, *hi = P.text_end;
    if constexpr (MODE == M_LEFTMOST) {
        if (m == Machine::Lm) return run_machine<LmMachine, LmMachine, LaneLm, Emitter>(P, S.Ev, lo, 1, n_warps);
    } else {
        switch (m) {
            case Machine::Std: return run_machine<StdMachine<MODE>, StdMachine<MODE>, LaneStd, Emitter>(P, S.Ev, lo, 1, n_warps);
            case Machine::Std2: return run_machine<StdMachine2<MODE>, StdMachine2<MODE>, Lane2, Emitter>(P, S.Ev, lo, 1, n_warps);
            case Machine::Std3:
            case Machine::Std3Direct: return run_machine<StdMachine3<MODE>, StdMachine3<MODE>, Lane3, Emitter>(P, S.Ev, lo, 1, n_warps);
            case Machine::Duo: {
                StdEnv Ev = S.Ev;
                Ev.hot_n = 0;
                return run_duo<MODE>(P, Ev, n_warps);
            }
            default: break;
        }
    }
    if (m == Machine::Cw) return run_machine<CwMachine<MODE>, CwMachine<MODE>, LaneCw, Emitter>(P, S.Ev, lo, 1, n_warps);
    return cw ? run_items<true, MODE, Emitter>(P, S.V, lo, hi) : run_items<false, MODE, Emitter>(P, S.V, lo, hi);
}

// launch_rk in dev_scan.cu: result kind RK of iterator MODE on machine m; the lane machines run n_ctas CTAs of n_warps
// warps.  FIRST is built for the iterators plan_scan leaves it, FIRST_STREAM for the two steppers.
template <int RK, int MODE>
void run_rk(Machine m, bool cw, const ScanParams& P, const Smem& S, int n_ctas, int n_warps) {
    constexpr bool built = RK == RK_FIRST ? MODE == M_OVERLAPPING || MODE == M_LEFTMOST
                           : RK == RK_FIRST_STREAM ? MODE == M_FIND || MODE == M_OVERLAPPING
                                                   : true;
    const uint8_t *lo = P.text_lo, *hi = P.text_end;
    if constexpr (built) {
        if constexpr (MODE != M_LEFTMOST)
            if (m == Machine::Std3)
                return run_machine<StdMachine3<MODE>, SinkOps<StdMachine3<MODE>, MODE, RK>, Lane3,
                                   typename SinkOps<StdMachine3<MODE>, MODE, RK>::Sink>(P, S.Ev, lo, n_ctas, n_warps);
        if (m == Machine::Cw)
            return run_machine<CwMachine<MODE>, SinkOps<CwMachine<MODE>, MODE, RK>, LaneCw, typename SinkOps<CwMachine<MODE>, MODE, RK>::Sink>(
                P, S.Ev, lo, n_ctas, n_warps);
        if constexpr (RK != RK_FIRST_STREAM) {
            using SINK = typename SinkOps<LmMachine, M_LEFTMOST, RK>::Sink;
            if constexpr (MODE == M_LEFTMOST)
                if (m == Machine::Lm)
                    return run_machine<LmMachine, SinkOps<LmMachine, M_LEFTMOST, RK>, LaneLm, SINK>(P, S.Ev, lo, n_ctas, n_warps);
            if (m == Machine::Lane) return cw ? run_items<true, MODE, SINK>(P, S.V, lo, hi) : run_items<false, MODE, SINK>(P, S.V, lo, hi);
        }
    }
}

template <int RK>
void run_rk_modes(const ScanPlan& plan, bool cw, const ScanParams& P, const Smem& S, int n_ctas, int n_warps) {
    for_mode(plan.mode, [&](auto M) { run_rk<RK, decltype(M)::value>(plan.machine, cw, P, S, n_ctas, n_warps); });
}

// ---- post-passes ----------------------------------------------------------------------------------------------------

// k_offsets_* and the per-haystack offsets of the matches paths, then finish_scan's refusals.  item_offs: the first
// match of every item.
inline int offsets(const Segments& S, uint64_t n, const std::vector<uint32_t>& counts, const ScanCtrl& ctrl, uint64_t out_cap,
                   std::vector<uint64_t>& item_offs, uint64_t* out_offs, uint64_t* needed) {
    item_offs.assign(S.n_items + 1, 0);
    for (uint64_t i = 0; i < S.n_items; ++i) item_offs[i + 1] = item_offs[i] + counts[i];
    const uint64_t total = item_offs[S.n_items] + ((uint64_t)ctrl.carries << 32);  // finish_scan: exact past 2^32
    for (uint64_t h = 0; h <= n; ++h) out_offs[h] = item_offs[S.first(h)];
    if (needed) *needed = total;
    if (ctrl.carries) return DACH_INVALID_ARGUMENT;  // a haystack with 2^32 or more matches cannot be placed
    if (ctrl.overflow || total > out_cap) return DACH_OUTPUT_OVERFLOW;
    return DACH_OK;
}

// k_add_base: stream chunks report positions in stream coordinates
inline void add_base(uint32_t* out_words, const uint64_t* out_offs, uint64_t n, const uint32_t* pos) {
    for (uint64_t h = 0; h < n; ++h)
        for (uint64_t m = out_offs[h]; m < out_offs[h + 1]; ++m) {
            out_words[m * 3 + 0] += pos[h];
            out_words[m * 3 + 1] += pos[h];
        }
}

// k_count_hay: a haystack's count is the sum over its items; returns the total
inline uint64_t fold_count(const Segments& S, uint64_t n, const std::vector<unsigned long long>& item_count, uint64_t* counts) {
    uint64_t tot = 0;
    for (uint64_t h = 0; h < n; ++h) {
        uint64_t v = 0;
        for (uint64_t i = S.first(h); i < S.first(h + 1); ++i) v += item_count[i];
        counts[h] = v;
        tot += v;
    }
    return tot;
}

// k_first_hay / k_first_stream: a haystack's first match is the one of its lowest item that has one, plus pos[h] where
// stream chunks report stream coordinates; returns the haystacks with a match
inline uint64_t fold_first(const Segments& S, uint64_t n, const std::vector<uint4>& item_first, const uint32_t* pos, uint32_t* first,
                           uint8_t* found) {
    uint64_t tot = 0;
    for (uint64_t h = 0; h < n; ++h) {
        const uint64_t a = S.first(h), b = S.first(h + 1);
        uint4 r = item_first[a];
        for (uint64_t i = a + 1; i < b && !r.w; ++i) r = item_first[i];
        const uint32_t base = (r.w && pos) ? pos[h] : 0u;
        first[h * 3 + 0] = r.x + base, first[h * 3 + 1] = r.y + base, first[h * 3 + 2] = r.z;
        found[h] = r.w ? 1 : 0;
        tot += r.w ? 1 : 0;
    }
    return tot;
}

// check_hist in dev_scan.cu: the key is 0 (output record) or 1 (value), and n_hist has room for every key
inline bool check_hist(const HostImage& img, int key, uint64_t n_hist) {
    const uint32_t n_out = (uint32_t)(img.outputs.size() / 4);
    uint32_t max_value = 0;
    for (uint32_t i = 0; i < n_out; ++i) max_value = std::max(max_value, img.outputs[(size_t)i * 4]);
    if (key != 0 && key != 1) return false;
    return !(key == 0 ? n_hist < n_out : (n_out && n_hist <= max_value));
}

// k_hist_heads (lane machines: events per compact slot -> per output record) and k_hist_fold (each record's count to
// its key, along the parent chain where an event stands for a whole find_overlapping list); returns the matches added
inline uint64_t hist_fold(const HostImage& img, bool machine, int mode, const std::vector<unsigned long long>& slot_hist,
                          std::vector<unsigned long long>& rec_hist, int key, uint64_t* hist) {
    if (machine)
        for (uint32_t s = 0; s < (uint32_t)img.opos_tab.size(); ++s)
            if (slot_hist[s] && img.opos_tab[s]) rec_hist[img.opos_tab[s] - 1] += slot_hist[s];
    const bool chain = machine && mode == M_OVERLAPPING;
    uint64_t tot = 0;
    for (uint32_t i = 0; i < (uint32_t)(img.outputs.size() / 4); ++i) {
        const unsigned long long v = rec_hist[i];
        for (uint32_t j = v ? i + 1 : 0; j;) {
            const uint32_t* o = img.outputs.data() + (size_t)(j - 1) * 4;
            hist[key ? o[0] : j - 1] += v;
            tot += v;
            j = chain ? o[2] : 0;
        }
    }
    return tot;
}

}  // namespace emu
