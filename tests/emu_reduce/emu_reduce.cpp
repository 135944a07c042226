// CPU emulation of COUNT / FIRST scans (TEST INFRASTRUCTURE ONLY).
//
// Compiles daachorse_b200/csrc/scan_lane.cuh -- the exact lane logic the CUDA kernels run -- with g++ (-DDACH_EMU)
// and drives it the way enqueue_rk() in dev_scan.cu does: items -> lanes of a warp (the warp collectives written out
// as loops over 32 lane states), the machine's step() with SinkOps' drain() / begin_item(), or the lane-per-haystack
// loops with a CountSink / FirstSink, then the per-haystack results of k_count_hay / k_first_hay.  It is never loaded
// by the product.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <vector>

#include "../../daachorse_b200/csrc/dev_image.h"
#include "../../daachorse_b200/csrc/host.h"
#include "../../daachorse_b200/csrc/scan_lane.cuh"

using namespace dach;

namespace dach {
EmuStats g_emu_stats;
}
extern "C" void emu_stats(unsigned long long* out, int reset) {
    memcpy(out, &g_emu_stats, sizeof(g_emu_stats));
    if (reset) memset(&g_emu_stats, 0, sizeof(g_emu_stats));
}

static uint32_t g_want_hot_slots = 65536;  // size of the hot region build_image() lays out
extern "C" void emu_set_hot_slots(uint32_t n) { g_want_hot_slots = n; }

// k_scan_rk: one lane per haystack, the reference-shaped loops
template <bool CW, int MODE, class SINK>
static void run_items(const ScanParams& P, const RecView& V, const uint8_t* lo, const uint8_t* hi) {
    for (uint64_t item = 0; item < P.n_items; ++item) {
        TextWin T;
        T.emu_lo = lo;
        T.emu_hi = hi;
        SINK E;
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

// k_scan_machine_rk: the service phase / lock-step loop of scan_machine() in dev_scan.cu, several warps interleaved
template <class M, class LANE, class OPS, class SINK>
static void run_machine(const ScanParams& P, const StdEnv& Ev0, const uint8_t* lo, int n_warps) {
    struct Warp {
        LANE L[32];
        SINK E[32];
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
    unsigned long long next_item = 0;
    bool any_left = true;
    while (any_left) {
        any_left = false;
        for (auto& w : warps) {
            if (w.finished) continue;
            for (int l = 0; l < 32; ++l)
                if (w.L[l].fl & F_ACTIVE) OPS::drain(w.L[l], w.Ev[l], P, w.E[l]);
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
                const unsigned long long base = next_item;
                next_item += __builtin_popcount(m);
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
                bool waiting[32] = {false};
                for (int k = 0; k < M::TOPUP; ++k)
                    for (int l = 0; l < 32; ++l)
                        if (!M::step(w.L[l], w.Ev[l], lo)) waiting[l] = true;
                for (int l = 0; l < 32; ++l) {
                    if (M::LEAN && (w.L[l].fl & (F_ACTIVE | M::IDLE)) == (F_ACTIVE | M::IDLE)) stop = true;
                    if (!M::LEAN && waiting[l] && (w.L[l].fl & F_ACTIVE)) stop = true;
                }
            }
        }
    }
}

// launch_rk in dev_scan.cu: which = 3 StdMachine3, 1 LmMachine / CwMachine, 0 lane per haystack
template <int RK>
static void run_rk(const ScanParams& P, const RecView& V, const StdEnv& Ev, const uint8_t* lo, const uint8_t* hi, bool cw, int which,
                   int mode) {
    using S = typename std::conditional<RK == RK_COUNT, CountSink, FirstSink>::type;
    const int nw = 3;
    if (which == 3) {
        if (mode == M_FIND) run_machine<StdMachine3<M_FIND>, Lane3, SinkOps<StdMachine3<M_FIND>, M_FIND, RK>, S>(P, Ev, lo, nw);
        if (mode == M_NO_SUFFIX)
            run_machine<StdMachine3<M_NO_SUFFIX>, Lane3, SinkOps<StdMachine3<M_NO_SUFFIX>, M_NO_SUFFIX, RK>, S>(P, Ev, lo, nw);
        if (mode == M_OVERLAPPING)
            run_machine<StdMachine3<M_OVERLAPPING>, Lane3, SinkOps<StdMachine3<M_OVERLAPPING>, M_OVERLAPPING, RK>, S>(P, Ev, lo, nw);
    } else if (which == 1 && cw) {
        if (mode == M_FIND) run_machine<CwMachine<M_FIND>, LaneCw, SinkOps<CwMachine<M_FIND>, M_FIND, RK>, S>(P, Ev, lo, nw);
        if (mode == M_NO_SUFFIX) run_machine<CwMachine<M_NO_SUFFIX>, LaneCw, SinkOps<CwMachine<M_NO_SUFFIX>, M_NO_SUFFIX, RK>, S>(P, Ev, lo, nw);
        if (mode == M_OVERLAPPING)
            run_machine<CwMachine<M_OVERLAPPING>, LaneCw, SinkOps<CwMachine<M_OVERLAPPING>, M_OVERLAPPING, RK>, S>(P, Ev, lo, nw);
        if (mode == M_LEFTMOST) run_machine<CwMachine<M_LEFTMOST>, LaneCw, SinkOps<CwMachine<M_LEFTMOST>, M_LEFTMOST, RK>, S>(P, Ev, lo, nw);
    } else if (which == 1) {
        run_machine<LmMachine, LaneLm, SinkOps<LmMachine, M_LEFTMOST, RK>, S>(P, Ev, lo, nw);
    } else {
        switch ((cw ? 4 : 0) + mode) {
            case 0: run_items<false, M_FIND, S>(P, V, lo, hi); break;
            case 1: run_items<false, M_OVERLAPPING, S>(P, V, lo, hi); break;
            case 2: run_items<false, M_NO_SUFFIX, S>(P, V, lo, hi); break;
            case 3: run_items<false, M_LEFTMOST, S>(P, V, lo, hi); break;
            case 4: run_items<true, M_FIND, S>(P, V, lo, hi); break;
            case 5: run_items<true, M_OVERLAPPING, S>(P, V, lo, hi); break;
            case 6: run_items<true, M_NO_SUFFIX, S>(P, V, lo, hi); break;
            case 7: run_items<true, M_LEFTMOST, S>(P, V, lo, hi); break;
        }
    }
}

// dach_dev_count_batch (rk = RK_COUNT: counts, n x u64) / dach_dev_first_batch (rk = RK_FIRST: first, n x 3 u32, and
// found, n x u8).  *total = the sum of the counts / the haystacks with a match.  hot_n: StdMachine3 records served from
// the "shared memory" copy (leftmost / charwise / kernel 0: leading wide records of k_scan_rk), kernel: the option
// (1, 2 and 4 run 3, as on the device), seg_len > 0: segments of that length where the device may cut.
extern "C" int emu_reduce_batch_wire(const uint8_t* wire, size_t wire_len, int charwise, int mode, int rk, const uint8_t* text,
                                     const uint64_t* offs, uint64_t n, uint32_t hot_n, int kernel, uint32_t seg_len,
                                     uint64_t* counts, uint32_t* first, uint8_t* found, uint64_t* total) {
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
    if (mode < M_FIND || mode > M_LEFTMOST || (rk != RK_COUNT && rk != RK_FIRST)) return DACH_INVALID_ARGUMENT;
    if ((mode == M_LEFTMOST) != lm) return DACH_MATCH_KIND_MISMATCH;
    // kernel choice and segments as enqueue_rk
    const int mmode = (rk == RK_FIRST && mode != M_LEFTMOST) ? M_OVERLAPPING : mode;
    const bool v1 = kernel >= 1 && !img.crec.empty() && !(mmode == M_FIND && img.root_opos != 0);
    const bool cw_machine = v1 && charwise;
    const bool lm_machine = v1 && !charwise && mmode == M_LEFTMOST;
    const bool std3 = v1 && !charwise && mmode != M_LEFTMOST && img.root_base != 0;
    const int which = std3 ? 3 : (cw_machine || lm_machine) ? 1 : 0;
    const bool seg = std3 && seg_len > 0 && (mmode == M_OVERLAPPING || mmode == M_NO_SUFFIX);
    std::vector<uint32_t> item_hay, item_beg;
    std::vector<uint64_t> seg_first(n + 1, 0);
    uint64_t n_items = n;
    if (seg) {  // k_seg_count / k_seg_fill
        for (uint64_t h = 0; h < n; ++h) {
            uint64_t k = (offs[h + 1] - offs[h] + seg_len - 1) / seg_len;
            if (k == 0) k = 1;
            seg_first[h + 1] = seg_first[h] + k;
            for (uint64_t j = 0; j < k; ++j) {
                item_hay.push_back((uint32_t)h);
                item_beg.push_back((uint32_t)(j * seg_len));
            }
        }
        n_items = seg_first[n];
    }
    std::vector<unsigned long long> item_count(n_items ? n_items : 1, 0);
    std::vector<uint4> item_first(n_items ? n_items : 1);
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
    P.text = text;
    P.text_lo = text + (n ? offs[0] : 0);
    P.text_end = text + (n ? offs[n] : 0);
    P.offs = offs;
    P.n_items = n_items;
    if (seg) {
        P.item_hay = item_hay.data();
        P.item_beg = item_beg.data();
        P.seg_len = seg_len;
        P.warm = img.max_pattern_len ? img.max_pattern_len - 1 : 0;
    }
    P.ctrl = &ctrl;
    P.item_count = item_count.data();
    P.item_first = item_first.data();
    const uint8_t* lo = P.text_lo;
    const uint8_t* hi = P.text_end;
    // k_scan_rk: leading wide records from a "shared memory" copy
    const uint32_t hot_w = which == 0 ? std::min<uint32_t>(hot_n, img.n_slots) : 0;
    P.hot_n = hot_w;
    std::vector<uint32_t> hot(img.rec.begin(), img.rec.begin() + (size_t)hot_w * 4);
    hot.resize(hot.size() + 4);
    RecView V{P.rec, reinterpret_cast<const uint4*>(hot.data()), hot_w, img.root_table.data()};
    // StdMachine3: the leading compact records from a copy whose remainder is poison, so that a wrong prefix compare
    // cannot go unnoticed
    const uint32_t entries = which == 3 ? std::min<uint32_t>(hot_n, img.hot_slots) : 0;
    std::vector<uint32_t> tab(img.crec.size() ? img.crec.size() : 4, 0xdeadbeefu);
    if (entries) memcpy(tab.data(), img.crec.data(), (size_t)entries * 16);
    StdEnv Ev{};
    if (v1)
        Ev = StdEnv{reinterpret_cast<const uint4*>(img.crec.data()), reinterpret_cast<const uint4*>(tab.data()), 0u, entries,
                    img.opos_tab.data(), P.text_end, P.text_lo, img.root_base, P.root_opos ? CF_OUT : 0u, nullptr, 0, 0, P.mapper,
                    P.mapper_len, reinterpret_cast<const uint4*>(img.crec.data())[D_ROOT]};
    if (rk == RK_COUNT)
        run_rk<RK_COUNT>(P, V, Ev, lo, hi, charwise != 0, which, mmode);
    else
        run_rk<RK_FIRST>(P, V, Ev, lo, hi, charwise != 0, which, mmode);
    uint64_t tot = 0;  // k_count_hay / k_first_hay
    for (uint64_t h = 0; h < n; ++h) {
        const uint64_t a = seg ? seg_first[h] : h, b = seg ? seg_first[h + 1] : h + 1;
        if (rk == RK_COUNT) {
            uint64_t v = 0;
            for (uint64_t i = a; i < b; ++i) v += item_count[i];
            counts[h] = v;
            tot += v;
        } else {
            uint4 r = item_first[a];
            for (uint64_t i = a + 1; i < b && !r.w; ++i) r = item_first[i];
            first[h * 3 + 0] = r.x, first[h * 3 + 1] = r.y, first[h * 3 + 2] = r.z;
            found[h] = r.w ? 1 : 0;
            tot += r.w ? 1 : 0;
        }
    }
    if (total) *total = tot;
    return DACH_OK;
}

// the device image's output records {value, length, parent, chain} (dev_image.cpp): up to cap records, returns their number
extern "C" long long emu_image_outputs(const uint8_t* wire, size_t wire_len, int charwise, uint32_t* out, size_t cap) {
    dach_pma* pma = nullptr;
    size_t used = 0;
    if (wire_read(wire, wire_len, charwise != 0, &pma, &used)) return -1;
    HostImage img;
    const int rc = build_image(pma, &img);
    delete pma;
    if (rc) return -1;
    const size_t k = img.outputs.size() / 4;
    if (out) memcpy(out, img.outputs.data(), std::min(k, cap) * 16);
    return (long long)k;
}

// HostImage::segmentable of a serialized bytewise automaton: 1 / 0, -1 for a refused one
extern "C" int emu_image_segmentable(const uint8_t* wire, size_t wire_len) {
    dach_pma* pma = nullptr;
    size_t used = 0;
    if (wire_read(wire, wire_len, false, &pma, &used)) return -1;
    HostImage img;
    const int rc = build_image(pma, &img);
    delete pma;
    return rc ? -1 : (img.segmentable ? 1 : 0);
}
