// CPU emulation of per-pattern histograms (TEST INFRASTRUCTURE ONLY).
//
// Compiles daachorse_b200/csrc/scan_lane.cuh -- the exact lane logic the CUDA kernels run -- with g++ (-DDACH_EMU)
// and drives it the way enqueue_rk() in dev_scan.cu does for RK_HIST: items -> lanes of warps of CTAs (the warp
// collectives written out as loops over 32 lane states), the machine's step() with SinkOps' drain() / begin_item()
// and a HistSink whose leading slots count in per-CTA counters flushed when the CTA ends; or the lane-per-haystack
// loops with a HistSink; then k_hist_heads / k_hist_fold.  It is never loaded by the product.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
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

static uint32_t g_want_hot_slots = 65536;  // size of the hot region build_image() lays out
extern "C" void emu_hist_set_hot_slots(uint32_t n) { g_want_hot_slots = n; }

// k_scan_rk<..., RK_HIST>: one lane per haystack, the reference-shaped loops
template <bool CW, int MODE>
static void run_items(const ScanParams& P, const RecView& V, const uint8_t* lo, const uint8_t* hi) {
    for (uint64_t item = 0; item < P.n_items; ++item) {
        TextWin T;
        T.emu_lo = lo;
        T.emu_hi = hi;
        HistSink E;
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

// k_scan_machine_rk<..., RK_HIST>: the service phase / lock-step loop of scan_machine() in dev_scan.cu; n_ctas CTAs of
// n_warps warps interleaved, each CTA with its own shared-memory counters
template <class M, class LANE, int MODE>
static void run_machine(const ScanParams& P, const StdEnv& Ev0, const uint8_t* lo, int n_ctas, int n_warps) {
    using OPS = SinkOps<M, MODE, RK_HIST>;
    struct Warp {
        LANE L[32];
        HistSink E[32];
        StdEnv Ev[32];
        std::vector<QEntry> queue;
        bool exhausted[32];
        bool finished;
    };
    std::vector<std::vector<unsigned int>> cta_cnt(n_ctas, std::vector<unsigned int>(P.hist_smem + 1, 0));
    std::vector<Warp> warps(n_ctas * n_warps);
    for (size_t wi = 0; wi < warps.size(); ++wi) {
        Warp& w = warps[wi];
        w.queue.assign((size_t)LANE_Q * 32, QEntry{0, 0});
        for (int l = 0; l < 32; ++l) {
            w.L[l].fl = M::IDLE;
            w.L[l].qn = 0;
            w.E[l].begin(0);
            w.E[l].s_cnt = cta_cnt[wi / n_warps].data();
            w.E[l].k = P.hist_smem;
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
    for (auto& c : cta_cnt)  // the end of every CTA: its counters go to global memory once
        for (uint32_t i = 0; i < P.hist_smem; ++i) P.slot_hist[i] += c[i];
}

// launch_rk<RK_HIST> in dev_scan.cu: which = 3 StdMachine3, 1 LmMachine / CwMachine, 0 lane per haystack
static void run_hist(const ScanParams& P, const RecView& V, const StdEnv& Ev, const uint8_t* lo, const uint8_t* hi, bool cw, int which,
                     int mode) {
    const int nc = 2, nw = 2;
    if (which == 3) {
        if (mode == M_FIND) run_machine<StdMachine3<M_FIND>, Lane3, M_FIND>(P, Ev, lo, nc, nw);
        if (mode == M_NO_SUFFIX) run_machine<StdMachine3<M_NO_SUFFIX>, Lane3, M_NO_SUFFIX>(P, Ev, lo, nc, nw);
        if (mode == M_OVERLAPPING) run_machine<StdMachine3<M_OVERLAPPING>, Lane3, M_OVERLAPPING>(P, Ev, lo, nc, nw);
    } else if (which == 1 && cw) {
        if (mode == M_FIND) run_machine<CwMachine<M_FIND>, LaneCw, M_FIND>(P, Ev, lo, nc, nw);
        if (mode == M_NO_SUFFIX) run_machine<CwMachine<M_NO_SUFFIX>, LaneCw, M_NO_SUFFIX>(P, Ev, lo, nc, nw);
        if (mode == M_OVERLAPPING) run_machine<CwMachine<M_OVERLAPPING>, LaneCw, M_OVERLAPPING>(P, Ev, lo, nc, nw);
        if (mode == M_LEFTMOST) run_machine<CwMachine<M_LEFTMOST>, LaneCw, M_LEFTMOST>(P, Ev, lo, nc, nw);
    } else if (which == 1) {
        run_machine<LmMachine, LaneLm, M_LEFTMOST>(P, Ev, lo, nc, nw);
    } else {
        switch ((cw ? 4 : 0) + mode) {
            case 0: run_items<false, M_FIND>(P, V, lo, hi); break;
            case 1: run_items<false, M_OVERLAPPING>(P, V, lo, hi); break;
            case 2: run_items<false, M_NO_SUFFIX>(P, V, lo, hi); break;
            case 3: run_items<false, M_LEFTMOST>(P, V, lo, hi); break;
            case 4: run_items<true, M_FIND>(P, V, lo, hi); break;
            case 5: run_items<true, M_OVERLAPPING>(P, V, lo, hi); break;
            case 6: run_items<true, M_NO_SUFFIX>(P, V, lo, hi); break;
            case 7: run_items<true, M_LEFTMOST>(P, V, lo, hi); break;
        }
    }
}

// dach_dev_hist_batch: adds into hist[0 .. n_hist) by key (0 = output record, 1 = value); *total = the matches added.
// hot_n: StdMachine3 records served from the "shared memory" copy (kernel 0: leading wide records), kernel: the option
// (1, 2 and 4 run 3, as on the device), seg_len > 0: segments of that length where the device may cut, hist_smem: the
// option of that name.  *which_out: the kernel that ran (3, 1, 0) and whether the parent chains were walked (+ 8).
extern "C" int emu_hist_batch_wire(const uint8_t* wire, size_t wire_len, int charwise, int mode, int key, const uint8_t* text,
                                   const uint64_t* offs, uint64_t n, uint32_t hot_n, int kernel, uint32_t seg_len, int64_t hist_smem,
                                   uint64_t* hist, uint64_t n_hist, uint64_t* total, int* which_out) {
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
    // check_hist, then check_mode
    const uint32_t n_out = (uint32_t)(img.outputs.size() / 4);
    uint32_t max_value = 0;
    for (uint32_t i = 0; i < n_out; ++i) max_value = std::max(max_value, img.outputs[(size_t)i * 4]);
    if (key != 0 && key != 1) return DACH_INVALID_ARGUMENT;
    if (key == 0 ? n_hist < n_out : (n_out && n_hist <= max_value)) return DACH_INVALID_ARGUMENT;
    if (mode < M_FIND || mode > M_LEFTMOST) return DACH_INVALID_ARGUMENT;
    if ((mode == M_LEFTMOST) != lm) return DACH_MATCH_KIND_MISMATCH;
    if (total) *total = 0;
    if (n == 0) return DACH_OK;
    // kernel choice and segments as enqueue_rk
    const ScanPlan plan = plan_scan({.opt_kernel = kernel, .compact = !img.crec.empty(), .charwise = charwise != 0,
                                     .root_opos = img.root_opos != 0, .root_base = img.root_base != 0,
                                     .segmentable = img.segmentable, .matches = false, .mode = mode});
    const bool machine = plan.lane_machine();
    const int which = plan.machine == Machine::Std3 ? 3 : machine ? 1 : 0;
    const bool seg = plan.seg && seg_len > 0;
    std::vector<uint32_t> item_hay, item_beg;
    uint64_t n_items = n;
    if (seg) {  // k_seg_count / k_seg_fill
        n_items = 0;
        for (uint64_t h = 0; h < n; ++h) {
            uint64_t k = (offs[h + 1] - offs[h] + seg_len - 1) / seg_len;
            if (k == 0) k = 1;
            for (uint64_t j = 0; j < k; ++j) {
                item_hay.push_back((uint32_t)h);
                item_beg.push_back((uint32_t)(j * seg_len));
            }
            n_items += k;
        }
    }
    const uint32_t n_cslots = (uint32_t)img.opos_tab.size();
    std::vector<unsigned long long> slot_hist(n_cslots + 1, 0), rec_hist(n_out + 1, 0);
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
    P.text_lo = text + offs[0];
    P.text_end = text + offs[n];
    P.offs = offs;
    P.n_items = n_items;
    if (seg) {
        P.item_hay = item_hay.data();
        P.item_beg = item_beg.data();
        P.seg_len = seg_len;
        P.warm = img.max_pattern_len ? img.max_pattern_len - 1 : 0;
    }
    P.ctrl = &ctrl;
    P.slot_hist = slot_hist.data();
    P.rec_hist = rec_hist.data();
    P.hist_smem = machine ? (uint32_t)std::min<int64_t>(std::max<int64_t>(hist_smem, 0), std::min<int64_t>(n_cslots, 16384)) : 0;
    const uint8_t* lo = P.text_lo;
    const uint8_t* hi = P.text_end;
    const uint32_t hot_w = which == 0 ? std::min<uint32_t>(hot_n, img.n_slots) : 0;
    P.hot_n = hot_w;
    std::vector<uint32_t> hot(img.rec.begin(), img.rec.begin() + (size_t)hot_w * 4);
    hot.resize(hot.size() + 4);
    RecView V{P.rec, reinterpret_cast<const uint4*>(hot.data()), hot_w, img.root_table.data()};
    const uint32_t entries = which == 3 ? std::min<uint32_t>(hot_n, img.hot_slots) : 0;
    std::vector<uint32_t> tab(img.crec.size() ? img.crec.size() : 4, 0xdeadbeefu);
    if (entries) memcpy(tab.data(), img.crec.data(), (size_t)entries * 16);
    StdEnv Ev{};
    if (machine)
        Ev = StdEnv{reinterpret_cast<const uint4*>(img.crec.data()), reinterpret_cast<const uint4*>(tab.data()), 0u, entries,
                    img.opos_tab.data(), P.text_end, P.text_lo, img.root_base, P.root_opos ? CF_OUT : 0u, nullptr, 0, 0, P.mapper,
                    P.mapper_len, reinterpret_cast<const uint4*>(img.crec.data())[D_ROOT]};
    run_hist(P, V, Ev, lo, hi, charwise != 0, which, mode);
    // k_hist_heads
    if (machine)
        for (uint32_t s = 0; s < n_cslots; ++s)
            if (slot_hist[s] && img.opos_tab[s]) rec_hist[img.opos_tab[s] - 1] += slot_hist[s];
    // k_hist_fold
    const bool chain = machine && mode == M_OVERLAPPING;
    uint64_t tot = 0;
    for (uint32_t i = 0; i < n_out; ++i) {
        const unsigned long long v = rec_hist[i];
        for (uint32_t j = v ? i + 1 : 0; j;) {
            const uint32_t* o = img.outputs.data() + (size_t)(j - 1) * 4;
            hist[key ? o[0] : j - 1] += v;
            tot += v;
            j = chain ? o[2] : 0;
        }
    }
    if (total) *total = tot;
    if (which_out) *which_out = which + (chain ? 8 : 0);
    return DACH_OK;
}

// shares of the lane machines' events (StdMachine3, LmMachine or CwMachine, by the automaton and mode) on compact slots:
// out[0] = all events, out[1 + i] = events on the top[i] most frequent slots, out[1 + n_top + i] = events on compact
// slots < top[i] (what hist_smem = top[i] counts in shared memory)
extern "C" int emu_hist_event_shares(const uint8_t* wire, size_t wire_len, int charwise, int mode, const uint8_t* text,
                                     const uint64_t* offs, uint64_t n, const uint32_t* top, int n_top, unsigned long long* out) {
    dach_pma* pma = nullptr;
    size_t used = 0;
    if (wire_read(wire, wire_len, charwise != 0, &pma, &used)) return -1;
    HostImage img;
    img.want_hot_slots = g_want_hot_slots;
    const int rc = build_image(pma, &img);
    const bool lm = is_leftmost(pma->match_kind);
    delete pma;
    if (rc || img.crec.empty() || (mode == M_LEFTMOST) != lm || (mode == M_FIND && img.root_opos)) return -1;
    const int which = (charwise || lm) ? 1 : 3;
    if (which == 3 && img.root_base == 0) return -1;
    const uint32_t n_cslots = (uint32_t)img.opos_tab.size();
    std::vector<unsigned long long> slot_hist(n_cslots, 0);
    ScanCtrl ctrl;
    memset(&ctrl, 0, sizeof(ctrl));
    ScanParams P;
    memset(&P, 0, sizeof(P));
    P.outputs = reinterpret_cast<const uint4*>(img.outputs.data());
    P.mapper = img.mapper.data();
    P.mapper_len = (uint32_t)img.mapper.size();
    P.n_slots = img.n_slots;
    P.root_opos = img.root_opos;
    P.text = text;
    P.text_lo = text + offs[0];
    P.text_end = text + offs[n];
    P.offs = offs;
    P.n_items = n;
    P.ctrl = &ctrl;
    P.slot_hist = slot_hist.data();
    std::vector<uint32_t> tab(img.crec.size(), 0xdeadbeefu);
    StdEnv Ev{reinterpret_cast<const uint4*>(img.crec.data()), reinterpret_cast<const uint4*>(tab.data()), 0u, 0u, img.opos_tab.data(),
              P.text_end, P.text_lo, img.root_base, P.root_opos ? CF_OUT : 0u, nullptr, 0, 0, P.mapper, P.mapper_len,
              reinterpret_cast<const uint4*>(img.crec.data())[D_ROOT]};
    RecView V{};
    run_hist(P, V, Ev, P.text_lo, P.text_end, charwise != 0, which, mode);
    std::vector<unsigned long long> sorted(slot_hist);
    std::sort(sorted.begin(), sorted.end(), std::greater<unsigned long long>());
    unsigned long long all = 0;
    for (auto v : slot_hist) all += v;
    out[0] = all;
    for (int t = 0; t < n_top; ++t) {
        unsigned long long a = 0, b = 0;
        for (uint32_t i = 0; i < std::min<uint32_t>(top[t], n_cslots); ++i) a += sorted[i], b += slot_hist[i];
        out[1 + t] = a;
        out[1 + n_top + t] = b;
    }
    return 0;
}
