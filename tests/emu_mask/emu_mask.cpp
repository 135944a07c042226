// CPU emulation of masked text (TEST INFRASTRUCTURE ONLY).
//
// Compiles daachorse_b200/csrc/scan_lane.cuh -- the exact lane logic the CUDA kernels run -- with g++ (-DDACH_EMU)
// and drives it the way enqueue_rk() in dev_scan.cu does for RK_MASK: k_mask_copy's copy of the text, then items ->
// lanes of warps of CTAs (the warp collectives written out as loops over 32 lane states), the machine's step() with
// SinkOps' drain() / begin_item() and a MaskSink; or the lane-per-haystack loops with a MaskSink.  It is never loaded
// by the product.
#include <algorithm>
#include <cstdint>
#include <cstdio>
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

// k_scan_rk<..., RK_MASK>: one lane per haystack, the reference-shaped loops (scan_items in dev_scan.cu)
template <bool CW, int MODE>
static void run_items(const ScanParams& P, const RecView& V, const uint8_t* lo, const uint8_t* hi) {
    for (uint64_t item = 0; item < P.n_items; ++item) {
        TextWin T;
        T.emu_lo = lo;
        T.emu_hi = hi;
        MaskSink E;
        const uint64_t o0 = P.offs[item], o1 = P.offs[item + 1];
        T.open(P.text + o0);
        E.begin((uint32_t)item);
        E.base = P.mask_out + o0;
        if (MODE == M_LEFTMOST)
            scan_leftmost<CW>(P, V, T, E, (uint32_t)(o1 - o0));
        else
            scan_standard<CW, MODE>(P, V, T, E, (uint32_t)(o1 - o0));
        E.finish(P);
    }
}

// k_scan_machine_rk<..., RK_MASK>: the service phase / lock-step loop of scan_machine() in dev_scan.cu, n_warps warps
// interleaved
template <class M, class LANE, int MODE>
static void run_machine(const ScanParams& P, const StdEnv& Ev0, const uint8_t* lo, int n_warps) {
    using OPS = SinkOps<M, MODE, RK_MASK>;
    struct Warp {
        LANE L[32];
        MaskSink E[32];
        StdEnv Ev[32];
        std::vector<QEntry> queue;
        bool exhausted[32];
        bool finished;
    };
    std::vector<Warp> warps(n_warps);
    for (Warp& w : warps) {
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

// launch_rk<RK_MASK> in dev_scan.cu: which = 3 StdMachine3, 1 LmMachine / CwMachine, 0 lane per haystack
static void run_mask(const ScanParams& P, const RecView& V, const StdEnv& Ev, const uint8_t* lo, const uint8_t* hi, bool cw, int which,
                     int mode) {
    const int nw = 3;
    if (which == 3) {
        if (mode == M_FIND) run_machine<StdMachine3<M_FIND>, Lane3, M_FIND>(P, Ev, lo, nw);
        if (mode == M_NO_SUFFIX) run_machine<StdMachine3<M_NO_SUFFIX>, Lane3, M_NO_SUFFIX>(P, Ev, lo, nw);
        if (mode == M_OVERLAPPING) run_machine<StdMachine3<M_OVERLAPPING>, Lane3, M_OVERLAPPING>(P, Ev, lo, nw);
    } else if (which == 1 && cw) {
        if (mode == M_FIND) run_machine<CwMachine<M_FIND>, LaneCw, M_FIND>(P, Ev, lo, nw);
        if (mode == M_NO_SUFFIX) run_machine<CwMachine<M_NO_SUFFIX>, LaneCw, M_NO_SUFFIX>(P, Ev, lo, nw);
        if (mode == M_OVERLAPPING) run_machine<CwMachine<M_OVERLAPPING>, LaneCw, M_OVERLAPPING>(P, Ev, lo, nw);
        if (mode == M_LEFTMOST) run_machine<CwMachine<M_LEFTMOST>, LaneCw, M_LEFTMOST>(P, Ev, lo, nw);
    } else if (which == 1) {
        run_machine<LmMachine, LaneLm, M_LEFTMOST>(P, Ev, lo, nw);
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

// dach_dev_mask_batch: out[0, text_bytes) = text, then `fill` over every match.  hot_n: StdMachine3 records served from
// the "shared memory" copy (kernel 0: leading wide records), kernel: the option (1, 2 and 4 run 3, as on the device),
// seg_len > 0: segments of that length where the device may cut.  *which_out: the kernel that ran (3, 1, 0) and whether
// segments were cut (+ 8).
extern "C" int emu_mask_batch_wire(const uint8_t* wire, size_t wire_len, int charwise, int mode, const uint8_t* text, const uint64_t* offs,
                                   uint64_t n, uint64_t text_bytes, uint8_t fill, uint32_t hot_n, int kernel, uint32_t seg_len, uint8_t* out,
                                   int* which_out) {
    dach_pma* pma = nullptr;
    size_t used = 0;
    int rc = wire_read(wire, wire_len, charwise != 0, &pma, &used);
    if (rc) return rc;
    HostImage img;
    rc = build_image(pma, &img);
    const bool lm = is_leftmost(pma->match_kind);
    delete pma;
    if (rc) return rc;
    if (charwise && fill >= 0x80) return DACH_INVALID_ARGUMENT;
    if (mode < M_FIND || mode > M_LEFTMOST) return DACH_INVALID_ARGUMENT;
    if ((mode == M_LEFTMOST) != lm) return DACH_MATCH_KIND_MISMATCH;
    for (uint64_t h = 0; h < n; ++h)  // k_check_offsets: a refused call writes nothing
        if (offs[h + 1] < offs[h] || offs[h + 1] - offs[h] > 0xffffffffull || offs[h + 1] > text_bytes) return DACH_INVALID_ARGUMENT;
    if (text_bytes) memcpy(out, text, text_bytes);  // k_mask_copy
    if (which_out) *which_out = -1;
    if (n == 0) return DACH_OK;
    // kernel choice and segments as enqueue_rk
    const bool v1 = kernel >= 1 && !img.crec.empty() && !(mode == M_FIND && img.root_opos != 0);
    const bool cw_machine = v1 && charwise;
    const bool lm_machine = v1 && !charwise && mode == M_LEFTMOST;
    const bool std3 = v1 && !charwise && mode != M_LEFTMOST && img.root_base != 0;
    const bool machine = cw_machine || lm_machine || std3;
    const int which = std3 ? 3 : machine ? 1 : 0;
    const bool seg = std3 && seg_len > 0 && (mode == M_OVERLAPPING || mode == M_NO_SUFFIX) && img.segmentable;
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
    ScanCtrl ctrl;
    memset(&ctrl, 0, sizeof(ctrl));
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
    P.mask_out = out;
    P.mask_fill = fill;
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
    if (v1)
        Ev = StdEnv{reinterpret_cast<const uint4*>(img.crec.data()), reinterpret_cast<const uint4*>(tab.data()), 0u, entries,
                    img.opos_tab.data(), P.text_end, P.text_lo, img.root_base, P.root_opos ? CF_OUT : 0u, nullptr, 0, 0, P.mapper,
                    P.mapper_len, reinterpret_cast<const uint4*>(img.crec.data())[D_ROOT]};
    run_mask(P, V, Ev, lo, hi, charwise != 0, which, mode);
    if (which_out) *which_out = which + (seg ? 8 : 0);
    return DACH_OK;
}
