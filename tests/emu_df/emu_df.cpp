// CPU emulation of per-pattern document frequencies (TEST INFRASTRUCTURE ONLY).
//
// Compiles daachorse_b200/csrc/scan_lane.cuh -- the exact lane logic the CUDA kernels run -- with g++ (-DDACH_EMU)
// and drives it the way df_windows() / enqueue_rk() in dev_scan.cu do for RK_DF: items -> lanes of warps of CTAs (the
// warp collectives written out as loops over 32 lane states), the machine's step() with SinkOps' drain() /
// begin_item() and a DfSink whose inserts go into the same open-addressing sets (df_insert); or the lane-per-haystack
// loops with a DfSink; then k_df_expand, k_df_add and k_df_clear restated, window by window, with the split of a
// window that overflows.  It is never loaded by the product.
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

// k_scan_rk<..., RK_DF>: one lane per haystack, the reference-shaped loops
template <bool CW, int MODE>
static void run_items(const ScanParams& P, const RecView& V, const uint8_t* lo, const uint8_t* hi) {
    for (uint64_t item = 0; item < P.n_items; ++item) {
        TextWin T;
        T.emu_lo = lo;
        T.emu_hi = hi;
        DfSink E;
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

// k_scan_machine_rk<..., RK_DF>: the service phase / lock-step loop of scan_machine() in dev_scan.cu; n_warps warps
// interleaved, so lanes of different warps insert into the sets in turn
template <class M, class LANE, int MODE>
static void run_machine(const ScanParams& P, const StdEnv& Ev0, const uint8_t* lo, int n_warps) {
    using OPS = SinkOps<M, MODE, RK_DF>;
    struct Warp {
        LANE L[32];
        DfSink E[32];
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

// launch_rk<RK_DF> in dev_scan.cu: which = 3 StdMachine3, 1 LmMachine / CwMachine, 0 lane per haystack
static void run_scan(const ScanParams& P, const RecView& V, const StdEnv& Ev, const uint8_t* lo, const uint8_t* hi, bool cw, int which,
                     int mode) {
    const int nw = 4;
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

struct Sets {  // the handle's two pair sets (dach_dev::df_tab / df_list / df_n)
    std::vector<unsigned long long> tab[2];
    std::vector<uint32_t> list[2];
    unsigned int n[2] = {0, 0};
    uint32_t mask = 0, limit = 0;
    DfSet set(int i) { return DfSet{tab[i].data(), list[i].data(), &n[i], mask, limit}; }
};

// dach_dev_df_batch / dach_df_batch_host: adds into df[0 .. n_df) by key (0 = output record, 1 = value); *total = the
// (haystack, key) pairs added.  hot_n, kernel, seg_len as in emu_hist_batch_wire; df_pairs: the option of that name
// (raised to max(compact slots, output records) as df_prepare does).  split = 1: a window that overflows is scanned
// again as two halves (df_windows); split = 0: the whole batch is one window, and one that overflows adds nothing and
// returns DACH_OUTPUT_OVERFLOW -- what the device does with such a window before it splits it.
// out[0] = windows, out[1] = re-scans, out[2] = the kernel that ran (3, 1, 0) + 8 if parent chains were expanded,
// out[3] = the pair-set entries left taken after the call (0: k_df_clear emptied both sets), out[4] / out[5] = the most
// (haystack, slot) / (haystack, key) pairs one window put into its sets (tools/lane_stats.py --pairs).
extern "C" int emu_df_batch_wire(const uint8_t* wire, size_t wire_len, int charwise, int mode, int key, const uint8_t* text,
                                 const uint64_t* offs, uint64_t n, uint32_t hot_n, int kernel, uint32_t seg_len, int64_t df_pairs, int split,
                                 uint64_t* df, uint64_t n_df, uint64_t* total, uint64_t* out) {
    dach_pma* pma = nullptr;
    size_t used = 0;
    int rc = wire_read(wire, wire_len, charwise != 0, &pma, &used);
    if (rc) return rc;
    HostImage img;
    rc = build_image(pma, &img);
    const bool lm = is_leftmost(pma->match_kind);
    delete pma;
    if (rc) return rc;
    // check_hist, then check_mode
    const uint32_t n_out = (uint32_t)(img.outputs.size() / 4);
    uint32_t max_value = 0;
    for (uint32_t i = 0; i < n_out; ++i) max_value = std::max(max_value, img.outputs[(size_t)i * 4]);
    if (key != 0 && key != 1) return DACH_INVALID_ARGUMENT;
    if (key == 0 ? n_df < n_out : (n_out && n_df <= max_value)) return DACH_INVALID_ARGUMENT;
    if (mode < M_FIND || mode > M_LEFTMOST) return DACH_INVALID_ARGUMENT;
    if ((mode == M_LEFTMOST) != lm) return DACH_MATCH_KIND_MISMATCH;
    if (total) *total = 0;
    for (int i = 0; i < 6; ++i) out[i] = 0;
    if (n == 0) return DACH_OK;
    // kernel choice as enqueue_rk
    const ScanPlan plan = plan_scan({.opt_kernel = kernel, .compact = !img.crec.empty(), .charwise = charwise != 0,
                                     .root_opos = img.root_opos != 0, .root_base = img.root_base != 0,
                                     .segmentable = img.segmentable, .matches = false, .mode = mode});
    const bool machine = plan.lane_machine();
    const int which = plan.machine == Machine::Std3 ? 3 : machine ? 1 : 0;
    const bool seg = plan.seg && seg_len > 0;
    const bool chain = machine && mode == M_OVERLAPPING;
    const uint32_t n_cslots = (uint32_t)img.opos_tab.size();
    // df_prepare
    Sets S;
    const uint64_t limit = std::min<uint64_t>(std::max<uint64_t>({(uint64_t)std::max<int64_t>(df_pairs, 1), n_cslots, n_out}), 1ull << 30);
    uint64_t cap = 2;
    while (cap < 2 * limit) cap <<= 1;
    S.mask = (uint32_t)(cap - 1);
    S.limit = (uint32_t)limit;
    for (int i = 0; i < 2; ++i) {
        S.tab[i].assign(cap, DF_EMPTY);
        S.list[i].assign(cap, 0);
    }
    std::vector<unsigned long long> acc(std::max<uint64_t>(n_df, 1), 0);
    // the image, as enqueue_rk's ScanParams and StdEnv
    const uint32_t hot_w = which == 0 ? std::min<uint32_t>(hot_n, img.n_slots) : 0;
    std::vector<uint32_t> hot(img.rec.begin(), img.rec.begin() + (size_t)hot_w * 4);
    hot.resize(hot.size() + 4);
    const uint32_t entries = which == 3 ? std::min<uint32_t>(hot_n, img.hot_slots) : 0;
    std::vector<uint32_t> tab(img.crec.size() ? img.crec.size() : 4, 0xdeadbeefu);
    if (entries) memcpy(tab.data(), img.crec.data(), (size_t)entries * 16);
    const uint8_t* lo = text + offs[0];
    const uint8_t* hi = text + offs[n];

    // one window: haystacks [a, b); returns whether it overflowed (and then added nothing)
    auto window = [&](uint64_t a, uint64_t b, uint64_t* added) -> bool {
        const uint64_t* wo = offs + a;
        const uint64_t wn = b - a;
        std::vector<uint32_t> item_hay, item_beg;
        uint64_t n_items = wn;
        if (seg) {  // k_seg_count / k_seg_fill
            n_items = 0;
            for (uint64_t h = 0; h < wn; ++h) {
                uint64_t k = (wo[h + 1] - wo[h] + seg_len - 1) / seg_len;
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
        P.text_lo = lo;
        P.text_end = hi;
        P.offs = wo;
        P.n_items = n_items;
        if (seg) {
            P.item_hay = item_hay.data();
            P.item_beg = item_beg.data();
            P.seg_len = seg_len;
            P.warm = img.max_pattern_len ? img.max_pattern_len - 1 : 0;
        }
        P.ctrl = &ctrl;
        P.df_key_value = key == 1;
        P.df_slots = S.set(0);
        P.df_keys = S.set(1);
        P.hot_n = hot_w;
        RecView V{P.rec, reinterpret_cast<const uint4*>(hot.data()), hot_w, img.root_table.data()};
        StdEnv Ev{};
        if (machine)
            Ev = StdEnv{reinterpret_cast<const uint4*>(img.crec.data()), reinterpret_cast<const uint4*>(tab.data()), 0u, entries,
                        img.opos_tab.data(), P.text_end, P.text_lo, img.root_base, P.root_opos ? CF_OUT : 0u, nullptr, 0, 0, P.mapper,
                        P.mapper_len, reinterpret_cast<const uint4*>(img.crec.data())[D_ROOT]};
        run_scan(P, V, Ev, lo, hi, charwise != 0, which, mode);
        // k_df_expand
        if (machine && !ctrl.overflow) {
            for (unsigned int i = 0; i < S.n[0]; ++i) {
                const unsigned long long pair = S.tab[0][S.list[0][i]];
                const unsigned long long hay = pair & 0xffffffff00000000ull;
                bool full = false;
                for (uint32_t j = img.opos_tab[(uint32_t)pair]; j && !full;) {
                    const uint32_t* o = img.outputs.data() + (size_t)(j - 1) * 4;
                    full = df_insert(P.df_keys, hay | (key ? o[0] : j - 1), &ctrl) == DF_FULL;
                    j = chain ? o[2] : 0;
                }
            }
        }
        // k_df_add
        if (!ctrl.overflow) {
            for (unsigned int i = 0; i < S.n[1]; ++i) acc[(uint32_t)S.tab[1][S.list[1][i]]] += 1;
            *added += S.n[1];
        }
        out[4] = std::max<uint64_t>(out[4], S.n[0]);
        out[5] = std::max<uint64_t>(out[5], S.n[1]);
        // k_df_clear, then the counters
        for (int s = 0; s < 2; ++s)
            for (unsigned int i = 0; i < S.n[s]; ++i) S.tab[s][S.list[s][i]] = DF_EMPTY;
        S.n[0] = S.n[1] = 0;
        return ctrl.overflow != 0;
    };

    uint64_t sum = 0, win = ~0ull;
    for (uint64_t a = 0; a < n;) {
        const uint64_t b = n - a <= win ? n : a + win;
        if (window(a, b, &sum)) {
            ++out[1];
            if (!split) return DACH_OUTPUT_OVERFLOW;
            if (b - a == 1) return DACH_CUDA_ERROR;
            win = (b - a + 1) / 2;
            continue;
        }
        ++out[0];
        a = b;
    }
    for (int s = 0; s < 2; ++s)
        for (unsigned long long v : S.tab[s]) out[3] += v != DF_EMPTY;
    for (uint64_t i = 0; i < n_df; ++i) df[i] += acc[i];
    if (total) *total = sum;
    out[2] = which + (chain ? 8 : 0);
    return DACH_OK;
}
