// CPU emulation of counts, first matches and per-pattern histograms of stream chunks (TEST INFRASTRUCTURE ONLY).
//
// Compiles daachorse_b200/csrc/scan_lane.cuh -- the exact lane logic the CUDA kernels run -- with g++ (-DDACH_EMU)
// and drives it the way enqueue_rk() in dev_scan.cu does for dach_dev_count_stream / dach_dev_first_stream /
// dach_dev_hist_stream: one item per chunk (no segments), the state read and written through ScanParams::state_io,
// items -> lanes of warps of CTAs (the warp collectives written out as loops over 32 lane states), the machine's
// step() with SinkOps' drain() / begin_item(); then k_count_hay / k_first_stream / k_hist_heads + k_hist_fold.
// It is never loaded by the product.
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

static uint32_t g_want_hot_slots = 65536;  // size of the hot region build_image() lays out
extern "C" void emu_stream_rk_set_hot_slots(uint32_t n) { g_want_hot_slots = n; }

// k_scan_machine_rk: the service phase / lock-step loop of scan_machine() in dev_scan.cu; n_ctas CTAs of n_warps warps
// interleaved, each CTA with its own shared-memory HIST counters (flushed when the CTA ends)
template <class M, class LANE, int MODE, int RK>
static void run_machine(const ScanParams& P, const StdEnv& Ev0, int n_ctas, int n_warps) {
    using OPS = SinkOps<M, MODE, RK>;
    using SINK = typename OPS::Sink;
    struct Warp {
        LANE L[32];
        SINK E[32];
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
            if constexpr (RK == RK_HIST) {
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
    const uint8_t* lo = P.text_lo;
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
    if constexpr (RK == RK_HIST)
        for (auto& c : cta_cnt)
            for (uint32_t i = 0; i < P.hist_smem; ++i) P.slot_hist[i] += c[i];
}

// launch_rk<RK_COUNT / RK_HIST> and launch_first_stream in dev_scan.cu, for the two stepper iterators
template <int RK>
static void run_rk(const ScanParams& P, const StdEnv& Ev, bool cw, int mode) {
    const int nc = 2, nw = 2;
    if (cw) {
        if (mode == M_FIND) run_machine<CwMachine<M_FIND>, LaneCw, M_FIND, RK>(P, Ev, nc, nw);
        else run_machine<CwMachine<M_OVERLAPPING>, LaneCw, M_OVERLAPPING, RK>(P, Ev, nc, nw);
    } else {
        if (mode == M_FIND) run_machine<StdMachine3<M_FIND>, Lane3, M_FIND, RK>(P, Ev, nc, nw);
        else run_machine<StdMachine3<M_OVERLAPPING>, Lane3, M_OVERLAPPING, RK>(P, Ev, nc, nw);
    }
}

// dach_dev_count_stream (rk = 1: counts, n x u64), dach_dev_first_stream (rk = 2: first, n x 3 u32, and found, n x u8;
// positions plus pos[i], or chunk-relative if pos is nullptr) and dach_dev_hist_stream (rk = 3: added into hist by key,
// 0 = output record, 1 = value).  Haystack i is the next chunk of stream i, resumed in state_io[i] (crate state ids)
// and leaving its state there.  hot_n: StdMachine3 records served from the "shared memory" copy; kernel: the option
// (1, 2 and 4 run 3, as on the device; 0 is refused); hist_smem: the option of that name.  *total: the matches (COUNT,
// HIST) or the chunks with a match (FIRST).
extern "C" int emu_rk_stream_wire(const uint8_t* wire, size_t wire_len, int charwise, int mode, int rk, int key, const uint8_t* text,
                                  const uint64_t* offs, uint64_t n, uint32_t* state_io, const uint32_t* pos, uint32_t hot_n, int kernel,
                                  int64_t hist_smem, uint64_t* counts, uint32_t* first, uint8_t* found, uint64_t* hist, uint64_t n_hist,
                                  uint64_t* total) {
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
    const uint32_t n_out = (uint32_t)(img.outputs.size() / 4);
    if (rk == RK_HIST) {  // check_hist
        uint32_t max_value = 0;
        for (uint32_t i = 0; i < n_out; ++i) max_value = std::max(max_value, img.outputs[(size_t)i * 4]);
        if (key != 0 && key != 1) return DACH_INVALID_ARGUMENT;
        if (key == 0 ? n_hist < n_out : (n_out && n_hist <= max_value)) return DACH_INVALID_ARGUMENT;
    }
    if (mode != M_FIND && mode != M_OVERLAPPING) return DACH_INVALID_ARGUMENT;  // the crate's two steppers
    if (lm) return DACH_MATCH_KIND_MISMATCH;
    if (rk != RK_COUNT && rk != RK_FIRST && rk != RK_HIST) return DACH_INVALID_ARGUMENT;
    if (total) *total = 0;
    if (n == 0) return DACH_OK;
    // the refusal of enqueue_rk / enqueue_scan: stream chunks need a Standard lane machine
    const bool v1 = kernel >= 1 && !img.crec.empty() && !(mode == M_FIND && img.root_opos != 0);
    const bool cw_machine = v1 && charwise;
    const bool std3 = v1 && !charwise && img.root_base != 0;
    if (!std3 && !cw_machine) return DACH_INVALID_ARGUMENT;
    const uint32_t n_cslots = (uint32_t)img.opos_tab.size();
    std::vector<unsigned long long> item_count(n, 0), slot_hist(n_cslots + 1, 0), rec_hist(n_out + 1, 0);
    std::vector<uint4> item_first(n);
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
    P.n_items = n;
    P.state_io = state_io;
    if (img.hot_slots) {  // the compact image is renumbered: state ids are translated at the boundary
        P.id_in = img.new_of_old.data();
        P.id_out = img.old_of_new.data();
    }
    P.ctrl = &ctrl;
    P.item_count = item_count.data();
    P.item_first = item_first.data();
    P.slot_hist = slot_hist.data();
    P.rec_hist = rec_hist.data();
    P.hist_smem = rk == RK_HIST ? (uint32_t)std::min<int64_t>(std::max<int64_t>(hist_smem, 0), std::min<int64_t>(n_cslots, 16384)) : 0;
    // StdMachine3: the leading compact records from a copy whose remainder is poison, so that a wrong prefix compare
    // cannot go unnoticed
    const uint32_t entries = std3 ? std::min<uint32_t>(hot_n, img.hot_slots) : 0;
    std::vector<uint32_t> tab(img.crec.size() ? img.crec.size() : 4, 0xdeadbeefu);
    if (entries) memcpy(tab.data(), img.crec.data(), (size_t)entries * 16);
    const StdEnv Ev{reinterpret_cast<const uint4*>(img.crec.data()), reinterpret_cast<const uint4*>(tab.data()), 0u, entries,
                    img.opos_tab.data(), P.text_end, P.text_lo, img.root_base, P.root_opos ? CF_OUT : 0u, nullptr, 0, 0, P.mapper,
                    P.mapper_len, reinterpret_cast<const uint4*>(img.crec.data())[D_ROOT]};
    const bool cw = charwise != 0;
    if (rk == RK_COUNT)
        run_rk<RK_COUNT>(P, Ev, cw, mode);
    else if (rk == RK_FIRST)
        run_rk<RK_FIRST_STREAM>(P, Ev, cw, mode);
    else
        run_rk<RK_HIST>(P, Ev, cw, mode);
    uint64_t tot = 0;
    if (rk == RK_COUNT) {  // k_count_hay, one item per chunk
        for (uint64_t h = 0; h < n; ++h) counts[h] = item_count[h], tot += item_count[h];
    } else if (rk == RK_FIRST) {  // k_first_stream
        for (uint64_t h = 0; h < n; ++h) {
            const uint4 r = item_first[h];
            const uint32_t b = (r.w && pos) ? pos[h] : 0u;
            first[h * 3 + 0] = r.x + b, first[h * 3 + 1] = r.y + b, first[h * 3 + 2] = r.z;
            found[h] = r.w ? 1 : 0;
            tot += r.w ? 1 : 0;
        }
    } else {
        for (uint32_t s = 0; s < n_cslots; ++s)  // k_hist_heads
            if (slot_hist[s] && img.opos_tab[s]) rec_hist[img.opos_tab[s] - 1] += slot_hist[s];
        const bool chain = mode == M_OVERLAPPING;  // k_hist_fold<true>: an event reports the head's whole list
        for (uint32_t i = 0; i < n_out; ++i) {
            const unsigned long long v = rec_hist[i];
            for (uint32_t j = v ? i + 1 : 0; j;) {
                const uint32_t* o = img.outputs.data() + (size_t)(j - 1) * 4;
                hist[key ? o[0] : j - 1] += v;
                tot += v;
                j = chain ? o[2] : 0;
            }
        }
    }
    if (total) *total = tot;
    return DACH_OK;
}
