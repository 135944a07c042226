// CPU emulation of per-pattern histograms (TEST INFRASTRUCTURE ONLY): dach_dev_hist_batch, with each CTA's
// shared-memory counters and k_hist_heads / k_hist_fold, and the share of the lane machines' events that fall on the
// hottest compact slots.  The drivers are emu_driver.h's.
#include <functional>

#include "emu_driver.h"

using namespace emu;

// dach_dev_hist_batch: adds into hist[0 .. n_hist) by key (0 = output record, 1 = value); *total = the matches added.
// hot_n: StdMachine3 records served from the "shared memory" copy (kernel 0: leading wide records), kernel: the option
// (1, 2 and 4 run 3, as on the device), seg_len > 0: segments of that length where the device may cut, hist_smem: the
// option of that name.  *which_out: the kernel that ran (3, 1, 0) and whether the parent chains were walked (+ 8).
extern "C" int emu_hist_batch_wire(const uint8_t* wire, size_t wire_len, int charwise, int mode, int key, const uint8_t* text,
                                   const uint64_t* offs, uint64_t n, uint32_t hot_n, int kernel, uint32_t seg_len, int64_t hist_smem,
                                   uint64_t* hist, uint64_t n_hist, uint64_t* total, int* which_out) {
    HostImage img;
    bool lm = false;
    const int rc = load(wire, wire_len, charwise != 0, &img, &lm);
    if (rc) return rc;
    if (!check_hist(img, key, n_hist)) return DACH_INVALID_ARGUMENT;
    if (mode < M_FIND || mode > M_LEFTMOST) return DACH_INVALID_ARGUMENT;
    if ((mode == M_LEFTMOST) != lm) return DACH_MATCH_KIND_MISMATCH;
    if (total) *total = 0;
    if (n == 0) return DACH_OK;
    ScanInputs in = plan_inputs(img, charwise != 0, mode);
    in.opt_kernel = kernel;
    in.matches = false;
    const ScanPlan plan = plan_scan(in);
    const bool machine = plan.lane_machine();
    const Segments S = seg_table(offs, n, plan.seg ? seg_len : 0, 0);
    const uint32_t n_cslots = (uint32_t)img.opos_tab.size();
    std::vector<unsigned long long> slot_hist(n_cslots + 1, 0), rec_hist(img.outputs.size() / 4 + 1, 0);
    ScanCtrl ctrl;
    memset(&ctrl, 0, sizeof(ctrl));
    ScanParams P = scan_params(img, text, offs, n, S, &ctrl);
    P.slot_hist = slot_hist.data();
    P.rec_hist = rec_hist.data();
    P.hist_smem = machine ? (uint32_t)std::min<int64_t>(std::max<int64_t>(hist_smem, 0), std::min<int64_t>(n_cslots, 16384)) : 0;
    const Smem sm(img, plan, hot_n, P.text_lo, P.text_end);
    run_rk_modes<RK_HIST>(plan, charwise != 0, P, sm, 2, 2);
    const uint64_t tot = hist_fold(img, machine, mode, slot_hist, rec_hist, key, hist);
    if (total) *total = tot;
    if (which_out) *which_out = (plan.machine == Machine::Std3 ? 3 : machine ? 1 : 0) + (machine && mode == M_OVERLAPPING ? 8 : 0);
    return DACH_OK;
}

// shares of the lane machines' events (StdMachine3, LmMachine or CwMachine, by the automaton and mode) on compact slots:
// out[0] = all events, out[1 + i] = events on the top[i] most frequent slots, out[1 + n_top + i] = events on compact
// slots < top[i] (what hist_smem = top[i] counts in shared memory).  -1: no lane machine runs this automaton and mode.
extern "C" int emu_hist_event_shares(const uint8_t* wire, size_t wire_len, int charwise, int mode, const uint8_t* text,
                                     const uint64_t* offs, uint64_t n, const uint32_t* top, int n_top, unsigned long long* out) {
    HostImage img;
    bool lm = false;
    if (load(wire, wire_len, charwise != 0, &img, &lm) || (mode == M_LEFTMOST) != lm) return -1;
    ScanInputs in = plan_inputs(img, charwise != 0, mode);
    in.matches = false;
    const ScanPlan plan = plan_scan(in);
    if (!plan.lane_machine()) return -1;
    const uint32_t n_cslots = (uint32_t)img.opos_tab.size();
    std::vector<unsigned long long> slot_hist(n_cslots, 0);
    const Segments S = seg_table(offs, n, 0, 0);
    ScanCtrl ctrl;
    memset(&ctrl, 0, sizeof(ctrl));
    ScanParams P = scan_params(img, text, offs, n, S, &ctrl);
    P.slot_hist = slot_hist.data();  // hist_smem = 0: every event counts here
    const Smem sm(img, plan, 0, P.text_lo, P.text_end);
    run_rk_modes<RK_HIST>(plan, charwise != 0, P, sm, 2, 2);
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
