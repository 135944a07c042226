// CPU emulation of counts and first matches (TEST INFRASTRUCTURE ONLY): dach_dev_count_batch / dach_dev_first_batch,
// and counts, first matches and per-pattern histograms of stream chunks (dach_dev_count_stream / dach_dev_first_stream /
// dach_dev_hist_stream), each with the per-haystack fold of its results.  The drivers are emu_driver.h's.
#include "emu_driver.h"

using namespace emu;

// dach_dev_count_batch (rk = RK_COUNT: counts, n x u64) / dach_dev_first_batch (rk = RK_FIRST: first, n x 3 u32, and
// found, n x u8).  *total = the sum of the counts / the haystacks with a match.  hot_n: StdMachine3 records served from
// the "shared memory" copy (leftmost / charwise / kernel 0: leading wide records of k_scan_rk), kernel: the option
// (1, 2 and 4 run 3, as on the device), seg_len > 0: segments of that length where the device may cut.
extern "C" int emu_reduce_batch_wire(const uint8_t* wire, size_t wire_len, int charwise, int mode, int rk, const uint8_t* text,
                                     const uint64_t* offs, uint64_t n, uint32_t hot_n, int kernel, uint32_t seg_len,
                                     uint64_t* counts, uint32_t* first, uint8_t* found, uint64_t* total) {
    HostImage img;
    bool lm = false;
    const int rc = load(wire, wire_len, charwise != 0, &img, &lm);
    if (rc) return rc;
    if (mode < M_FIND || mode > M_LEFTMOST || (rk != RK_COUNT && rk != RK_FIRST)) return DACH_INVALID_ARGUMENT;
    if ((mode == M_LEFTMOST) != lm) return DACH_MATCH_KIND_MISMATCH;
    ScanInputs in = plan_inputs(img, charwise != 0, mode);
    in.opt_kernel = kernel;
    in.matches = false;
    in.first = rk == RK_FIRST;
    const ScanPlan plan = plan_scan(in);
    const Segments S = seg_table(offs, n, plan.seg ? seg_len : 0, 0);
    std::vector<unsigned long long> item_count(S.n_items ? S.n_items : 1, 0);
    std::vector<uint4> item_first(S.n_items ? S.n_items : 1);
    ScanCtrl ctrl;
    memset(&ctrl, 0, sizeof(ctrl));
    ScanParams P = scan_params(img, text, offs, n, S, &ctrl);
    P.item_count = item_count.data();
    P.item_first = item_first.data();
    const Smem sm(img, plan, hot_n, P.text_lo, P.text_end);
    if (rk == RK_COUNT) {
        run_rk_modes<RK_COUNT>(plan, charwise != 0, P, sm, 1, 3);
        const uint64_t tot = fold_count(S, n, item_count, counts);
        if (total) *total = tot;
    } else {
        run_rk_modes<RK_FIRST>(plan, charwise != 0, P, sm, 1, 3);
        const uint64_t tot = fold_first(S, n, item_first, nullptr, first, found);
        if (total) *total = tot;
    }
    return DACH_OK;
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
    HostImage img;
    bool lm = false;
    const int rc = load(wire, wire_len, charwise != 0, &img, &lm);
    if (rc) return rc;
    if (rk == RK_HIST && !check_hist(img, key, n_hist)) return DACH_INVALID_ARGUMENT;
    if (mode != M_FIND && mode != M_OVERLAPPING) return DACH_INVALID_ARGUMENT;  // the crate's two steppers
    if (lm) return DACH_MATCH_KIND_MISMATCH;
    if (rk != RK_COUNT && rk != RK_FIRST && rk != RK_HIST) return DACH_INVALID_ARGUMENT;
    if (total) *total = 0;
    if (n == 0) return DACH_OK;
    // the refusal of enqueue_rk / enqueue_scan: stream chunks need a Standard lane machine
    ScanInputs in = plan_inputs(img, charwise != 0, mode);
    in.opt_kernel = kernel;
    in.stream = true;
    in.matches = false;
    in.first = rk == RK_FIRST;
    const ScanPlan plan = plan_scan(in);
    if (plan.refused) return DACH_INVALID_ARGUMENT;
    const uint32_t n_cslots = (uint32_t)img.opos_tab.size();
    std::vector<unsigned long long> item_count(n, 0), slot_hist(n_cslots + 1, 0), rec_hist(img.outputs.size() / 4 + 1, 0);
    std::vector<uint4> item_first(n);
    const Segments S = seg_table(offs, n, 0, 0);  // one item per chunk
    ScanCtrl ctrl;
    memset(&ctrl, 0, sizeof(ctrl));
    ScanParams P = scan_params(img, text, offs, n, S, &ctrl);
    P.state_io = state_io;
    P.item_count = item_count.data();
    P.item_first = item_first.data();
    P.slot_hist = slot_hist.data();
    P.rec_hist = rec_hist.data();
    P.hist_smem = rk == RK_HIST ? (uint32_t)std::min<int64_t>(std::max<int64_t>(hist_smem, 0), std::min<int64_t>(n_cslots, 16384)) : 0;
    const Smem sm(img, plan, hot_n, P.text_lo, P.text_end);
    uint64_t tot = 0;
    if (rk == RK_COUNT) {
        run_rk_modes<RK_COUNT>(plan, charwise != 0, P, sm, 2, 2);
        tot = fold_count(S, n, item_count, counts);
    } else if (rk == RK_FIRST) {
        run_rk_modes<RK_FIRST_STREAM>(plan, charwise != 0, P, sm, 2, 2);
        tot = fold_first(S, n, item_first, pos, first, found);
    } else {
        run_rk_modes<RK_HIST>(plan, charwise != 0, P, sm, 2, 2);
        tot = hist_fold(img, true, mode, slot_hist, rec_hist, key, hist);
    }
    if (total) *total = tot;
    return DACH_OK;
}
