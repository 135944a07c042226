// CPU emulation of masked text (TEST INFRASTRUCTURE ONLY): dach_dev_mask_batch -- k_check_offsets, k_mask_copy's copy
// of the text, then the scan with a MaskSink that fills every byte of every match.  The drivers are emu_driver.h's.
#include "emu_driver.h"

using namespace emu;

// dach_dev_mask_batch: out[0, text_bytes) = text, then `fill` over every match.  hot_n: StdMachine3 records served from
// the "shared memory" copy (kernel 0: leading wide records), kernel: the option (1, 2 and 4 run 3, as on the device),
// seg_len > 0: segments of that length where the device may cut.  *which_out: the kernel that ran (3, 1, 0) and whether
// segments were cut (+ 8).
extern "C" int emu_mask_batch_wire(const uint8_t* wire, size_t wire_len, int charwise, int mode, const uint8_t* text, const uint64_t* offs,
                                   uint64_t n, uint64_t text_bytes, uint8_t fill, uint32_t hot_n, int kernel, uint32_t seg_len, uint8_t* out,
                                   int* which_out) {
    HostImage img;
    bool lm = false;
    const int rc = load(wire, wire_len, charwise != 0, &img, &lm);
    if (rc) return rc;
    if (charwise && fill >= 0x80) return DACH_INVALID_ARGUMENT;
    if (mode < M_FIND || mode > M_LEFTMOST) return DACH_INVALID_ARGUMENT;
    if ((mode == M_LEFTMOST) != lm) return DACH_MATCH_KIND_MISMATCH;
    for (uint64_t h = 0; h < n; ++h)  // k_check_offsets: a refused call writes nothing
        if (offs[h + 1] < offs[h] || offs[h + 1] - offs[h] > 0xffffffffull || offs[h + 1] > text_bytes) return DACH_INVALID_ARGUMENT;
    if (text_bytes) memcpy(out, text, text_bytes);  // k_mask_copy
    if (which_out) *which_out = -1;
    if (n == 0) return DACH_OK;
    ScanInputs in = plan_inputs(img, charwise != 0, mode);
    in.opt_kernel = kernel;
    in.matches = false;
    const ScanPlan plan = plan_scan(in);
    const Segments S = seg_table(offs, n, plan.seg ? seg_len : 0, 0);
    ScanCtrl ctrl;
    memset(&ctrl, 0, sizeof(ctrl));
    ScanParams P = scan_params(img, text, offs, n, S, &ctrl);
    P.mask_out = out;
    P.mask_fill = fill;
    const Smem sm(img, plan, hot_n, P.text_lo, P.text_end);
    run_rk_modes<RK_MASK>(plan, charwise != 0, P, sm, 1, 3);
    if (which_out) *which_out = (plan.machine == Machine::Std3 ? 3 : plan.lane_machine() ? 1 : 0) + (S.seg_len ? 8 : 0);
    return DACH_OK;
}
