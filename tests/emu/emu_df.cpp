// CPU emulation of per-pattern document frequencies (TEST INFRASTRUCTURE ONLY): dach_dev_df_batch as df_windows() in
// dev_scan.cu runs it -- the scan of each window with a DfSink whose inserts go into the handle's open-addressing pair
// sets (df_insert), then k_df_expand, k_df_add and k_df_clear restated, with the split of a window that overflows.
// The drivers are emu_driver.h's.
#include "emu_driver.h"

using namespace emu;

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
    HostImage img;
    bool lm = false;
    const int rc = load(wire, wire_len, charwise != 0, &img, &lm);
    if (rc) return rc;
    if (!check_hist(img, key, n_df)) return DACH_INVALID_ARGUMENT;
    if (mode < M_FIND || mode > M_LEFTMOST) return DACH_INVALID_ARGUMENT;
    if ((mode == M_LEFTMOST) != lm) return DACH_MATCH_KIND_MISMATCH;
    if (total) *total = 0;
    for (int i = 0; i < 6; ++i) out[i] = 0;
    if (n == 0) return DACH_OK;
    ScanInputs in = plan_inputs(img, charwise != 0, mode);
    in.opt_kernel = kernel;
    in.matches = false;
    const ScanPlan plan = plan_scan(in);
    const bool machine = plan.lane_machine();
    const bool chain = machine && mode == M_OVERLAPPING;
    const uint32_t n_cslots = (uint32_t)img.opos_tab.size(), n_out = (uint32_t)(img.outputs.size() / 4);
    // df_prepare
    Sets D;
    const uint64_t limit = std::min<uint64_t>(std::max<uint64_t>({(uint64_t)std::max<int64_t>(df_pairs, 1), n_cslots, n_out}), 1ull << 30);
    uint64_t cap = 2;
    while (cap < 2 * limit) cap <<= 1;
    D.mask = (uint32_t)(cap - 1);
    D.limit = (uint32_t)limit;
    for (int i = 0; i < 2; ++i) {
        D.tab[i].assign(cap, DF_EMPTY);
        D.list[i].assign(cap, 0);
    }
    std::vector<unsigned long long> acc(std::max<uint64_t>(n_df, 1), 0);
    const Smem sm(img, plan, hot_n, text + offs[0], text + offs[n]);

    // one window: haystacks [a, b); returns whether it overflowed (and then added nothing)
    auto window = [&](uint64_t a, uint64_t b, uint64_t* added) -> bool {
        const Segments S = seg_table(offs + a, b - a, plan.seg ? seg_len : 0, 0);
        ScanCtrl ctrl;
        memset(&ctrl, 0, sizeof(ctrl));
        ScanParams P = scan_params(img, text, offs, n, S, &ctrl);
        P.offs = offs + a;  // the window's haystacks; the text bounds stay the batch's
        P.df_key_value = key == 1;
        P.df_slots = D.set(0);
        P.df_keys = D.set(1);
        run_rk_modes<RK_DF>(plan, charwise != 0, P, sm, 1, 4);
        // k_df_expand
        if (machine && !ctrl.overflow) {
            for (unsigned int i = 0; i < D.n[0]; ++i) {
                const unsigned long long pair = D.tab[0][D.list[0][i]];
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
            for (unsigned int i = 0; i < D.n[1]; ++i) acc[(uint32_t)D.tab[1][D.list[1][i]]] += 1;
            *added += D.n[1];
        }
        out[4] = std::max<uint64_t>(out[4], D.n[0]);
        out[5] = std::max<uint64_t>(out[5], D.n[1]);
        // k_df_clear, then the counters
        for (int s = 0; s < 2; ++s)
            for (unsigned int i = 0; i < D.n[s]; ++i) D.tab[s][D.list[s][i]] = DF_EMPTY;
        D.n[0] = D.n[1] = 0;
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
        for (unsigned long long v : D.tab[s]) out[3] += v != DF_EMPTY;
    for (uint64_t i = 0; i < n_df; ++i) df[i] += acc[i];
    if (total) *total = sum;
    out[2] = (plan.machine == Machine::Std3 ? 3 : machine ? 1 : 0) + (chain ? 8 : 0);
    return DACH_OK;
}
