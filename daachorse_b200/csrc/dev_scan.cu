// CUDA kernels (sm_90a) and the device half of the C ABI of libdaachorse_b200.
//
// One scan is two phases that only enqueue work (enqueue_scan / enqueue_place; dach_dev_scan_batch runs them back to
// back on one stream, dach_job_* exposes them, dach_group_* makes the second one the exchange step of a sharded batch):
//   phase 1
//     k_check_offsets           the caller's offsets: ascending, inside the text, no haystack of 4 GiB or more
//     k_seg_*                   (find_overlapping / no_suffix) cut haystacks into segments with a warm-up
//     k_scan_machine<M, LANE>   persistent grid (CTAs = SMs x ctas_per_sm); warps of 32 independent walkers pull
//                               items from one atomic counter and step them in lock step through the automaton
//                               image -- one record fetch per lane per iteration (scan_lane.cuh: StdMachine3,
//                               LmMachine, CwMachine); matches go to pooled 256-byte blocks -- StdMachine3 stores
//                               its output events there as they are (event blocks), the others match tuples.
//       k_scan_duo<MODE>        StdMachine3 with two haystacks per lane (option kernel = 4; measured slower)
//       k_scan<CHARWISE, MODE>  lane per haystack, reference-shaped loop: automata above 2^24 slots, find_iter with
//                               an empty pattern, and option kernel = 0
//     k_scan_machine_rk / k_scan_rk  the same machines / loops with a COUNT, FIRST, HIST or DF sink (dach_dev_count_batch,
//                               dach_dev_first_batch, dach_dev_hist_batch, dach_dev_df_batch), followed by k_count_hay /
//                               k_first_hay (per-haystack results), k_hist_heads / k_hist_fold (per-pattern counts) or
//                               k_df_expand / k_df_add / k_df_clear (document frequencies, window by window); on stream
//                               chunks (dach_dev_count_stream, dach_dev_first_stream, dach_dev_hist_stream) with the
//                               state carried, FIRST's lanes running to the chunk's end and k_first_stream after them
//     k_offsets_*               exclusive scan of the per-item match counts
//     k_blk_index               pool blocks listed in output order (large batches)
//   phase 2
//     k_gather                  every pooled block to its final place: dense, ordered exactly like the crate's
//                               iterators, at a device-side base, into any buffer (the caller's, a job's packed copy)
//     k_expand                  the same for event blocks: every event expanded into its output list's tuples
//     k_final_offsets           the caller's per-haystack offsets (+ base)
//     k_add_base                stream chunks: positions in stream coordinates
//   shard groups (dach_group_place)
//     k_group_publish / k_group_wait_base / k_group_signal_done / k_group_wait_all / k_group_release
//                               counts published into every rank's control block, bases derived from them, done
//                               flags -- system-scope releases, local polling; the packed matches go to rank 0 through
//                               a copy engine (or k_push: destination-aligned 16-byte peer stores)
// No CPU fallback exists: every entry point here fails with DACH_CUDA_ERROR without a device.
#include <cuda_runtime.h>

#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "dev_image.h"
#include "host.h"
#include "scan_lane.cuh"

namespace dach {

// ------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------

constexpr int kMaxThreads = 1024;
constexpr int kMaxDevices = 64;
constexpr uint32_t kRootBytes = 1024;  // 256 x u32 at the front of dynamic shared memory
// Staged hot records (option hot_entries; DESIGN.md section 4.1).  kHotAuto, the default, stages kHotQueued records in the
// kernels with event queues and fills kDirectSmemBudget in k_scan_direct, which has none.
constexpr int64_t kHotAuto = -2;
constexpr int64_t kHotQueued = 6144;
// H100 splits 256 KiB per SM between shared memory and L1 in steps; past the 196 KiB step the next is 228 KiB, which
// leaves L1 28 KiB instead of 60 KiB -- too little for the record fetches in flight.  A CTA's dynamic shared memory must
// stay below the step by the 1 KiB the system reserves per CTA and the kernel's static shared memory (512 B allowed).
constexpr uint32_t kSmemCarveoutStep = 196 * 1024, kSmemPerSmMax = 228 * 1024;
constexpr uint32_t kDirectSmemBudget = kSmemCarveoutStep - 1024 - 512;
constexpr int kDirectCarveoutPct = (int)(100ull * kSmemCarveoutStep / kSmemPerSmMax);  // rounds up to the 196 KiB step
// DF: pairs per window by default (option df_pairs).  DESIGN.md section 4.9 measures the distinct pairs per MiB of
// text (tools/lane_stats.py --pairs): at most 84 k (C2), so the largest slice cut_slices makes on the bench workloads
// (540 MiB of C3 find_iter, 26 k pairs per MiB) fits in one window.  Cost: 2 sets x 2^25 entries x 12 B = 768 MiB.
constexpr int64_t kDefaultDfPairs = 1 << 24;

// the result sink of each result kind
template <int RK>
using SinkOf = typename std::conditional<
    RK == RK_COUNT, CountSink,
    typename std::conditional<
        RK == RK_FIRST || RK == RK_FIRST_STREAM, FirstSink,
        typename std::conditional<
            RK == RK_HIST, HistSink,
            typename std::conditional<RK == RK_DF, DfSink, typename std::conditional<RK == RK_MASK, MaskSink, Emitter>::type>::type>::type>::type>::type;

template <bool CHARWISE, int MODE, class SINK>
__device__ __forceinline__ void scan_items(const ScanParams& P) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint32_t* s_root = reinterpret_cast<uint32_t*>(smem_raw);
    uint4* s_hot = reinterpret_cast<uint4*>(smem_raw + kRootBytes);
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) s_root[i] = P.root_table[i];
    for (uint32_t i = threadIdx.x; i < P.hot_n; i += blockDim.x) s_hot[i] = P.rec[i];
    __syncthreads();

    RecView V{P.rec, s_hot, P.hot_n, s_root};
    TextWin T;
    SINK E;
    for (;;) {
        const unsigned long long item = bump_u64(&P.ctrl->next_item);
        if (item >= P.n_items) break;
        const uint64_t o0 = P.offs[item], o1 = P.offs[item + 1];
        const uint32_t len = (uint32_t)(o1 - o0);
        T.open(P.text + o0);
        E.begin((uint32_t)item);
        if constexpr (SINK::KIND == RK_MASK) E.base = P.mask_out + o0;
        if (MODE == M_LEFTMOST)
            scan_leftmost<CHARWISE>(P, V, T, E, len);
        else
            scan_standard<CHARWISE, MODE>(P, V, T, E, len);
        E.finish(P);
    }
}

template <bool CHARWISE, int MODE>
__global__ void __launch_bounds__(kMaxThreads, 1) k_scan(ScanParams P) {
    scan_items<CHARWISE, MODE, Emitter>(P);
}
// COUNT / FIRST / HIST / DF (result kind RK) on the lane-per-haystack loops
template <bool CHARWISE, int MODE, int RK>
__global__ void __launch_bounds__(kMaxThreads, 1) k_scan_rk(ScanParams P) {
    scan_items<CHARWISE, MODE, SinkOf<RK>>(P);
}

// ---- v1: warp-synchronous lane machine for the bytewise Standard modes ---------------------------
// One warp = 32 independent haystack walkers kept in lock step: every iteration each lane does at
// most one record fetch (shared memory for the hot prefix, L1/L2 otherwise).  When any lane's
// event queue is full or its haystack is finished, the whole warp runs the service phase: drain
// all queues (output-list walks, match stores), close finished items, pull new items with one
// warp-aggregated atomic.

// ---- TMA bulk copy global -> shared (cp.async.bulk, completion on an mbarrier) -----------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    }
}

// M: the lane machine (StdMachine3 / StdMachine2 / StdMachine / LmMachine / CwMachine), LANE: its per-lane state.
// OPS: where drain() and begin_item() come from (M itself for matches, SinkOps for COUNT / FIRST), SINK: the result.
// HOT: the leading P.hot_entries compact records (the front of the hot region, dev_image.cpp) are staged in
// shared memory by TMA bulk copies and served from there (StdMachine3).
template <class M, class OPS, class LANE, class SINK, bool HOT>
__device__ __forceinline__ void scan_machine(const ScanParams& P) {
    // dynamic shared memory: [hot records hot_entries x 16 B (HOT only)][event queues LANE_Q x blockDim x 8 B]
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint4* s_hot = reinterpret_cast<uint4*>(smem_raw);
    QEntry* s_queue = reinterpret_cast<QEntry*>(smem_raw + (HOT ? (size_t)P.hot_entries * 16 : 0));
    __shared__ __align__(8) uint64_t s_bar;
    if (HOT) {
        // one elected thread arms the mbarrier and lets the TMA engine stage the hot records
        // (up to 144 KiB) while the other threads set up
        if (threadIdx.x == 0) mbar_init(&s_bar, 1);
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t hot_bytes = P.hot_entries * 16u;
            mbar_expect_tx(&s_bar, hot_bytes);
            for (uint32_t off = 0; off < hot_bytes; off += 32768u)
                tma_bulk_g2s(reinterpret_cast<unsigned char*>(s_hot) + off, reinterpret_cast<const unsigned char*>(P.crec) + off,
                             min(32768u, hot_bytes - off), &s_bar);
        }
    }

    const StdEnv Ev{P.crec,      s_hot,       smem_u32(s_hot), HOT ? P.hot_entries : 0u, P.opos_tab, P.text_end, P.text_lo, P.root_base, P.root_opos ? CF_OUT : 0u,
                    s_queue + threadIdx.x, blockDim.x, 0u, P.mapper, P.mapper_len, ld_u4(P.crec + D_ROOT)};
    const unsigned FULL = 0xffffffffu;
    const unsigned lane = threadIdx.x & 31u;
    LANE L;
    L.fl = M::IDLE;
    L.qn = 0;
    SINK E;
    E.begin(0);
    if constexpr (SINK::KIND == RK_HIST) {
        // HIST: u32 counters of compact slots [0, hist_smem) behind the queues
        E.s_cnt = reinterpret_cast<unsigned int*>(s_queue + (size_t)LANE_Q * blockDim.x);
        E.k = P.hist_smem;
        for (uint32_t i = threadIdx.x; i < P.hist_smem; i += blockDim.x) E.s_cnt[i] = 0;
        __syncthreads();
    }
    bool exhausted = false;
    const unsigned long long n_items = P.n_items_dev ? *P.n_items_dev : P.n_items;
    if (HOT) mbar_wait(&s_bar, 0);
    for (;;) {
        // ---- service phase (the warp is converged here) ----
        if constexpr (std::is_same<SINK, EventSink>::value) {
            // event blocks: the lanes that need one this phase take them with one atomic for the warp
            const bool want = (L.fl & F_ACTIVE) && OPS::need_block(L, Ev, E);
            const unsigned mb = __ballot_sync(FULL, want);
            uint32_t blk = 0;
            if (mb) {
                const int leader = __ffs(mb) - 1;
                unsigned int b0 = 0;
                if ((int)lane == leader) b0 = atomicAdd(&P.ctrl->blk_cursor, (unsigned int)__popc(mb));
                blk = __shfl_sync(FULL, b0, leader) + __popc(mb & ((1u << lane) - 1u));
            }
            if (L.fl & F_ACTIVE) OPS::drain(L, Ev, P, E, blk);
        } else {
            if (L.fl & F_ACTIVE) OPS::drain(L, Ev, P, E);
        }
        if ((L.fl & (F_ACTIVE | F_DONE)) == (F_ACTIVE | F_DONE)) {
            E.finish(P);
            M::finish_item(L, P);
            L.fl = M::IDLE;
        }
        const bool need = !(L.fl & F_ACTIVE) && !exhausted;
        const unsigned m = __ballot_sync(FULL, need);
        if (m) {
            const int leader = __ffs(m) - 1;
            unsigned long long base = 0;
            if ((int)lane == leader) base = atomicAdd(&P.ctrl->next_item, (unsigned long long)__popc(m));
            base = __shfl_sync(FULL, base, leader);
            if (need) {
                const unsigned long long item = base + __popc(m & ((1u << lane) - 1u));
                if (item < n_items)
                    OPS::begin_item(L, P, Ev, E, item, nullptr);
                else
                    exhausted = true;
            }
        }
        if (!__any_sync(FULL, (L.fl & F_ACTIVE) != 0)) break;
        // ---- lock-step iterations until some lane needs service ----
        bool stop = false;
        while (!stop) {
            M::text_topup(L, Ev, nullptr);
            if (M::LEAN) {  // the lane's stop bit says it all; read once per top-up period
#pragma unroll 1
                for (int k = 0; k < M::TOPUP; ++k) (void)M::step(L, Ev, nullptr);
                stop = __any_sync(FULL, (L.fl & (F_ACTIVE | M::IDLE)) == (F_ACTIVE | M::IDLE));
            } else if (M::LAZY) {  // look for lanes that need service once per top-up period, not per iteration
                // (batching further -- wait for four lanes or four periods -- idles lanes that have
                // finished short haystacks while the rest of the warp runs on)
                bool waiting = false;
#pragma unroll 1
                for (int k = 0; k < M::TOPUP; ++k) {
                    const bool ok = M::step(L, Ev, nullptr);
                    waiting |= !ok;
                }
                stop = __any_sync(FULL, waiting && (L.fl & F_ACTIVE));
            } else {
#pragma unroll 1
                for (int k = 0; k < M::TOPUP; ++k) {
                    const bool ok = M::step(L, Ev, nullptr);
                    if (__any_sync(FULL, !ok && (L.fl & F_ACTIVE))) {
                        stop = true;
                        break;
                    }
                }
            }
        }
    }
    if constexpr (SINK::KIND == RK_HIST) {  // the CTA's shared-memory counts, once
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < P.hist_smem; i += blockDim.x)
            if (E.s_cnt[i]) red_add_u64(P.slot_hist + i, E.s_cnt[i]);
    }
}

// matches: StdMachine3 stores events (EventOps, expanded by k_expand), the other machines match tuples (k_gather)
template <class M, class LANE, int MAXT, int MINB, bool HOT>
__global__ void __launch_bounds__(MAXT, MINB) k_scan_machine(ScanParams P) {
    if constexpr (M::QLEN)
        scan_machine<M, EventOps<M::ITER>, LANE, EventSink, HOT>(P);
    else
        scan_machine<M, M, LANE, Emitter, HOT>(P);
}
// COUNT / FIRST (result kind RK) on the lane machine M running iterator MODE
template <class M, class LANE, int MODE, int RK, bool HOT>
__global__ void __launch_bounds__(1024, 1) k_scan_machine_rk(ScanParams P) {
    scan_machine<M, SinkOps<M, MODE, RK>, LANE, SinkOf<RK>, HOT>(P);
}

// ---- StdMachine3's matches path without the queue (DirectOps, scan_lane.cuh) --------------------------------------
// scan_machine's loop, but the lanes store their events at the landing that makes them.  Dynamic shared memory holds
// the hot records only.  Service phase: the lanes with a pending event that needs a block take one (one atomic for the
// warp) and store it, then finished items close and new ones start, as in scan_machine.
template <int MODE, bool HOT>
__global__ void __launch_bounds__(1024, 1) k_scan_direct(ScanParams P) {
    using M = StdMachine3<MODE>;
    using OPS = DirectOps<MODE>;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint4* s_hot = reinterpret_cast<uint4*>(smem_raw);
    __shared__ __align__(8) uint64_t s_bar;
    if (HOT) {
        if (threadIdx.x == 0) mbar_init(&s_bar, 1);
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t hot_bytes = P.hot_entries * 16u;
            mbar_expect_tx(&s_bar, hot_bytes);
            for (uint32_t off = 0; off < hot_bytes; off += 32768u)
                tma_bulk_g2s(reinterpret_cast<unsigned char*>(s_hot) + off, reinterpret_cast<const unsigned char*>(P.crec) + off,
                             min(32768u, hot_bytes - off), &s_bar);
        }
    }
    const StdEnv Ev{P.crec,  s_hot,   smem_u32(s_hot), HOT ? P.hot_entries : 0u, P.opos_tab, P.text_end, P.text_lo, P.root_base, P.root_opos ? CF_OUT : 0u,
                    nullptr, 0u,      0u,              P.mapper,                 P.mapper_len, ld_u4(P.crec + D_ROOT)};
    const unsigned FULL = 0xffffffffu;
    const unsigned lane = threadIdx.x & 31u;
    Lane3D L;
    L.fl = M::IDLE;
    L.qn = 0;
    L.E.begin(0);
    bool exhausted = false;
    const unsigned long long n_items = P.n_items_dev ? *P.n_items_dev : P.n_items;
    if (HOT) mbar_wait(&s_bar, 0);
    for (;;) {
        // ---- service phase (the warp is converged here) ----
        const bool want = OPS::need_block(L);
        const unsigned mb = __ballot_sync(FULL, want);
        uint32_t blk = 0;
        if (mb) {
            const int leader = __ffs(mb) - 1;
            unsigned int b0 = 0;
            if ((int)lane == leader) b0 = atomicAdd(&P.ctrl->blk_cursor, (unsigned int)__popc(mb));
            blk = __shfl_sync(FULL, b0, leader) + __popc(mb & ((1u << lane) - 1u));
        }
        if (L.fl & F_ACTIVE) OPS::drain(L, Ev, P, blk);
        if ((L.fl & (F_ACTIVE | F_DONE)) == (F_ACTIVE | F_DONE)) {
            L.E.finish(P);
            M::finish_item(L, P);
            L.fl = M::IDLE;
        }
        const bool need = !(L.fl & F_ACTIVE) && !exhausted;
        const unsigned m = __ballot_sync(FULL, need);
        if (m) {
            const int leader = __ffs(m) - 1;
            unsigned long long base = 0;
            if ((int)lane == leader) base = atomicAdd(&P.ctrl->next_item, (unsigned long long)__popc(m));
            base = __shfl_sync(FULL, base, leader);
            if (need) {
                const unsigned long long item = base + __popc(m & ((1u << lane) - 1u));
                if (item < n_items)
                    OPS::begin_item(L, P, Ev, item);
                else
                    exhausted = true;
            }
        }
        if (!__any_sync(FULL, (L.fl & F_ACTIVE) != 0)) break;
        // ---- lock-step iterations until some lane needs service ----
        bool stop = false;
        while (!stop) {
            M::text_topup(L, Ev, nullptr);
#pragma unroll 1
            for (int k = 0; k < M::TOPUP; ++k) (void)M::step(L, Ev, nullptr);
            stop = __any_sync(FULL, (L.fl & (F_ACTIVE | F3_STOP)) == (F_ACTIVE | F3_STOP));
        }
    }
}

// ---- StdMachine3, two haystacks per lane ------------------------------------------------------------------
// The lane machine is latency-bound: one dependent record fetch per lane and iteration, and a warp moves at
// the pace of its slowest lane (most stalls sit on the fetch's scoreboard).  Here every lane walks TWO independent haystacks:
// both fetches of an iteration are in flight before either result is looked at, so an SM has twice the loads
// outstanding with the same number of warps.  Lane logic: StdMachine3's probe / resolve, unchanged; the two
// walkers have their own event queues and take their items from the same counter.
template <int MODE, int MAXT, bool HOT>
__global__ void __launch_bounds__(MAXT, 1) k_scan_duo(ScanParams P) {
    using M = StdMachine3<MODE>;
    // dynamic shared memory: [hot records hot_entries x 16 B (HOT only)][event queues 2 x LANE_Q x blockDim x 8 B]
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint4* s_hot = reinterpret_cast<uint4*>(smem_raw);
    QEntry* s_queue = reinterpret_cast<QEntry*>(smem_raw + (HOT ? (size_t)P.hot_entries * 16 : 0));
    __shared__ __align__(8) uint64_t s_bar;
    if (HOT) {
        if (threadIdx.x == 0) mbar_init(&s_bar, 1);
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t hot_bytes = P.hot_entries * 16u;
            mbar_expect_tx(&s_bar, hot_bytes);
            for (uint32_t off = 0; off < hot_bytes; off += 32768u)
                tma_bulk_g2s(reinterpret_cast<unsigned char*>(s_hot) + off, reinterpret_cast<const unsigned char*>(P.crec) + off,
                             min(32768u, hot_bytes - off), &s_bar);
        }
    }
    const StdEnv Ev0{P.crec, s_hot, smem_u32(s_hot), HOT ? P.hot_entries : 0u, P.opos_tab, P.text_end, P.text_lo, P.root_base, P.root_opos ? CF_OUT : 0u,
                     s_queue + threadIdx.x, blockDim.x, 0u, P.mapper, P.mapper_len, ld_u4(P.crec + D_ROOT)};
    StdEnv Ev1 = Ev0;
    Ev1.q = s_queue + (size_t)LANE_Q * blockDim.x + threadIdx.x;
    const unsigned FULL = 0xffffffffu;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned lt = (1u << lane) - 1u;
    Lane3 L0, L1;
    L0.fl = L1.fl = M::IDLE;
    L0.qn = L1.qn = 0;
    Emitter E0, E1;
    E0.begin(0);
    E1.begin(0);
    bool exhausted = false;
    const unsigned long long n_items = P.n_items_dev ? *P.n_items_dev : P.n_items;
    constexpr uint32_t WAIT = F_ACTIVE | F3_STOP;
    if (HOT) mbar_wait(&s_bar, 0);
    for (;;) {
        // ---- service phase (the warp is converged here) ----
        if (L0.fl & F_ACTIVE) M::drain(L0, Ev0, P, E0);
        if (L1.fl & F_ACTIVE) M::drain(L1, Ev1, P, E1);
        if ((L0.fl & (F_ACTIVE | F_DONE)) == (F_ACTIVE | F_DONE)) {
            E0.finish(P);
            M::finish_item(L0, P);
            L0.fl = M::IDLE;
        }
        if ((L1.fl & (F_ACTIVE | F_DONE)) == (F_ACTIVE | F_DONE)) {
            E1.finish(P);
            M::finish_item(L1, P);
            L1.fl = M::IDLE;
        }
        const bool need0 = !(L0.fl & F_ACTIVE) && !exhausted, need1 = !(L1.fl & F_ACTIVE) && !exhausted;
        const unsigned m0 = __ballot_sync(FULL, need0), m1 = __ballot_sync(FULL, need1);
        if (m0 | m1) {
            unsigned long long base = 0;
            if (lane == 0) base = atomicAdd(&P.ctrl->next_item, (unsigned long long)(__popc(m0) + __popc(m1)));
            base = __shfl_sync(FULL, base, 0);
            if (need0) {
                const unsigned long long item = base + __popc(m0 & lt);
                if (item < n_items)
                    M::begin_item(L0, P, Ev0, E0, item, nullptr);
                else
                    exhausted = true;
            }
            if (need1) {
                const unsigned long long item = base + __popc(m0) + __popc(m1 & lt);
                if (item < n_items)
                    M::begin_item(L1, P, Ev1, E1, item, nullptr);
                else
                    exhausted = true;
            }
        }
        if (!__any_sync(FULL, ((L0.fl | L1.fl) & F_ACTIVE) != 0)) break;
        // ---- lock-step iterations until some walker needs service ----
        bool stop = false;
        while (!stop) {
            M::text_topup(L0, Ev0, nullptr);
            M::text_topup(L1, Ev1, nullptr);
#pragma unroll 1
            for (int k = 0; k < M::TOPUP; ++k) {
                uint32_t own0, own1;
                const uint32_t a0 = M::probe(L0, own0), a1 = M::probe(L1, own1);
                const uint4 x0 = M::fetch(Ev0, a0);
                const uint4 x1 = M::fetch(Ev1, a1);
                M::resolve(L0, Ev0, x0, a0, own0);
                M::resolve(L1, Ev1, x1, a1, own1);
            }
            stop = __any_sync(FULL, (L0.fl & WAIT) == WAIT || (L1.fl & WAIT) == WAIT);
        }
    }
}

// ---- exclusive scan of counts (u32) into offsets (u64) -----------------------------------
constexpr int kScanThreads = 256;
constexpr int kScanPerThread = 8;
constexpr int kScanTile = kScanThreads * kScanPerThread;

__device__ __forceinline__ unsigned long long block_exclusive_scan(unsigned long long v, unsigned long long* total) {
    __shared__ unsigned long long warp_sums[kScanThreads / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned long long inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        unsigned long long t = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += t;
    }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        unsigned long long w = lane < kScanThreads / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            unsigned long long t = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= d) w += t;
        }
        if (lane < kScanThreads / 32) warp_sums[lane] = w;
    }
    __syncthreads();
    const unsigned long long before = wid ? warp_sums[wid - 1] : 0;
    *total = warp_sums[kScanThreads / 32 - 1];
    __syncthreads();
    return before + inc - v;
}

// PER > 1: scan ceil(count / PER) (pool blocks per item, PER entries a block) instead of the counts themselves
template <uint32_t PER>
__device__ __forceinline__ uint32_t scan_term(uint32_t count) {
    return PER > 1 ? (count + PER - 1) / PER : count;
}

template <uint32_t PER>
__global__ void __launch_bounds__(kScanThreads) k_offsets_tile_sums(const uint32_t* counts, uint64_t n,
                                                                      unsigned long long* tile_sums) {
    const uint64_t base = (uint64_t)blockIdx.x * kScanTile;
    unsigned long long s = 0;
    for (int k = 0; k < kScanPerThread; ++k) {
        const uint64_t i = base + (uint64_t)k * kScanThreads + threadIdx.x;
        if (i < n) s += scan_term<PER>(counts[i]);
    }
    unsigned long long total;
    (void)block_exclusive_scan(s, &total);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}

// one CTA turns the tile sums into exclusive tile offsets (in place)
__global__ void __launch_bounds__(kScanThreads) k_offsets_scan_tiles(unsigned long long* tile_sums, uint64_t n_tiles) {
    __shared__ unsigned long long carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint64_t base = 0; base < n_tiles; base += kScanThreads) {
        const uint64_t i = base + threadIdx.x;
        const unsigned long long v = i < n_tiles ? tile_sums[i] : 0;
        unsigned long long total;
        const unsigned long long ex = block_exclusive_scan(v, &total);
        if (i < n_tiles) tile_sums[i] = carry + ex;
        __syncthreads();
        if (threadIdx.x == 0) carry += total;
        __syncthreads();
    }
}

template <uint32_t PER>
__global__ void __launch_bounds__(kScanThreads) k_offsets_apply(const uint32_t* counts, uint64_t n,
                                                                  const unsigned long long* tile_offs,
                                                                  unsigned long long* out_offs) {
    // thread t owns kScanPerThread consecutive items so that one block scan suffices
    const uint64_t first = (uint64_t)blockIdx.x * kScanTile + (uint64_t)threadIdx.x * kScanPerThread;
    uint32_t c[kScanPerThread];
    unsigned long long s = 0;
#pragma unroll
    for (int k = 0; k < kScanPerThread; ++k) {
        const uint64_t i = first + k;
        c[k] = i < n ? scan_term<PER>(counts[i]) : 0;
        s += c[k];
    }
    unsigned long long total;
    unsigned long long run = tile_offs[blockIdx.x] + block_exclusive_scan(s, &total);
#pragma unroll
    for (int k = 0; k < kScanPerThread; ++k) {
        const uint64_t i = first + k;
        if (i < n) out_offs[i] = run;
        run += c[k];
        if (i + 1 == n) out_offs[n] = run;
    }
}

// ---- gather pooled blocks into the final, ordered match array ----------------------------
// Pool blocks are handed out in the order lanes ask for them, i.e. scattered over the items in flight;
// copying them in pool order makes every 240-byte write land somewhere else in the output (partial
// sectors, no DRAM locality: 0.93 ms per GiB scanned).  k_blk_index lists the blocks in output order
// (blkmap[first block of the item + seq] = pool block) and k_gather walks that list: scattered reads
// of whole aligned 256-byte blocks, sequential writes.
__global__ void __launch_bounds__(256) k_blk_index(const uint32_t* pool, const ScanCtrl* ctrl, uint32_t pool_blocks,
                                                    const unsigned long long* blk_first, uint32_t* blkmap) {
    if (ctrl->overflow) return;
    const uint32_t used = min(ctrl->blk_cursor, pool_blocks);
    for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; b < used; b += (uint64_t)gridDim.x * blockDim.x) {
        const uint2 h = *reinterpret_cast<const uint2*>(pool + b * BLK_WORDS);  // {item, seq}
        const unsigned long long j = blk_first[h.x] + h.y;
        if (j < used) blkmap[j] = (uint32_t)b;
    }
}

// One warp per block.  Skipped entirely when the batch overflowed the pool or out_cap.  `base` (device pointer
// or nullptr = 0) is the index of this batch's first match in `out_words` -- which may be peer-mapped memory
// of another GPU (dach_group_place): the copy then IS the exchange step, NVLink stores straight into the
// gathering rank's dense buffer.
template <int U>
__global__ void __launch_bounds__(256) k_gather(const uint32_t* pool, const ScanCtrl* ctrl, uint32_t pool_blocks,
                                                 const uint32_t* counts, const unsigned long long* item_offs,
                                                 uint64_t n_items, unsigned long long out_cap, const unsigned long long* base,
                                                 uint32_t* out_words, const uint32_t* blkmap, const unsigned long long* pad_like) {
    if (ctrl->overflow) return;
    const unsigned long long b0m = base ? *base : 0ull;
    if (b0m + item_offs[n_items] > out_cap) return;
    out_words += b0m * 3ull;
    // staged copy for k_push: start at the word offset (mod 4) the tuples will have at their final base, so that
    // source and destination of the push are congruent modulo 16 bytes
    if (pad_like) out_words += (*pad_like * 3ull) & 3ull;
    const uint32_t used = min(ctrl->blk_cursor, pool_blocks);
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warp = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const uint64_t n_warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    // U blocks in flight per warp: the header -> (count, offset) -> data chains overlap
    for (uint64_t b0 = warp * U; b0 < used; b0 += n_warps * U) {
        // output word k of a block = word k % 3 of match k / 3 = block word 4 * (1 + k / 3) + k % 3
        const uint32_t k0 = lane, k1 = lane + 32;
        const uint32_t s0 = BLK_SLOT_WORDS * (1 + k0 / 3) + k0 % 3, s1 = BLK_SLOT_WORDS * (1 + k1 / 3) + k1 % 3;
        const uint32_t* blk[U];
        uint32_t item[U], seq[U], w0[U], w1[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const uint64_t b = b0 + u;
            const uint64_t bb = b < used ? b : b0;
            blk[u] = pool + (blkmap ? (uint64_t)blkmap[bb] : bb) * BLK_WORDS;
            item[u] = blk[u][0];
            seq[u] = blk[u][1];
            w0[u] = blk[u][s0];
            w1[u] = k1 < BLK_MATCHES * 3 ? blk[u][s1] : 0;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (b0 + u >= used) continue;
            const uint32_t first = seq[u] * BLK_MATCHES;
            const uint32_t nw = min(BLK_MATCHES, counts[item[u]] - first) * 3;
            uint32_t* dst = out_words + (item_offs[item[u]] + first) * 3ull;
            if (lane < nw) dst[lane] = w0[u];
            if (lane + 32 < nw) dst[lane + 32] = w1[u];
        }
    }
}

// Placement of event blocks (StdMachine3's matches path): k_gather's walk, contract and arguments, but every event
// is expanded here -- output_pos of its slot, the head record, for find_overlapping the whole parent chain.  The
// scan loop stays free of these dependent loads; here they overlap across U blocks per warp and many warps.
// Lane j of a warp takes event j of a block: a warp scan of the list lengths gives its place behind the block's
// first match (header word 2), and the lane writes its list as consecutive 12-byte tuples.
template <bool OVERLAP, int U>
__global__ void __launch_bounds__(256) k_expand(const uint32_t* pool, const ScanCtrl* ctrl, uint32_t pool_blocks,
                                                 const uint32_t* ev_counts, const unsigned long long* item_offs,
                                                 uint64_t n_items, unsigned long long out_cap, const unsigned long long* base,
                                                 uint32_t* out_words, const uint32_t* blkmap, const unsigned long long* pad_like,
                                                 const uint4* outputs, const uint32_t* opos_tab) {
    if (ctrl->overflow) return;
    const unsigned long long b0m = base ? *base : 0ull;
    if (b0m + item_offs[n_items] > out_cap) return;
    out_words += b0m * 3ull;
    if (pad_like) out_words += (*pad_like * 3ull) & 3ull;  // staged copy for k_push (k_gather)
    const uint32_t used = min(ctrl->blk_cursor, pool_blocks);
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warp = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const uint64_t n_warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t b0 = warp * U; b0 < used; b0 += n_warps * U) {
        uint4 h[U], o[U];
        uint2 ev[U];
        uint32_t len[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const uint64_t b = b0 + u < used ? b0 + u : b0;
            const uint32_t* blk = pool + (blkmap ? (uint64_t)blkmap[b] : b) * BLK_WORDS;
            h[u] = *reinterpret_cast<const uint4*>(blk);  // {item, seq, first, -}
            ev[u] = lane < BLK_EVENTS ? reinterpret_cast<const uint2*>(blk + BLK_HDR_WORDS)[lane] : make_uint2(0u, 0u);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const uint32_t nev = min(BLK_EVENTS, ev_counts[h[u].x] - h[u].y * BLK_EVENTS);
            const bool on = b0 + u < used && lane < nev;
            const uint32_t op = on ? ld_u32(opos_tab + (ev[u].y & QSLOT_MASK)) : 0u;
            o[u] = on ? ld_u4(outputs + (op - 1)) : make_uint4(0u, 0u, 0u, 0u);
            len[u] = on ? (OVERLAP ? o[u].w : 1u) : 0u;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            uint32_t inc = len[u];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
                if (lane >= (uint32_t)d) inc += t;
            }
            if (!len[u]) continue;
            uint32_t* dst = out_words + (item_offs[h[u].x] + h[u].z + (inc - len[u])) * 3ull;
            const uint32_t end = ev[u].x;
            uint4 r = o[u];
            for (uint32_t k = 0;;) {
                dst[0] = end - r.y;
                dst[1] = end;
                dst[2] = r.x;
                if (++k == len[u]) break;
                dst += 3;
                r = ld_u4(outputs + (r.z - 1));
            }
        }
    }
}

// Block descriptors of the ordered event placement (k_expand_desc): desc[j] = {pool block, its events, u64 index of its
// first match in the batch} for the j-th block in output order.  k_blk_index's walk; the header, ev_counts and
// item_offs are looked up here, on the scan stream, so that the placement's chain of dependent loads starts at the
// block's events.
__global__ void __launch_bounds__(256) k_blk_desc(const uint32_t* pool, const ScanCtrl* ctrl, uint32_t pool_blocks,
                                                   const unsigned long long* blk_first, const uint32_t* ev_counts,
                                                   const unsigned long long* item_offs, uint4* desc) {
    if (ctrl->overflow) return;
    const uint32_t used = min(ctrl->blk_cursor, pool_blocks);
    for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; b < used; b += (uint64_t)gridDim.x * blockDim.x) {
        const uint4 h = *reinterpret_cast<const uint4*>(pool + b * BLK_WORDS);  // {item, seq, first, -}
        const unsigned long long j = blk_first[h.x] + h.y;
        if (j < used) {
            const unsigned long long at = item_offs[h.x] + h.z;
            desc[j] = make_uint4((uint32_t)b, min(BLK_EVENTS, ev_counts[h.x] - h.y * BLK_EVENTS), (uint32_t)at, (uint32_t)(at >> 32));
        }
    }
}

// k_expand's contract from block descriptors and two-entry lists.  Per warp, U blocks: descriptor, events, output_pos
// of the slot and the list's pair entry are four dependent loads, issued for all U blocks before any is expanded; only
// lists of three or more (class 3) walk the outputs from the head.  No shared memory: a CTA must fit beside a resident
// scan CTA, whose staged records leave a few KiB of the carveout at most (staging a warp's run of tuples in 1 KiB for
// 16-byte stores kept the placement of step s off the SMs of the scan of step s+1: the pipelined step got slower).
constexpr uint32_t EXP_THREADS = 256;
template <bool OVERLAP, int U>
__global__ void __launch_bounds__(EXP_THREADS) k_expand_desc(const uint32_t* pool, const ScanCtrl* ctrl, uint32_t pool_blocks,
                                                            const uint4* desc, const unsigned long long* item_offs,
                                                            uint64_t n_items, unsigned long long out_cap, const unsigned long long* base,
                                                            uint32_t* out_words, const unsigned long long* pad_like,
                                                            const uint4* pairs, const uint4* outputs, const uint32_t* opos_tab) {
    if (ctrl->overflow) return;
    const unsigned long long b0m = base ? *base : 0ull;
    if (b0m + item_offs[n_items] > out_cap) return;
    out_words += b0m * 3ull;
    if (pad_like) out_words += (*pad_like * 3ull) & 3ull;  // staged copy for k_push (k_gather)
    const uint32_t used = min(ctrl->blk_cursor, pool_blocks);
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warp = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const uint64_t n_warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t b0 = warp * U; b0 < used; b0 += n_warps * U) {
        uint4 dsc[U], p[U];
        uint2 ev[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            dsc[u] = desc[b0 + u < used ? b0 + u : b0];
            if (b0 + u >= used) dsc[u].y = 0;
        }
#pragma unroll
        for (int u = 0; u < U; ++u)
            ev[u] = lane < dsc[u].y ? reinterpret_cast<const uint2*>(pool + (uint64_t)dsc[u].x * BLK_WORDS + BLK_HDR_WORDS)[lane]
                                    : make_uint2(0u, 0u);
        uint32_t op[U];
#pragma unroll
        for (int u = 0; u < U; ++u) op[u] = lane < dsc[u].y ? ld_u32(opos_tab + (ev[u].y & QSLOT_MASK)) : 0u;
#pragma unroll
        for (int u = 0; u < U; ++u) p[u] = op[u] ? ld_u4(pairs + (op[u] - 1)) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (!dsc[u].y) continue;  // (warp-uniform)
            const uint32_t cls = OVERLAP ? p[u].w >> PAIR_CLASS_SHIFT : (op[u] ? 1u : 0u);
            uint4 r = make_uint4(0u, 0u, 0u, 0u);
            if (cls == 3u) r = ld_u4(outputs + (op[u] - 1));  // head record: the chain word is the length
            const uint32_t len = cls == 3u ? r.w : cls;
            uint32_t inc = len;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
                if (lane >= (uint32_t)d) inc += t;
            }
            uint32_t* w = out_words + (((unsigned long long)dsc[u].w << 32 | dsc[u].z) + (inc - len)) * 3ull;
            const uint32_t end = ev[u].x;
            if (cls == 1u || cls == 2u) {
                w[0] = end - p[u].y;
                w[1] = end;
                w[2] = p[u].x;
                if (cls == 2u) {
                    w[3] = end - (p[u].w & PAIR_LEN_MASK);
                    w[4] = end;
                    w[5] = p[u].z;
                }
            } else if (cls == 3u) {
                for (uint32_t k = 0;;) {
                    w[0] = end - r.y;
                    w[1] = end;
                    w[2] = r.x;
                    if (++k == len) break;
                    w += 3;
                    r = ld_u4(outputs + (r.z - 1));
                }
            }
        }
    }
}

// The exchange step proper: `total` dense 12-byte tuples from local memory to out_words + 3 * base in (peer)
// memory, as DESTINATION-ALIGNED 16-byte stores -- a warp store is 512 contiguous bytes, whole 128-byte lines on
// NVLink.  (k_gather's own stores are 4 bytes per lane at the 4-byte alignment of a tuple array: as peer stores
// they split lines and reach well below what the link takes.)
// 128 threads x at most 51 registers: two CTAs fit into the registers an SM has left beside a resident scan CTA
// (1024 threads x 48), so the push of step s really runs while step s+1 is scanned.
__global__ void __launch_bounds__(128, 10) k_push(const uint32_t* src, const unsigned long long* total_ptr, const unsigned long long* base,
                                               unsigned long long out_cap, const ScanCtrl* ctrl, uint32_t* out_words) {
    if (ctrl->overflow) return;
    const unsigned long long b0 = base ? *base : 0ull, total = *total_ptr;
    if (b0 + total > out_cap) return;
    uint32_t* dst = out_words + b0 * 3ull;
    src += (b0 * 3ull) & 3ull;  // the staged copy starts at the destination's word offset modulo 4 (k_gather, pad_like)
    const unsigned long long n_words = total * 3ull;
    const unsigned long long head = min((unsigned long long)((4u - (uint32_t)(((uintptr_t)dst >> 2) & 3u)) & 3u), n_words);
    const unsigned long long n_vec = (n_words - head) / 4ull;
    const unsigned long long tid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long nth = (unsigned long long)gridDim.x * blockDim.x;
    const uint4* s4 = reinterpret_cast<const uint4*>(src + head);  // 16-byte aligned: congruent with dst + head
    uint4* d4 = reinterpret_cast<uint4*>(dst + head);
    unsigned long long v = tid;
#pragma unroll 1
    for (; v + 3ull * nth < n_vec; v += 4ull * nth) {  // four 16-byte loads, then four 16-byte peer stores in flight per thread
        const uint4 a = s4[v], b = s4[v + nth], c = s4[v + 2ull * nth], e = s4[v + 3ull * nth];
        d4[v] = a;
        d4[v + nth] = b;
        d4[v + 2ull * nth] = c;
        d4[v + 3ull * nth] = e;
    }
#pragma unroll 1
    for (; v < n_vec; v += nth) d4[v] = s4[v];
    const unsigned long long tail0 = head + 4ull * n_vec;
    if (tid < head) dst[tid] = src[tid];
    if (tid < n_words - tail0) dst[tail0 + tid] = src[tail0 + tid];
}

// per-haystack offsets of the caller: out_offs[h] = base + item_offs[first item of haystack h]; entry n (the
// batch's end) only if `last` -- a shard that is not the last one of a gathered result leaves it to its successor
__global__ void __launch_bounds__(256) k_final_offsets(const unsigned long long* seg_first, const unsigned long long* item_offs,
                                                        uint64_t n, const unsigned long long* base, int last,
                                                        unsigned long long* out_offs, const ScanCtrl* ctrl) {
    if (ctrl->bad_offsets) return;  // the scan is refused: the caller's offsets stay as they were
    const uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (h < n || (h == n && last)) out_offs[h] = (base ? *base : 0ull) + item_offs[seg_first ? seg_first[h] : h];
}

// Stream chunks: positions are reported in stream coordinates -- add the position of the chunk's first byte
// to start and end of every match of that chunk (haystack found by binary search in out_offs).
__global__ void __launch_bounds__(256) k_add_base(const ScanCtrl* ctrl, const unsigned long long* out_offs, uint64_t n,
                                                   unsigned long long out_cap, const uint32_t* pos_in, uint32_t* out_words) {
    if (ctrl->overflow || ctrl->bad_offsets) return;  // (refused: out_offs was not written)
    const unsigned long long total = out_offs[n];
    if (total > out_cap) return;
    for (unsigned long long m = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; m < total;
         m += (unsigned long long)gridDim.x * blockDim.x) {
        uint64_t lo = 0, hi = n;  // largest h with out_offs[h] <= m
        while (lo + 1 < hi) {
            const uint64_t mid = (lo + hi) / 2;
            if (out_offs[mid] <= m)
                lo = mid;
            else
                hi = mid;
        }
        const uint32_t b = pos_in[lo];
        out_words[m * 3 + 0] += b;
        out_words[m * 3 + 1] += b;
    }
}

// L2 eviction policy descriptors (see c_l2pol in scan_lane.cuh): made once per device
__global__ void k_make_policies(unsigned long long* out, int hints) {
    unsigned long long normal, last, first;
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(normal));
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(last));
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(first));
    out[0] = hints ? last : normal;                     // automaton image
    out[1] = hints == 1 ? first : normal;               // haystack text
    out[2] = hints ? first : normal;                    // match blocks
}

// ---- shard groups: the exchange step over NVLink peer memory --------------------------------------
// Every rank owns one GroupCtl block in its HBM; peers write into it with system-scope releases and the owner
// polls it locally.  `step` numbers the exchange steps (1, 2, ...); slots alternate by step parity.
constexpr int kMaxRanks = 16;
struct GroupCtl {
    unsigned long long total[2][kMaxRanks];      // matches of rank j at the step named by total_seq
    unsigned long long total_seq[2][kMaxRanks];
    unsigned long long done_seq[kMaxRanks];      // gathering rank only: rank j's matches of that step have landed
    unsigned long long free_seq;                 // the gathering rank has released the result buffer of that step
    unsigned long long base[2];                  // this rank's first match index at the step (written locally)
    unsigned long long sum[2];                   // gathering rank: matches of all ranks at the step
    unsigned long long error;                    // a wait timed out
};
struct GroupPeers {
    GroupCtl* ctl[kMaxRanks];
};

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
constexpr unsigned long long kGroupTimeoutNs = 20ull * 1000 * 1000 * 1000;  // a peer that never arrives must not hang the GPU

// this rank's match count of the step goes to every rank's control block (exact past 2^32 matches per haystack:
// the carries of the per-item counts are added back, finish_scan)
__global__ void k_group_publish(GroupPeers peers, int world, int rank, unsigned long long step, const unsigned long long* total,
                                const ScanCtrl* ctrl) {
    const int j = threadIdx.x;
    if (j >= world) return;
    GroupCtl* c = peers.ctl[j];
    c->total[step & 1][rank] = *total + ((unsigned long long)ctrl->carries << 32);
    __threadfence_system();
    st_release_sys(&c->total_seq[step & 1][rank], step);
}
// base = matches of the lower ranks at this step; the result buffer of the previous step must have been released
__global__ void k_group_wait_base(GroupCtl* mine, int rank, unsigned long long step) {
    const unsigned long long t0 = global_ns();
    unsigned long long base = 0;
    for (int j = 0; j < rank; ++j) {
        while (ld_acquire_sys(&mine->total_seq[step & 1][j]) != step)
            if (global_ns() - t0 > kGroupTimeoutNs) {
                mine->error = 1;
                break;
            }
        base += mine->total[step & 1][j];
    }
    if (rank != 0)
        while (ld_acquire_sys(&mine->free_seq) + 1 < step)
            if (global_ns() - t0 > kGroupTimeoutNs) {
                mine->error = 1;
                break;
            }
    mine->base[step & 1] = base;
}
__global__ void k_group_signal_done(GroupCtl* gather_ctl, int rank, unsigned long long step) {
    __threadfence_system();
    st_release_sys(&gather_ctl->done_seq[rank], step);
}
// gathering rank: all ranks' matches of the step have landed in its buffers
__global__ void k_group_wait_all(GroupCtl* mine, int world, unsigned long long step) {
    const unsigned long long t0 = global_ns();
    unsigned long long sum = 0;
    for (int j = 0; j < world; ++j) {
        while (ld_acquire_sys(&mine->done_seq[j]) != step)
            if (global_ns() - t0 > kGroupTimeoutNs) {
                mine->error = 1;
                break;
            }
        sum += mine->total[step & 1][j];
    }
    mine->sum[step & 1] = sum;
}
// gathering rank: the result of `step` has been consumed, its buffers may be overwritten
__global__ void k_group_release(GroupPeers peers, int world, unsigned long long step) {
    const int j = threadIdx.x;
    if (j < world) st_release_sys(&peers.ctl[j]->free_seq, step);
}

// ---- offsets of a device-resident batch are the caller's: check them before anything indexes with them ----
// ascending, inside text_bytes, no haystack of 4 GiB or more (positions are u32).  A bad batch scans nothing
// (the item counter is pushed past every item) and the call reports DACH_INVALID_ARGUMENT.
__global__ void __launch_bounds__(256) k_check_offsets(const uint64_t* offs, uint64_t n, uint64_t text_bytes, ScanCtrl* ctrl) {
    const uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n) return;
    const uint64_t a = offs[h], b = offs[h + 1];
    if (b < a || b - a > 0xffffffffull || b > text_bytes) {
        ctrl->bad_offsets = 1u;
        ctrl->next_item = 1ull << 62;
    }
}

// ---- segment table (intra-haystack chunking for find_overlapping / no_suffix) --------------------
__global__ void __launch_bounds__(256) k_seg_count(const uint64_t* offs, uint64_t n, uint32_t seg_len, uint32_t seg_from,
                                                    uint32_t* nseg, const ScanCtrl* ctrl) {
    const uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n) return;
    const uint64_t len = ctrl->bad_offsets ? 0 : offs[h + 1] - offs[h];
    const uint64_t k = h < seg_from ? 1 : (len + seg_len - 1) / seg_len;
    nseg[h] = k ? (uint32_t)k : 1u;  // an empty haystack still is one item (ROOT's outputs at position 0)
}

__global__ void __launch_bounds__(256) k_seg_fill(const unsigned long long* seg_first, const uint32_t* nseg, uint64_t n,
                                                   uint32_t seg_len, uint32_t* item_hay, uint32_t* item_beg,
                                                   unsigned long long* n_items_dev) {
    const uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (h == 0) *n_items_dev = seg_first[n];
    if (h >= n) return;
    const unsigned long long first = seg_first[h];
    const uint32_t k = nseg[h];
    for (uint32_t j = 0; j < k; ++j) {
        item_hay[first + j] = (uint32_t)h;
        item_beg[first + j] = j * seg_len;
    }
}

// ---- COUNT / FIRST: per-haystack results from per-item results -----------------------------------------------
// The items of haystack h are [seg_first[h], seg_first[h + 1]) (nullptr: item h alone).  A haystack's count is the
// sum over its segments, its first match the one of its lowest segment that has one; the totals go to *total.
__device__ __forceinline__ void add_block_total(unsigned long long v, unsigned long long* total) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(total, v);
}

__global__ void __launch_bounds__(256) k_count_hay(const unsigned long long* seg_first, const unsigned long long* item_count, uint64_t n,
                                                    unsigned long long* counts, unsigned long long* total, const ScanCtrl* ctrl) {
    if (ctrl->bad_offsets) return;  // the call is refused: the caller's counts stay as they were
    const uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long v = 0;
    if (h < n) {
        const uint64_t lo = seg_first ? seg_first[h] : h, hi = seg_first ? seg_first[h + 1] : h + 1;
        for (uint64_t i = lo; i < hi; ++i) v += item_count[i];
        counts[h] = v;
    }
    add_block_total(v, total);
}

// ---- MASK: the text copied into the masked buffer before the scan fills its spans --------------------------------
// dst[i] = src[i] for i < bytes, at any alignment of src and dst to each other.  A thread writes one 16-byte-aligned chunk
// of dst with one 16-byte store, built from the two aligned 16-byte loads of src that cover it: the shift between them,
// (src - dst) mod 16, is the same for every chunk.  A chunk whose loads or store would reach outside the buffers (at
// most two at each end) goes byte by byte.  A refused call (bad offsets) writes nothing.
__device__ __forceinline__ uint32_t word_of(const uint4& x, const uint4& y, uint32_t i) {  // word i of the 32 bytes x, y
    const uint32_t lo = (i & 2u) ? ((i & 1u) ? x.w : x.z) : ((i & 1u) ? x.y : x.x);
    const uint32_t hi = (i & 2u) ? ((i & 1u) ? y.w : y.z) : ((i & 1u) ? y.y : y.x);
    return (i & 4u) ? hi : lo;
}
__global__ void __launch_bounds__(256) k_mask_copy(const uint8_t* src, uint8_t* dst, uint64_t bytes, const ScanCtrl* ctrl) {
    if (ctrl->bad_offsets) return;
    const uintptr_t s_lo = (uintptr_t)src, s_hi = s_lo + bytes, d_lo = (uintptr_t)dst, d_hi = d_lo + bytes;
    const uintptr_t d0 = d_lo & ~(uintptr_t)15, delta = s_lo - d_lo;  // source byte of dst byte q: q + delta (mod 2^64)
    const uint32_t sh = (uint32_t)delta & 15u, q = sh >> 2, r = (sh & 3u) * 8u;
    const uint64_t n_chunks = (d_hi - d0 + 15) >> 4;
    for (uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += (uint64_t)gridDim.x * blockDim.x) {
        const uintptr_t d = d0 + (c << 4), a = (d + delta) & ~(uintptr_t)15;
        if (d >= d_lo && d + 16 <= d_hi && a >= s_lo && a + (sh ? 32u : 16u) <= s_hi) {
            const uint4 x = __ldg(reinterpret_cast<const uint4*>(a));
            const uint4 y = sh ? __ldg(reinterpret_cast<const uint4*>(a + 16)) : x;
            uint4 o;
            o.x = __funnelshift_r(word_of(x, y, q), word_of(x, y, q + 1), r);
            o.y = __funnelshift_r(word_of(x, y, q + 1), word_of(x, y, q + 2), r);
            o.z = __funnelshift_r(word_of(x, y, q + 2), word_of(x, y, q + 3), r);
            o.w = __funnelshift_r(word_of(x, y, q + 3), word_of(x, y, q + 4), r);
            *reinterpret_cast<uint4*>(d) = o;
        } else {
            for (uintptr_t b = d; b < d + 16; ++b)
                if (b >= d_lo && b < d_hi) *reinterpret_cast<uint8_t*>(b) = *reinterpret_cast<const uint8_t*>(b + delta);
        }
    }
}

__global__ void __launch_bounds__(256) k_first_hay(const unsigned long long* seg_first, const uint4* item_first, uint64_t n,
                                                    uint32_t* first_words, uint8_t* found, unsigned long long* n_found,
                                                    const ScanCtrl* ctrl) {
    if (ctrl->bad_offsets) return;  // the call is refused: the caller's first / found stay as they were
    const uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long v = 0;
    if (h < n) {
        const uint64_t lo = seg_first ? seg_first[h] : h, hi = seg_first ? seg_first[h + 1] : h + 1;
        uint4 r = item_first[lo];
        for (uint64_t i = lo + 1; i < hi && !r.w; ++i) r = item_first[i];
        first_words[h * 3 + 0] = r.x;  // all-ones when there is no match (the sinks start that way)
        first_words[h * 3 + 1] = r.y;
        first_words[h * 3 + 2] = r.z;
        found[h] = r.w ? 1 : 0;
        v = r.w ? 1 : 0;
    }
    add_block_total(v, n_found);
}

// FIRST of stream chunks (one item per chunk, never segments): the item's answer, its start and end in stream
// coordinates -- plus pos[h], modulo 2^32, as k_add_base does for the matches -- or chunk-relative if pos is nullptr
__global__ void __launch_bounds__(256) k_first_stream(const uint4* item_first, uint64_t n, const uint32_t* pos, uint32_t* first_words,
                                                       uint8_t* found, unsigned long long* n_found, const ScanCtrl* ctrl) {
    if (ctrl->bad_offsets) return;  // the call is refused: the caller's first / found stay as they were
    const uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long v = 0;
    if (h < n) {
        const uint4 r = item_first[h];
        const uint32_t b = (r.w && pos) ? pos[h] : 0u;  // no match: the all-ones sentinel stays as it is
        first_words[h * 3 + 0] = r.x + b;
        first_words[h * 3 + 1] = r.y + b;
        first_words[h * 3 + 2] = r.z;
        found[h] = r.w ? 1 : 0;
        v = r.w ? 1 : 0;
    }
    add_block_total(v, n_found);
}

// ---- HIST: per-record counts from per-slot counts, then the caller's keys -------------------------------------------
// k_hist_heads   (lane machines) slot s counted events of its state: they go to the record that heads the state's
//                list (opos[s]).  Several slots may share a head.
// k_hist_fold    every record i with a count v: hist[key(j)] += v for j = i, and with CHAIN (find_overlapping on the
//                lane machines, where an event reports the whole list) for every record on i's parent chain too.
//                key(j) = j (output key) or value(j) (value key).  *total += the matches added.
__global__ void __launch_bounds__(256) k_hist_heads(const unsigned long long* slot_hist, const uint32_t* opos, uint32_t n_slots,
                                                     unsigned long long* rec_hist) {
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n_slots; s += gridDim.x * blockDim.x) {
        const unsigned long long v = slot_hist[s];
        const uint32_t op = v ? opos[s] : 0u;
        if (op) red_add_u64(rec_hist + (op - 1), v);
    }
}

template <bool CHAIN>
__global__ void __launch_bounds__(256) k_hist_fold(const unsigned long long* rec_hist, const uint4* outputs, uint32_t n_out, int key_value,
                                                    unsigned long long* hist, unsigned long long* total) {
    unsigned long long added = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_out; i += gridDim.x * blockDim.x) {
        const unsigned long long v = rec_hist[i];
        uint32_t j = v ? i + 1 : 0u;  // 1-based
        while (j) {
            const uint4 o = outputs[j - 1];
            red_add_u64(hist + (key_value ? o.x : j - 1), v);
            added += v;
            j = CHAIN ? o.z : 0u;
        }
    }
    add_block_total(added, total);
}

// ---- DF: the window's (haystack, key) pairs, then one per pair into the document frequencies ------------------------
// k_df_expand  (lane machines) every (haystack, slot) pair of the scan: the records its events reported -- the head
//              opos[slot], with CHAIN (find_overlapping) its whole parent chain, exactly what k_hist_fold<true> adds
//              to -- each mapped to its key and put into the key set as (haystack, key).
// k_df_add     df_acc[key] += 1 and *total += 1 per (haystack, key) pair of the window.
// Both do nothing once the window has overflowed (either set took more than df_pairs pairs), so df_acc only ever
// holds whole windows; k_df_clear then empties both sets for the next window by their lists.
template <bool CHAIN>
__global__ void __launch_bounds__(256) k_df_expand(ScanParams P) {
    const volatile unsigned int* over = &P.ctrl->overflow;
    if (*over) return;
    const unsigned int n = *P.df_slots.n;
    for (unsigned int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long pair = P.df_slots.keys[P.df_slots.list[i]];
        const unsigned long long hay = pair & 0xffffffff00000000ull;
        uint32_t j = P.opos_tab[(uint32_t)pair];
        while (j) {
            const uint4 o = P.outputs[j - 1];
            if (df_insert(P.df_keys, hay | (P.df_key_value ? o.x : j - 1), P.ctrl) == DF_FULL) return;
            j = CHAIN ? o.z : 0u;
        }
    }
}

__global__ void __launch_bounds__(256) k_df_add(DfSet keys, const ScanCtrl* ctrl, unsigned long long* df_acc, unsigned long long* total) {
    if (ctrl->overflow) return;
    const unsigned int n = *keys.n;
    if (blockIdx.x == 0 && threadIdx.x == 0) *total += n;
    for (unsigned int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        red_add_u64(df_acc + (uint32_t)keys.keys[keys.list[i]], 1);
}

__global__ void __launch_bounds__(256) k_df_clear(DfSet a, DfSet b) {
    const unsigned int na = *a.n, nb = *b.n;  // both at most mask + 1 (one list position per taken entry)
    for (unsigned int i = blockIdx.x * blockDim.x + threadIdx.x; i < na; i += gridDim.x * blockDim.x) a.keys[a.list[i]] = DF_EMPTY;
    for (unsigned int i = blockIdx.x * blockDim.x + threadIdx.x; i < nb; i += gridDim.x * blockDim.x) b.keys[b.list[i]] = DF_EMPTY;
}

// df[i] += acc[i]: a call's counts reach the caller's buffer only once all its windows are done
__global__ void __launch_bounds__(256) k_df_commit(const unsigned long long* acc, unsigned long long* df, uint64_t n) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) df[i] += acc[i];
}

}  // namespace dach

// ------------------------------------------------------------------------------------------
// device handle
// ------------------------------------------------------------------------------------------

using namespace dach;

namespace {

struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
};

bool cuda_ok(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return true;
    set_error(std::string(what) + ": " + cudaGetErrorString(e));
    return false;
}

bool ensure(DevBuf& b, size_t bytes) {
    if (b.bytes >= bytes && b.p) return true;
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.bytes = 0;
    const size_t want = std::max<size_t>(bytes, 256);
    if (!cuda_ok(cudaMalloc(&b.p, want), "cudaMalloc")) return false;
    b.bytes = want;
    return true;
}

struct HostPinned {
    unsigned long long total;
    ScanCtrl ctrl;
    unsigned long long tail_offs[2];
    unsigned long long total_rk;  // COUNT / FIRST: total count / haystacks with a match  // offs[seg_from], offs[n]: exact size of the segmented tail
};

// Everything one in-flight scan needs besides the automaton image.  A scan runs in two phases that may sit on
// different streams: enqueue_scan (items, scan kernel, offsets, block index) and enqueue_place (gather into the
// caller's -- possibly peer-mapped -- buffers); finish_scan waits for the second and reports.
struct Workspace {
    DevBuf counts, ev_counts, tiles, ctrl, pool;  // ev_counts: events per item (event blocks)
    DevBuf nseg, seg_first, item_hay, item_beg, item_offs, n_items_dev;  // segment table, per-item offsets
    DevBuf blk_first, blkmap, tiles2;  // pool blocks in output order (k_blk_index)
    DevBuf desc;                       // ... as block descriptors (k_blk_desc, event blocks)
    DevBuf stage;  // shard groups: the job's dense matches, pushed to the gathering rank by k_push
    DevBuf items_rk, total_rk;  // COUNT / FIRST: per-item results, the batch's total (u64)
    DevBuf slot_hist, rec_hist, hist_acc;  // HIST: per compact slot, per output record; host form: the batch's histogram
    HostPinned* pinned = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};  // pipeline start, scan end, pipeline end, scan start
    cudaEvent_t ev_scanned = nullptr, ev_placed = nullptr;
    cudaEvent_t ev_push[2] = {nullptr, nullptr};  // around k_push (shard groups)
    // the scan in flight (phase 1 -> phase 2)
    uint64_t job_n = 0, job_items = 0;
    uint32_t job_pool_blocks = 0;
    uint64_t job_cap = 0;
    bool job_seg = false, job_ordered = false, job_open = false, job_placed = false;
    bool job_events = false;
    bool job_desc = false;  // ordered event blocks with descriptors: k_expand_desc places them
    bool refused = false;  // finish_scan: a haystack passed 2^32 matches (*needed exact, status DACH_INVALID_ARGUMENT)
    int job_mode = 0;  // the pool holds event blocks (StdMachine3): k_expand places them, not k_gather
    cudaStream_t job_stream = nullptr;
    // host-batch slices only: device staging and the slice's stream
    DevBuf text, offs, out, out_offs;
    void* offs_stage = nullptr;  // pinned staging of the slice's offsets (the caller's array may be pageable)
    size_t offs_stage_bytes = 0;
    cudaStream_t stream = nullptr;
    bool init(bool with_stream) {
        if (!pinned && !cuda_ok(cudaMallocHost(reinterpret_cast<void**>(&pinned), sizeof(HostPinned)), "cudaMallocHost"))
            return false;
        for (int i = 0; i < 4; ++i)
            if (!ev[i] && !cuda_ok(cudaEventCreate(&ev[i]), "cudaEventCreate")) return false;
        if (!ev_scanned && !cuda_ok(cudaEventCreateWithFlags(&ev_scanned, cudaEventDisableTiming), "cudaEventCreate")) return false;
        if (!ev_placed && !cuda_ok(cudaEventCreateWithFlags(&ev_placed, cudaEventDisableTiming), "cudaEventCreate")) return false;
        for (int i = 0; i < 2; ++i)
            if (!ev_push[i] && !cuda_ok(cudaEventCreate(&ev_push[i]), "cudaEventCreate")) return false;
        if (with_stream && !stream && !cuda_ok(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking), "cudaStreamCreate"))
            return false;
        return true;
    }
    void release() {
        for (DevBuf* b : {&counts, &ev_counts, &tiles, &ctrl, &pool, &text, &offs, &out, &out_offs, &nseg, &seg_first, &item_hay, &item_beg,
                          &item_offs, &n_items_dev, &blk_first, &blkmap, &desc, &tiles2, &stage, &items_rk, &total_rk, &slot_hist, &rec_hist,
                          &hist_acc})
            if (b->p) {
                cudaFree(b->p);
                b->p = nullptr;
                b->bytes = 0;
            }
        if (pinned) cudaFreeHost(pinned);
        pinned = nullptr;
        if (offs_stage) cudaFreeHost(offs_stage);
        offs_stage = nullptr;
        offs_stage_bytes = 0;
        for (int i = 0; i < 4; ++i)
            if (ev[i]) {
                cudaEventDestroy(ev[i]);
                ev[i] = nullptr;
            }
        for (int i = 0; i < 2; ++i)
            if (ev_push[i]) {
                cudaEventDestroy(ev_push[i]);
                ev_push[i] = nullptr;
            }
        if (ev_scanned) cudaEventDestroy(ev_scanned);
        if (ev_placed) cudaEventDestroy(ev_placed);
        ev_scanned = ev_placed = nullptr;
        if (stream) cudaStreamDestroy(stream);
        stream = nullptr;
    }
};

}  // namespace

struct dach_dev {
    int device = 0;
    bool charwise = false;
    uint8_t match_kind = 0;
    uint32_t n_slots = 0, root_opos = 0, mapper_len = 0, max_pattern_len = 0;
    bool segmentable = false;  // HostImage::segmentable: long haystacks may be cut into segments
    uint32_t n_outputs = 0, max_value = 0, n_cslots = 0;  // output records, their largest value, compact slots
    size_t image_bytes = 0;
    int sm_count = 0;
    size_t smem_optin = 0;
    // image
    uint4* d_rec = nullptr;
    uint4* d_outputs = nullptr;
    uint32_t* d_root = nullptr;
    uint4* d_crec = nullptr;
    uint32_t* d_opos = nullptr;
    uint4* d_pairs = nullptr;  // two-entry output lists (nullptr: a pattern length reaches PAIR_CLASS_SHIFT)
    uint32_t* d_id_in = nullptr;   // crate slot -> compact slot (stream chunks)
    uint32_t* d_id_out = nullptr;  // compact slot -> crate slot
    uint32_t hot_slots = 0;        // size of the hot region of the compact image
    uint32_t root_base = 0;
    uint32_t* d_mapper = nullptr;
    void* image_base = nullptr;
    size_t image_alloc = 0;
    // workspaces (guarded by mu; dach_job handles own theirs)
    std::mutex mu;
    Workspace ws;        // dach_dev_scan_batch
    static constexpr int kSlots = 4;
    Workspace slot[kSlots];  // dach_scan_batch_host: slices in flight (H2D of k+1 and k+2 | scan of k | D2H of k-1)
    // ---- options (dach_dev_set_option) ----
    int64_t opt_slice_mib = 64;
    // Records of the hot region staged in shared memory by StdMachine3 (the region is laid out hottest first, so
    // any prefix is the best set of its size).  Staged records take fetches off L1 and L2 up to the point where the
    // total of shared memory crosses the 196 KiB carveout step and L1 shrinks (DESIGN.md section 4.1).
    // kHotAuto: kHotQueued beside the event queues, as many as kDirectSmemBudget holds in k_scan_direct.
    // 0 = off, -1 = as many as fit (next to the event queues, if any).
    int64_t opt_hot_entries = kHotAuto;
    // StdMachine3's matches path: 0 = events stored at their landing (k_scan_direct) when the scan runs one CTA per
    // SM, 1 = through the per-lane event queue (scan_machine with EventOps)
    int64_t opt_event_queue = 0;
    int64_t opt_expand_desc = 1;  // ordered event blocks: 1 = k_expand_desc (descriptors, pairs), 0 = k_expand
    int64_t opt_expand_u = 2;     // blocks in flight per warp of k_expand_desc (2, 4 or 8); 2: 60 registers, fits beside a scan CTA
    // HIST on the lane machines: events of the leading compact slots are counted in shared memory per CTA (4 B
    // each, next to the hot records and the queues) before they reach global memory.  0 = off.
    int64_t opt_hist_smem = 1024;
    // DF: the most (haystack, state) and (haystack, key) pairs one window may hold; both sets take the next power of
    // two at or above twice that many entries, 12 B each.  At least max(compact slots, output records), so that one
    // haystack always fits.  The default: kDefaultDfPairs.
    int64_t opt_df_pairs = kDefaultDfPairs;
    int64_t opt_slice_ramp = 1;     // host path: small slices at the head and the tail of a batch
    int64_t opt_tail_seg = 0;        // cut only the last 2 x lanes haystacks of a large batch (off by default)
    int64_t opt_gather_ordered = 1;  // copy pool blocks in output order (sequential writes)
    int64_t opt_gather_u = 4;     // pooled blocks in flight per warp of k_gather (2, 4 or 8)
    int64_t opt_reserve_sms = 0;  // SMs left free for concurrent kernels
    int64_t opt_smem_pad_kib = 0;  // lane machines: extra dynamic shared memory per CTA, i.e. that much less L1 (experiments)
    int64_t opt_seg_len = 0;  // 0: automatic; > 0: forced segment length; < 0: no segmentation
    int64_t opt_hot_records = 0;  // lane-per-haystack kernels: leading wide records staged in shared memory (-1 = as many as fit)
    int64_t opt_threads = 1024;
    int64_t opt_ctas_per_sm = 1;
    int64_t opt_l2_hints = 2;  // L2 eviction policies: 2 = image evict_last, match blocks evict_first, text normal; 1 = text
                               // evict_first too; 0 = none
    int64_t opt_kernel = 3;  // 3: lane machines, StdMachine3 for the bytewise Standard iterators; 4: StdMachine3 with two
                             // haystacks per lane; 2: StdMachine2 instead; 1: StdMachine instead; 0: always the
                             // lane-per-haystack kernels
    // stats
    std::atomic<uint64_t> launches{0};
    cudaEvent_t ev_ref = nullptr;  // time zero of dach_job_times (recorded at the handle's first job operation)
    std::mutex ev_ref_mu;           // ... set under this lock, not d->mu: a job never waits for a synchronous call
    double last_scan_ms = 0, last_total_ms = 0;
    uint64_t last_h2d = 0, last_d2h = 0;
    // DF (dach_dev_df_batch / dach_df_batch_host, both under mu): the two pair sets, shared by every window of both
    // forms -- each window is finished before the next is enqueued -- and the call's document frequencies
    DevBuf df_tab[2], df_list[2], df_n, df_acc;
    uint32_t df_mask = 0, df_limit = 0;
    bool df_clean = false;  // both sets are empty (false after a failed window: the next call empties them in full)
    uint64_t last_df_windows = 0, last_df_rescans = 0;
    // the handle's owner plus one per live job: dach_dev_free may come before the jobs are freed (a garbage collector
    // finalises in any order), and the jobs still read the image and d->device until then
    std::atomic<int> refs{1};
};

// one asynchronous scan with its own workspace (dach_job_*)
struct dach_job {
    dach_dev* d = nullptr;
    Workspace W;
    uint64_t out_cap = ~0ull;  // capacity the placement was given (for the overflow report)
    // the job's last operation, which dach_job_wait reports: RK_MATCHES (dach_job_scan, then dach_job_place or
    // dach_group_place), or RK_COUNT / RK_FIRST / RK_HIST / RK_MASK (dach_job_count ... dach_job_mask)
    int rk = RK_MATCHES;
    bool unplaced = false;  // a dach_job_scan whose placement has not been enqueued: a reduction may not reuse its buffers
};

namespace {

struct DeviceGuard {
    int prev = -1;
    bool ok = false;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        ok = cuda_ok(cudaSetDevice(dev), "cudaSetDevice");
        if (!ok) cudaGetLastError();  // reported here; it must not resurface as the error of a later, unrelated launch
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

template <bool CW, int MODE>
cudaError_t launch_scan_t(const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    static bool attr_done[kMaxDevices] = {};  // per instantiation and per device (the attribute is per device)
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= kMaxDevices || !attr_done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(k_scan<CW, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < kMaxDevices) attr_done[dev] = true;
    }
    k_scan<CW, MODE><<<grid, threads, smem, st>>>(P);
    return cudaGetLastError();
}

template <class M, class LANE, int MAXT, int MINB, bool HOT>
cudaError_t launch_machine_t(const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    static bool attr_done[kMaxDevices] = {};  // per instantiation and per device
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= kMaxDevices || !attr_done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(k_scan_machine<M, LANE, MAXT, MINB, HOT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < kMaxDevices) attr_done[dev] = true;
    }
    k_scan_machine<M, LANE, MAXT, MINB, HOT><<<grid, threads, smem, st>>>(P);
    return cudaGetLastError();
}

template <template <int> class M, class LANE, int MAXT, int MINB, bool HOT>
cudaError_t launch_std_modes(int mode, const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    switch (mode) {
        case M_FIND: return launch_machine_t<M<M_FIND>, LANE, MAXT, MINB, HOT>(P, grid, threads, smem, st);
        case M_NO_SUFFIX: return launch_machine_t<M<M_NO_SUFFIX>, LANE, MAXT, MINB, HOT>(P, grid, threads, smem, st);
        case M_OVERLAPPING: return launch_machine_t<M<M_OVERLAPPING>, LANE, MAXT, MINB, HOT>(P, grid, threads, smem, st);
    }
    return cudaErrorInvalidValue;
}

// bytewise Standard iterators: which = 3 StdMachine3 (hot records in shared memory if P.hot_entries), 2 StdMachine2,
// 1 StdMachine; dense = two CTAs of up to 768 threads per SM (40 registers) instead of one of 1024
cudaError_t launch_std(int which, int mode, const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st,
                       bool dense) {
    if (which >= 3) {
        if (P.hot_entries)
            return dense ? launch_std_modes<StdMachine3, Lane3, 768, 2, true>(mode, P, grid, threads, smem, st)
                         : launch_std_modes<StdMachine3, Lane3, 1024, 1, true>(mode, P, grid, threads, smem, st);
        return dense ? launch_std_modes<StdMachine3, Lane3, 768, 2, false>(mode, P, grid, threads, smem, st)
                     : launch_std_modes<StdMachine3, Lane3, 1024, 1, false>(mode, P, grid, threads, smem, st);
    }
    if (which == 2)
        return dense ? launch_std_modes<StdMachine2, Lane2, 768, 2, false>(mode, P, grid, threads, smem, st)
                     : launch_std_modes<StdMachine2, Lane2, 1024, 1, false>(mode, P, grid, threads, smem, st);
    return dense ? launch_std_modes<StdMachine, LaneStd, 768, 2, false>(mode, P, grid, threads, smem, st)
                 : launch_std_modes<StdMachine, LaneStd, 1024, 1, false>(mode, P, grid, threads, smem, st);
}

template <int MODE, int MAXT, bool HOT>
cudaError_t launch_duo_t(const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    static bool attr_done[kMaxDevices] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= kMaxDevices || !attr_done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(k_scan_duo<MODE, MAXT, HOT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < kMaxDevices) attr_done[dev] = true;
    }
    k_scan_duo<MODE, MAXT, HOT><<<grid, threads, smem, st>>>(P);
    return cudaGetLastError();
}
template <int MAXT, bool HOT>
cudaError_t launch_duo_m(int mode, const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    switch (mode) {
        case M_FIND: return launch_duo_t<M_FIND, MAXT, HOT>(P, grid, threads, smem, st);
        case M_NO_SUFFIX: return launch_duo_t<M_NO_SUFFIX, MAXT, HOT>(P, grid, threads, smem, st);
        case M_OVERLAPPING: return launch_duo_t<M_OVERLAPPING, MAXT, HOT>(P, grid, threads, smem, st);
    }
    return cudaErrorInvalidValue;
}
// two haystacks per lane (option kernel = 4): 1024 threads (64 registers) or up to 768 (85 registers)
cudaError_t launch_duo(int mode, const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    if (threads > 768)
        return P.hot_entries ? launch_duo_m<1024, true>(mode, P, grid, threads, smem, st) : launch_duo_m<1024, false>(mode, P, grid, threads, smem, st);
    return P.hot_entries ? launch_duo_m<768, true>(mode, P, grid, threads, smem, st) : launch_duo_m<768, false>(mode, P, grid, threads, smem, st);
}

template <int MODE, bool HOT>
cudaError_t launch_direct_t(const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    static bool attr_done[kMaxDevices] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= kMaxDevices || !attr_done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(k_scan_direct<MODE, HOT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
        // the smallest carveout that holds kDirectSmemBudget: L1 keeps what it has beside the queue kernel
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(k_scan_direct<MODE, HOT>, cudaFuncAttributePreferredSharedMemoryCarveout, kDirectCarveoutPct);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < kMaxDevices) attr_done[dev] = true;
    }
    k_scan_direct<MODE, HOT><<<grid, threads, smem, st>>>(P);
    return cudaGetLastError();
}
// StdMachine3's matches path without the queue (option event_queue = 0, one CTA per SM)
cudaError_t launch_direct(int mode, const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    switch (mode) {
        case M_FIND:
            return P.hot_entries ? launch_direct_t<M_FIND, true>(P, grid, threads, smem, st) : launch_direct_t<M_FIND, false>(P, grid, threads, smem, st);
        case M_NO_SUFFIX:
            return P.hot_entries ? launch_direct_t<M_NO_SUFFIX, true>(P, grid, threads, smem, st)
                                 : launch_direct_t<M_NO_SUFFIX, false>(P, grid, threads, smem, st);
        case M_OVERLAPPING:
            return P.hot_entries ? launch_direct_t<M_OVERLAPPING, true>(P, grid, threads, smem, st)
                                 : launch_direct_t<M_OVERLAPPING, false>(P, grid, threads, smem, st);
    }
    return cudaErrorInvalidValue;
}

cudaError_t launch_cw(int mode, const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    switch (mode) {
        case M_FIND: return launch_machine_t<CwMachine<M_FIND>, LaneCw, 1024, 1, false>(P, grid, threads, smem, st);
        case M_OVERLAPPING: return launch_machine_t<CwMachine<M_OVERLAPPING>, LaneCw, 1024, 1, false>(P, grid, threads, smem, st);
        case M_NO_SUFFIX: return launch_machine_t<CwMachine<M_NO_SUFFIX>, LaneCw, 1024, 1, false>(P, grid, threads, smem, st);
        default: return launch_machine_t<CwMachine<M_LEFTMOST>, LaneCw, 1024, 1, false>(P, grid, threads, smem, st);
    }
}

cudaError_t launch_lm(const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    return launch_machine_t<LmMachine, LaneLm, 1024, 1, false>(P, grid, threads, smem, st);
}

cudaError_t launch_scan(bool cw, int mode, const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    switch ((cw ? 4 : 0) + mode) {
        case 0: return launch_scan_t<false, M_FIND>(P, grid, threads, smem, st);
        case 1: return launch_scan_t<false, M_OVERLAPPING>(P, grid, threads, smem, st);
        case 2: return launch_scan_t<false, M_NO_SUFFIX>(P, grid, threads, smem, st);
        case 3: return launch_scan_t<false, M_LEFTMOST>(P, grid, threads, smem, st);
        case 4: return launch_scan_t<true, M_FIND>(P, grid, threads, smem, st);
        case 5: return launch_scan_t<true, M_OVERLAPPING>(P, grid, threads, smem, st);
        case 6: return launch_scan_t<true, M_NO_SUFFIX>(P, grid, threads, smem, st);
        case 7: return launch_scan_t<true, M_LEFTMOST>(P, grid, threads, smem, st);
    }
    return cudaErrorInvalidValue;
}

// ---- COUNT / FIRST launchers: StdMachine3, LmMachine, CwMachine, or the lane-per-haystack kernels --------------
template <class M, class LANE, int MODE, int RK, bool HOT>
cudaError_t launch_rk_t(const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    static bool attr_done[kMaxDevices] = {};  // per instantiation and per device
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= kMaxDevices || !attr_done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(k_scan_machine_rk<M, LANE, MODE, RK, HOT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < kMaxDevices) attr_done[dev] = true;
    }
    k_scan_machine_rk<M, LANE, MODE, RK, HOT><<<grid, threads, smem, st>>>(P);
    return cudaGetLastError();
}
template <bool CW, int MODE, int RK>
cudaError_t launch_scan_rk_t(const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    static bool attr_done[kMaxDevices] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= kMaxDevices || !attr_done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(k_scan_rk<CW, MODE, RK>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < kMaxDevices) attr_done[dev] = true;
    }
    k_scan_rk<CW, MODE, RK><<<grid, threads, smem, st>>>(P);
    return cudaGetLastError();
}

// which: 3 StdMachine3 (bytewise Standard), 1 LmMachine / CwMachine (by the automaton), 0 lane per haystack.
// FIRST only runs M_OVERLAPPING (Standard) and M_LEFTMOST: the caller folds the Standard modes.  HIST and DF run all
// of COUNT's kernels.
template <int RK>
cudaError_t launch_rk(int which, bool cw, int mode, const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    if (which == 3) {
        switch (mode) {
            case M_FIND:
                if constexpr (RK != RK_FIRST)
                    return P.hot_entries ? launch_rk_t<StdMachine3<M_FIND>, Lane3, M_FIND, RK, true>(P, grid, threads, smem, st)
                                         : launch_rk_t<StdMachine3<M_FIND>, Lane3, M_FIND, RK, false>(P, grid, threads, smem, st);
                break;
            case M_NO_SUFFIX:
                if constexpr (RK != RK_FIRST)
                    return P.hot_entries ? launch_rk_t<StdMachine3<M_NO_SUFFIX>, Lane3, M_NO_SUFFIX, RK, true>(P, grid, threads, smem, st)
                                         : launch_rk_t<StdMachine3<M_NO_SUFFIX>, Lane3, M_NO_SUFFIX, RK, false>(P, grid, threads, smem, st);
                break;
            case M_OVERLAPPING:
                return P.hot_entries ? launch_rk_t<StdMachine3<M_OVERLAPPING>, Lane3, M_OVERLAPPING, RK, true>(P, grid, threads, smem, st)
                                     : launch_rk_t<StdMachine3<M_OVERLAPPING>, Lane3, M_OVERLAPPING, RK, false>(P, grid, threads, smem, st);
        }
        return cudaErrorInvalidValue;
    }
    if (which == 1 && cw) {
        switch (mode) {
            case M_FIND:
                if constexpr (RK != RK_FIRST) return launch_rk_t<CwMachine<M_FIND>, LaneCw, M_FIND, RK, false>(P, grid, threads, smem, st);
                break;
            case M_NO_SUFFIX:
                if constexpr (RK != RK_FIRST) return launch_rk_t<CwMachine<M_NO_SUFFIX>, LaneCw, M_NO_SUFFIX, RK, false>(P, grid, threads, smem, st);
                break;
            case M_OVERLAPPING: return launch_rk_t<CwMachine<M_OVERLAPPING>, LaneCw, M_OVERLAPPING, RK, false>(P, grid, threads, smem, st);
            case M_LEFTMOST: return launch_rk_t<CwMachine<M_LEFTMOST>, LaneCw, M_LEFTMOST, RK, false>(P, grid, threads, smem, st);
        }
        return cudaErrorInvalidValue;
    }
    if (which == 1) return mode == M_LEFTMOST ? launch_rk_t<LmMachine, LaneLm, M_LEFTMOST, RK, false>(P, grid, threads, smem, st) : cudaErrorInvalidValue;
    switch ((cw ? 4 : 0) + mode) {
        case 0: if constexpr (RK != RK_FIRST) return launch_scan_rk_t<false, M_FIND, RK>(P, grid, threads, smem, st); break;
        case 1: return launch_scan_rk_t<false, M_OVERLAPPING, RK>(P, grid, threads, smem, st);
        case 2: if constexpr (RK != RK_FIRST) return launch_scan_rk_t<false, M_NO_SUFFIX, RK>(P, grid, threads, smem, st); break;
        case 3: return launch_scan_rk_t<false, M_LEFTMOST, RK>(P, grid, threads, smem, st);
        case 4: if constexpr (RK != RK_FIRST) return launch_scan_rk_t<true, M_FIND, RK>(P, grid, threads, smem, st); break;
        case 5: return launch_scan_rk_t<true, M_OVERLAPPING, RK>(P, grid, threads, smem, st);
        case 6: if constexpr (RK != RK_FIRST) return launch_scan_rk_t<true, M_NO_SUFFIX, RK>(P, grid, threads, smem, st); break;
        case 7: return launch_scan_rk_t<true, M_LEFTMOST, RK>(P, grid, threads, smem, st);
    }
    return cudaErrorInvalidValue;
}

// FIRST of stream chunks: the caller's iterator (find / find_overlapping) on StdMachine3 or CwMachine
cudaError_t launch_first_stream(bool cw, int mode, const ScanParams& P, int grid, int threads, size_t smem, cudaStream_t st) {
    constexpr int R = RK_FIRST_STREAM;
    if (cw)
        return mode == M_FIND ? launch_rk_t<CwMachine<M_FIND>, LaneCw, M_FIND, R, false>(P, grid, threads, smem, st)
                              : launch_rk_t<CwMachine<M_OVERLAPPING>, LaneCw, M_OVERLAPPING, R, false>(P, grid, threads, smem, st);
    if (mode == M_FIND)
        return P.hot_entries ? launch_rk_t<StdMachine3<M_FIND>, Lane3, M_FIND, R, true>(P, grid, threads, smem, st)
                             : launch_rk_t<StdMachine3<M_FIND>, Lane3, M_FIND, R, false>(P, grid, threads, smem, st);
    return P.hot_entries ? launch_rk_t<StdMachine3<M_OVERLAPPING>, Lane3, M_OVERLAPPING, R, true>(P, grid, threads, smem, st)
                         : launch_rk_t<StdMachine3<M_OVERLAPPING>, Lane3, M_OVERLAPPING, R, false>(P, grid, threads, smem, st);
}

int check_mode(const dach_dev* d, int mode) {
    if (mode < DACH_FIND || mode > DACH_LEFTMOST_FIND) {
        set_error("unknown scan mode");
        return DACH_INVALID_ARGUMENT;
    }
    const bool lm = is_leftmost(d->match_kind);
    if ((mode == DACH_LEFTMOST_FIND) != lm) {
        set_error(lm ? "Error: match_kind must be standard." : "Error: match_kind must be leftmost.");
        return DACH_MATCH_KIND_MISMATCH;
    }
    return DACH_OK;
}

// L2 policy descriptors of this device (c_l2pol): made by a one-thread kernel, kept in constant memory
bool install_policies(int hints) {
    unsigned long long* d_pol = nullptr;
    unsigned long long h_pol[3] = {0, 0, 0};
    if (!cuda_ok(cudaMalloc(reinterpret_cast<void**>(&d_pol), 24), "cudaMalloc policies")) return false;
    k_make_policies<<<1, 1>>>(d_pol, hints);
    bool ok = cuda_ok(cudaMemcpy(h_pol, d_pol, 24, cudaMemcpyDeviceToHost), "read policies");
    cudaFree(d_pol);
    return ok && cuda_ok(cudaMemcpyToSymbol(c_l2pol, h_pol, 24), "install policies");
}

// the automaton image and the batch of a scan's ScanParams (results, options and the segment table are set by the caller)
ScanParams image_params(const dach_dev* d, const uint8_t* d_text, const uint8_t* text_lo, const uint8_t* text_end,
                        const uint64_t* d_offs, uint64_t n) {
    ScanParams P;
    memset(&P, 0, sizeof(P));
    P.rec = d->d_rec;
    P.outputs = d->d_outputs;
    P.root_table = d->d_root;
    P.crec = d->d_crec;
    P.opos_tab = d->d_opos;
    P.root_base = d->root_base;
    P.mapper = d->d_mapper;
    P.mapper_len = d->mapper_len;
    P.n_slots = d->n_slots;
    P.id_in = d->d_id_in;
    P.id_out = d->d_id_out;
    P.root_opos = d->root_opos;
    P.text = d_text;
    P.text_lo = text_lo;
    P.text_end = text_end;
    P.offs = d_offs;
    P.n_items = n;
    return P;
}

// dynamic shared memory of the scan kernel: the lane machines' event queues (queue_sets per lane; 0 for
// k_scan_direct) and, for StdMachine3, the front of the hot region; the lane-per-haystack kernels stage leading wide
// records
size_t plan_smem(const dach_dev* d, ScanParams& P, bool v1, bool std3, int threads, int ctas_per_sm, int queue_sets,
                 uint32_t hist_smem = 0) {
    const size_t smem_budget = std::min<size_t>(d->smem_optin, 226 * 1024) / ctas_per_sm - (ctas_per_sm > 1 ? 1024 : 0);
    size_t smem;
    if (v1) {
        // HIST: hist_smem u32 counters behind the queues (counted with them: they come before the hot records)
        const size_t queues = (size_t)LANE_Q * threads * sizeof(QEntry) * queue_sets + (size_t)hist_smem * 4;
        // StdMachine3: the front of the hot region next to the queues (whole 256-slot blocks)
        uint64_t want = 0;
        if (std3 && d->opt_hot_entries != 0 && smem_budget > queues + 512) {
            want = std::min<uint64_t>(d->hot_slots, (smem_budget - queues - 512) / 16);
            const int64_t hot = d->opt_hot_entries != kHotAuto ? d->opt_hot_entries : queue_sets ? kHotQueued : kDirectSmemBudget / 16;
            if (hot > 0) want = std::min<uint64_t>(want, (uint64_t)hot);
            want &= ~uint64_t(255);
        }
        smem = (size_t)want * 16 + queues;
        if (d->opt_smem_pad_kib > 0) smem = std::min<size_t>(smem + ((size_t)d->opt_smem_pad_kib << 10), smem_budget);
        P.hot_n = 0;
        P.hot_entries = (uint32_t)want;
    } else {
        uint64_t hot = smem_budget > kRootBytes ? (smem_budget - kRootBytes) / 16 : 0;
        if (d->opt_hot_records >= 0) hot = std::min<uint64_t>(hot, (uint64_t)d->opt_hot_records);
        hot = std::min<uint64_t>(hot, d->n_slots);
        P.hot_n = (uint32_t)hot;
        smem = kRootBytes + (size_t)hot * 16;
    }
    return smem;
}

// segment table: counts per haystack -> first item per haystack (W.seg_first) -> (haystack, begin) per item
void enqueue_seg_table(dach_dev* d, Workspace& W, const uint64_t* d_offs, uint64_t n, uint32_t seg_len, uint32_t seg_from,
                       ScanParams& P, cudaStream_t st) {
    unsigned long long* tiles = static_cast<unsigned long long*>(W.tiles.p);
    unsigned long long* seg_first = static_cast<unsigned long long*>(W.seg_first.p);
    const unsigned hb = (unsigned)((n + 255) / 256), hb1 = (unsigned)((n + 1 + 255) / 256);
    const uint64_t nt = (n + kScanTile - 1) / kScanTile;
    uint32_t* nseg = static_cast<uint32_t*>(W.nseg.p);
    k_seg_count<<<hb, 256, 0, st>>>(d_offs, n, seg_len, seg_from, nseg, P.ctrl);
    k_offsets_tile_sums<1><<<(unsigned)nt, kScanThreads, 0, st>>>(nseg, n, tiles);
    k_offsets_scan_tiles<<<1, kScanThreads, 0, st>>>(tiles, nt);
    k_offsets_apply<1><<<(unsigned)nt, kScanThreads, 0, st>>>(nseg, n, tiles, seg_first);
    k_seg_fill<<<hb1, 256, 0, st>>>(seg_first, nseg, n, seg_len, static_cast<uint32_t*>(W.item_hay.p),
                                    static_cast<uint32_t*>(W.item_beg.p), static_cast<unsigned long long*>(W.n_items_dev.p));
    d->launches += 5;
    P.item_hay = static_cast<const uint32_t*>(W.item_hay.p);
    P.item_beg = static_cast<const uint32_t*>(W.item_beg.p);
    P.n_items_dev = static_cast<const unsigned long long*>(W.n_items_dev.p);
    P.seg_len = seg_len;
    P.seg_from = seg_from;
    P.warm = d->max_pattern_len ? d->max_pattern_len - 1 : 0;
}

// ---- phase 1: items, scan kernel, per-item offsets, block index.  No synchronisation. ------------------
// d_text + d_offs[i] addresses haystack i; [text_lo, text_end) bounds what may be read; text_bytes is the
// number of text bytes this call covers (sizing only); cap_matches sizes the block pool.
int enqueue_scan(dach_dev* d, Workspace& W, int mode, const uint8_t* d_text, const uint8_t* text_lo, const uint8_t* text_end,
                 uint64_t text_bytes, const uint64_t* d_offs, uint64_t n, uint64_t cap_matches, cudaStream_t st,
                 uint32_t* d_state_io = nullptr) {
    W.refused = false;
    if (n > 0xfffffff0ull) {
        set_error("too many haystacks in one batch (max 2^32-16)");
        return DACH_INVALID_ARGUMENT;
    }
    // the previous placement out of this workspace (possibly on another stream) must be done before its
    // buffers are rewritten
    if (W.job_open) cudaStreamWaitEvent(st, W.ev_placed, 0);
    W.job_n = n;
    W.job_cap = cap_matches;
    W.job_items = n;
    W.job_seg = false;
    W.job_ordered = false;
    W.job_events = false;
    W.job_desc = false;
    W.job_stream = st;
    W.job_open = true;
    if (!ensure(W.ctrl, sizeof(ScanCtrl)) || !ensure(W.item_offs, 16)) return DACH_CUDA_ERROR;
    if (!cuda_ok(cudaMemsetAsync(W.ctrl.p, 0, sizeof(ScanCtrl), st), "memset ctrl")) return DACH_CUDA_ERROR;
    cudaEventRecord(W.ev[0], st);
    cudaEventRecord(W.ev[3], st);
    if (n == 0) {
        cudaMemsetAsync(W.item_offs.p, 0, 8, st);
        cudaEventRecord(W.ev[1], st);
        cudaEventRecord(W.ev_scanned, st);
        return DACH_OK;
    }
    int threads = (int)std::min<int64_t>(std::max<int64_t>(d->opt_threads, 32), kMaxThreads);
    threads = (threads / 32) * 32;
    int ctas_per_sm = (int)std::min<int64_t>(std::max<int64_t>(d->opt_ctas_per_sm, 1), 2048 / threads);
    const int free_sms = (int)std::min<int64_t>(std::max<int64_t>(d->opt_reserve_sms, 0), d->sm_count - 1);
    const int grid = (d->sm_count - free_sms) * ctas_per_sm;
    // the lane machines serve every iterator of both automata except find_iter with an empty pattern
    // (it only reports zero-length matches, src/bytewise/iter.rs:60-85), which keeps the simple kernel
    const bool v1 = d->opt_kernel >= 1 && d->d_crec && !(mode == M_FIND && d->root_opos != 0);
    const bool cw_machine = v1 && d->charwise;
    const bool lm_machine = v1 && !d->charwise && mode == M_LEFTMOST;
    // StdMachine2 / StdMachine3 keep ROOT's record in registers and probe it like any state: needs BASE(ROOT) != 0
    const bool std2 = v1 && !d->charwise && mode != M_LEFTMOST && d->opt_kernel >= 2 && d->root_base != 0;
    const bool std3 = std2 && d->opt_kernel >= 3;
    const bool duo = std3 && d->opt_kernel >= 4 && ctas_per_sm == 1;
    const bool events = std3 && !duo;  // StdMachine3's matches path stores events (k_scan_machine / k_scan_direct)
    // ... at their landing, without the queue: one CTA per SM, whose shared memory the staged records fill
    const bool direct = events && ctas_per_sm == 1 && d->opt_event_queue == 0;

    if (d_state_io && !std2 && !cw_machine) {
        set_error("stream chunks need a Standard lane machine (find / find_overlapping, at most 2^24 states, bytewise: "
                  "BASE(ROOT) != 0, no empty pattern for find)");
        return DACH_INVALID_ARGUMENT;
    }

    // Work items.  find_overlapping / no_suffix may cut haystacks into segments (exact with an
    // (L-1)-byte warm-up, SURVEY.md Appendix C.1) so that small batches and long haystacks still
    // fill the machine; everything else works on whole haystacks.
    // (a chunk of a stream resumes in a given state: it stays one item)
    bool seg = v1 && !d->charwise && !d_state_io && (mode == M_OVERLAPPING || mode == M_NO_SUFFIX) && d->opt_seg_len >= 0 && d->segmentable;
    uint32_t seg_len = 0, seg_from = 0;
    uint64_t n_items_max = n;
    if (seg) {
        const uint64_t lanes = (uint64_t)grid * threads;
        const uint64_t warm = d->max_pattern_len ? d->max_pattern_len - 1 : 0;
        const uint64_t floor_len = std::max<uint64_t>(256, 8 * warm);  // warm-up overhead <= 1/8
        uint64_t want;
        uint64_t tail_bytes = text_bytes;
        if (d->opt_seg_len > 0) {
            want = (uint64_t)d->opt_seg_len;
        } else if (d->opt_tail_seg && n >= 4 * lanes && n < 0xffffffffull) {
            // plenty of haystacks per lane: only the tail of the batch is cut, so that lanes that finish
            // early find short items instead of idling through the last wave
            const uint64_t n_tail = 2 * lanes;
            seg_from = (uint32_t)(n - n_tail);
            want = std::max(text_bytes / n / 8 + 1, floor_len);
            // the item tables are sized from the exact byte count of the tail (two 8-byte reads)
            cudaMemcpyAsync(&W.pinned->tail_offs[0], d_offs + seg_from, 8, cudaMemcpyDeviceToHost, st);
            cudaMemcpyAsync(&W.pinned->tail_offs[1], d_offs + n, 8, cudaMemcpyDeviceToHost, st);
            if (!cuda_ok(cudaStreamSynchronize(st), "read tail size")) return DACH_CUDA_ERROR;
            tail_bytes = W.pinned->tail_offs[1] - W.pinned->tail_offs[0];
        } else {
            want = std::max(text_bytes / (2 * lanes) + 1, floor_len);  // ~2 items per lane
        }
        want = (want + 255) & ~uint64_t(255);
        if (want >= text_bytes || want >= (1ull << 31)) {
            seg = false;  // every haystack fits one segment
        } else {
            seg_len = (uint32_t)want;
            n_items_max = n + tail_bytes / seg_len + 1;
            if (n_items_max > 0xfffffff0ull) seg = false, n_items_max = n;
        }
    }
    const uint64_t n_tiles = (n_items_max + kScanTile - 1) / kScanTile;
    uint64_t pool_blocks64 = cap_matches / BLK_MATCHES + n_items_max + 1024;
    if (pool_blocks64 > 0xffffff00ull) pool_blocks64 = 0xffffff00ull;
    const uint32_t pool_blocks = (uint32_t)pool_blocks64;
    if (!ensure(W.counts, n_items_max * 4) || !ensure(W.tiles, n_tiles * 8) || !ensure(W.item_offs, (n_items_max + 1) * 8) ||
        !ensure(W.pool, (size_t)pool_blocks * BLK_WORDS * 4) || (events && !ensure(W.ev_counts, n_items_max * 4)))
        return DACH_CUDA_ERROR;
    if (seg && (!ensure(W.nseg, n * 4) || !ensure(W.seg_first, (n + 1) * 8) || !ensure(W.item_hay, n_items_max * 4) ||
                !ensure(W.item_beg, n_items_max * 4) || !ensure(W.n_items_dev, 8)))
        return DACH_CUDA_ERROR;

    ScanParams P = image_params(d, d_text, text_lo, text_end, d_offs, n);
    P.counts = static_cast<uint32_t*>(W.counts.p);
    P.ev_counts = events ? static_cast<uint32_t*>(W.ev_counts.p) : nullptr;
    P.pool = static_cast<uint32_t*>(W.pool.p);
    P.pool_blocks = pool_blocks;
    P.ctrl = static_cast<ScanCtrl*>(W.ctrl.p);
    P.state_io = d_state_io;
    const size_t smem = plan_smem(d, P, v1, std3, threads, ctas_per_sm, duo ? 2 : direct ? 0 : 1);

    unsigned long long* tiles = static_cast<unsigned long long*>(W.tiles.p);
    unsigned long long* item_offs = static_cast<unsigned long long*>(W.item_offs.p);
    k_check_offsets<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_offs, n, (uint64_t)(text_end - d_text), P.ctrl);
    ++d->launches;
    if (seg) {
        cudaMemsetAsync(W.counts.p, 0, n_items_max * 4, st);  // items past the real count stay empty
        if (events) cudaMemsetAsync(W.ev_counts.p, 0, n_items_max * 4, st);
        enqueue_seg_table(d, W, d_offs, n, seg_len, seg_from, P, st);
    }
    cudaEventRecord(W.ev[3], st);
    if (!cuda_ok(cw_machine   ? launch_cw(mode, P, grid, std::min(threads, 1024), smem, st)
                 : lm_machine ? launch_lm(P, grid, std::min(threads, 1024), smem, st)
                 : duo        ? launch_duo(mode, P, grid, threads, smem, st)
                 : direct     ? launch_direct(mode, P, grid, threads, smem, st)
                 : v1        ? launch_std(std3 ? 3 : std2 ? 2 : 1, mode, P, grid, threads, smem, st,
                                           ctas_per_sm >= 2 && threads <= 768 && grid % 2 == 0)
                              : launch_scan(d->charwise, mode, P, grid, threads, smem, st),
                 "k_scan launch"))
        return DACH_CUDA_ERROR;
    cudaEventRecord(W.ev[1], st);
    k_offsets_tile_sums<1><<<(unsigned)n_tiles, kScanThreads, 0, st>>>(P.counts, n_items_max, tiles);
    k_offsets_scan_tiles<<<1, kScanThreads, 0, st>>>(tiles, n_tiles);
    k_offsets_apply<1><<<(unsigned)n_tiles, kScanThreads, 0, st>>>(P.counts, n_items_max, tiles, item_offs);
    d->launches += 4;
    // batches whose match blocks stay in L2 anyway are copied in pool order (four launches fewer)
    const bool ordered = d->opt_gather_ordered >= 2 || (d->opt_gather_ordered == 1 && text_bytes >= (256ull << 20));
    // ordered event blocks are placed from descriptors (k_blk_desc) if the image has two-entry lists
    const bool use_desc = ordered && events && d->d_pairs && d->opt_expand_desc != 0;
    if (ordered) {
        if (!ensure(W.blk_first, (n_items_max + 1) * 8) || !ensure(W.tiles2, n_tiles * 8) ||
            !(use_desc ? ensure(W.desc, (size_t)pool_blocks * 16) : ensure(W.blkmap, (size_t)pool_blocks * 4)))
            return DACH_CUDA_ERROR;
        unsigned long long* tiles2 = static_cast<unsigned long long*>(W.tiles2.p);
        unsigned long long* blk_first = static_cast<unsigned long long*>(W.blk_first.p);
        if (events) {  // blocks per item: ceil(events / BLK_EVENTS)
            k_offsets_tile_sums<BLK_EVENTS><<<(unsigned)n_tiles, kScanThreads, 0, st>>>(P.ev_counts, n_items_max, tiles2);
            k_offsets_scan_tiles<<<1, kScanThreads, 0, st>>>(tiles2, n_tiles);
            k_offsets_apply<BLK_EVENTS><<<(unsigned)n_tiles, kScanThreads, 0, st>>>(P.ev_counts, n_items_max, tiles2, blk_first);
        } else {
            k_offsets_tile_sums<BLK_MATCHES><<<(unsigned)n_tiles, kScanThreads, 0, st>>>(P.counts, n_items_max, tiles2);
            k_offsets_scan_tiles<<<1, kScanThreads, 0, st>>>(tiles2, n_tiles);
            k_offsets_apply<BLK_MATCHES><<<(unsigned)n_tiles, kScanThreads, 0, st>>>(P.counts, n_items_max, tiles2, blk_first);
        }
        if (use_desc)
            k_blk_desc<<<d->sm_count * 8, 256, 0, st>>>(P.pool, P.ctrl, pool_blocks, blk_first, P.ev_counts, item_offs,
                                                        static_cast<uint4*>(W.desc.p));
        else
            k_blk_index<<<d->sm_count * 8, 256, 0, st>>>(P.pool, P.ctrl, pool_blocks, blk_first, static_cast<uint32_t*>(W.blkmap.p));
        d->launches += 4;
    }
    if (!cuda_ok(cudaGetLastError(), "kernel launch")) return DACH_CUDA_ERROR;
    cudaEventRecord(W.ev_scanned, st);
    W.job_items = n_items_max;
    W.job_seg = seg;
    W.job_ordered = ordered;
    W.job_events = events;
    W.job_desc = use_desc;
    W.job_mode = mode;
    W.job_pool_blocks = pool_blocks;
    return DACH_OK;
}

// ---- phase 2: gather into the caller's buffers.  No synchronisation. -----------------------------------
// d_out / d_out_offs may be peer-mapped memory of another GPU.  d_base (device pointer or nullptr): index of
// this batch's first match in d_out, added to the offsets too; `last`: also write out_offs[n].
int enqueue_place(dach_dev* d, Workspace& W, dach_match* d_out, uint64_t out_cap, uint64_t* d_out_offs,
                  const unsigned long long* d_base, bool last, cudaStream_t st, const uint32_t* d_pos_in = nullptr,
                  bool staged = false, bool dma = false, uint64_t h_base = 0, uint64_t h_total = 0) {
    if (!W.job_open) {
        set_error("no scan to place");
        return DACH_INVALID_ARGUMENT;
    }
    if (st != W.job_stream) cudaStreamWaitEvent(st, W.ev_scanned, 0);
    const uint64_t n = W.job_n, n_items = W.job_items;
    const ScanCtrl* ctrl = static_cast<const ScanCtrl*>(W.ctrl.p);
    const unsigned long long* item_offs = static_cast<const unsigned long long*>(W.item_offs.p);
    unsigned long long* offs64 = reinterpret_cast<unsigned long long*>(d_out_offs);
    const int gather_grid = d->sm_count * 8;
    if (n) {
        const uint32_t* pool = static_cast<const uint32_t*>(W.pool.p);
        const uint32_t* counts = static_cast<const uint32_t*>(W.counts.p);
        const uint32_t* blkmap = W.job_ordered ? static_cast<const uint32_t*>(W.blkmap.p) : nullptr;
        uint32_t* out_words = reinterpret_cast<uint32_t*>(d_out);
        const unsigned long long* g_base = d_base;
        unsigned long long g_cap = out_cap;
        if (staged) {  // peer destination: pack locally, then push with destination-aligned 16-byte stores
            if (!ensure(W.stage, W.job_cap * sizeof(dach_match) + 256)) return DACH_CUDA_ERROR;
            out_words = static_cast<uint32_t*>(W.stage.p);
            g_base = nullptr;
            g_cap = W.job_cap;
        }
        const unsigned long long* pad_like = staged ? d_base : nullptr;
        if (W.job_desc) {
            const uint4* desc = static_cast<const uint4*>(W.desc.p);
            const int u = d->opt_expand_u >= 8 ? 8 : d->opt_expand_u <= 2 ? 2 : 4;
            const bool ov = W.job_mode == M_OVERLAPPING;
            auto kern = ov ? (u == 8 ? k_expand_desc<true, 8> : u == 2 ? k_expand_desc<true, 2> : k_expand_desc<true, 4>)
                           : (u == 8 ? k_expand_desc<false, 8> : u == 2 ? k_expand_desc<false, 2> : k_expand_desc<false, 4>);
            kern<<<gather_grid, EXP_THREADS, 0, st>>>(pool, ctrl, W.job_pool_blocks, desc, item_offs, n_items, g_cap, g_base, out_words,
                                                      pad_like, d->d_pairs, d->d_outputs, d->d_opos);
        } else if (W.job_events) {
            const uint32_t* ev_counts = static_cast<const uint32_t*>(W.ev_counts.p);
            if (W.job_mode == M_OVERLAPPING)
                k_expand<true, 2><<<gather_grid, 256, 0, st>>>(pool, ctrl, W.job_pool_blocks, ev_counts, item_offs, n_items, g_cap, g_base,
                                                                out_words, blkmap, pad_like, d->d_outputs, d->d_opos);
            else
                k_expand<false, 2><<<gather_grid, 256, 0, st>>>(pool, ctrl, W.job_pool_blocks, ev_counts, item_offs, n_items, g_cap, g_base,
                                                                 out_words, blkmap, pad_like, d->d_outputs, d->d_opos);
        } else if (d->opt_gather_u >= 8)
            k_gather<8><<<gather_grid, 256, 0, st>>>(pool, ctrl, W.job_pool_blocks, counts, item_offs, n_items, g_cap, g_base, out_words, blkmap, pad_like);
        else if (d->opt_gather_u <= 2)
            k_gather<2><<<gather_grid, 256, 0, st>>>(pool, ctrl, W.job_pool_blocks, counts, item_offs, n_items, g_cap, g_base, out_words, blkmap, pad_like);
        else
            k_gather<4><<<gather_grid, 256, 0, st>>>(pool, ctrl, W.job_pool_blocks, counts, item_offs, n_items, g_cap, g_base, out_words, blkmap, pad_like);
        ++d->launches;
        if (staged) {
            cudaEventRecord(W.ev_push[0], st);
            if (dma) {
                // base and count are known on the host: the packed tuples go out through a copy engine -- no SM, no
                // LSU slot and no L1 line is taken from the scan that runs beside the exchange
                if (h_total && h_base + h_total <= out_cap &&
                    !cuda_ok(cudaMemcpyAsync(reinterpret_cast<uint32_t*>(d_out) + h_base * 3ull, out_words + ((h_base * 3ull) & 3ull),
                                             h_total * sizeof(dach_match), cudaMemcpyDefault, st),
                             "peer copy"))
                    return DACH_CUDA_ERROR;
            } else {
                k_push<<<d->sm_count * 4, 128, 0, st>>>(out_words, item_offs + n_items, d_base, out_cap, ctrl, reinterpret_cast<uint32_t*>(d_out));
                ++d->launches;
            }
            cudaEventRecord(W.ev_push[1], st);
        }
    }
    k_final_offsets<<<(unsigned)((n + 1 + 255) / 256), 256, 0, st>>>(
        W.job_seg ? static_cast<const unsigned long long*>(W.seg_first.p) : nullptr, item_offs, n, d_base, last ? 1 : 0, offs64, ctrl);
    ++d->launches;
    if (d_pos_in && n) {
        k_add_base<<<gather_grid, 256, 0, st>>>(ctrl, offs64, n, out_cap, d_pos_in, reinterpret_cast<uint32_t*>(d_out));
        ++d->launches;
    }
    if (!cuda_ok(cudaGetLastError(), "kernel launch")) return DACH_CUDA_ERROR;
    cudaEventRecord(W.ev[2], st);
    cudaMemcpyAsync(&W.pinned->total, item_offs + n_items, 8, cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(&W.pinned->ctrl, W.ctrl.p, sizeof(ScanCtrl), cudaMemcpyDeviceToHost, st);
    cudaEventRecord(W.ev_placed, st);
    W.job_placed = true;
    return DACH_OK;
}

// ---- wait for the placement, report ----------------------------------------------------------------------
int finish_scan(dach_dev* d, Workspace& W, uint64_t out_cap, uint64_t* needed) {
    W.refused = false;
    if (!cuda_ok(cudaEventSynchronize(W.ev_placed), "scan pipeline")) return DACH_CUDA_ERROR;
    float ms = 0;
    if (cudaEventElapsedTime(&ms, W.ev[3], W.ev[1]) == cudaSuccess) d->last_scan_ms = ms;
    if (cudaEventElapsedTime(&ms, W.ev[0], W.ev[2]) == cudaSuccess) d->last_total_ms = ms;
    // every carry of a per-item u32 count is 2^32 matches item_offs[n] does not hold (count_carry, scan_lane.cuh)
    const uint64_t total = W.pinned->total + ((uint64_t)W.pinned->ctrl.carries << 32);
    if (needed) *needed = total;
    if (W.pinned->ctrl.bad_offsets) {
        set_error("haystack offsets must be ascending and inside text_bytes, and no haystack may reach 4 GiB (match positions are u32)");
        return DACH_INVALID_ARGUMENT;
    }
    if (W.pinned->ctrl.carries) {
        // no capacity helps: the match list of one haystack is indexed in 32 bits
        W.refused = true;
        char buf[256];
        snprintf(buf, sizeof(buf), "a haystack yields 2^32 or more matches (batch total %llu): its match list cannot be placed; "
                 "count it with dach_dev_count_batch / dach_dev_hist_batch instead", (unsigned long long)total);
        set_error(buf);
        return DACH_INVALID_ARGUMENT;
    }
    if (W.pinned->ctrl.overflow || total > out_cap) {
        char buf[256];
        snprintf(buf, sizeof(buf), "output capacity too small (needed %llu, out_cap %llu, pool blocks used %u of %u, overflow flag %u)",
                 (unsigned long long)total, (unsigned long long)out_cap, W.pinned->ctrl.blk_cursor, W.job_pool_blocks,
                 W.pinned->ctrl.overflow);
        set_error(buf);
        return DACH_OUTPUT_OVERFLOW;
    }
    return DACH_OK;
}

// the synchronous pipeline on one stream; caller holds d->mu (or owns W) and has set the device
int scan_locked(dach_dev* d, Workspace& W, int mode, const uint8_t* d_text, const uint8_t* text_lo, const uint8_t* text_end, uint64_t text_bytes,
                const uint64_t* d_offs, uint64_t n, dach_match* d_out, uint64_t out_cap, uint64_t* d_out_offs, uint64_t* needed, cudaStream_t st,
                uint32_t* d_state_io = nullptr, const uint32_t* d_pos_in = nullptr) {
    int rc = enqueue_scan(d, W, mode, d_text, text_lo, text_end, text_bytes, d_offs, n, out_cap, st, d_state_io);
    if (rc) return rc;
    rc = enqueue_place(d, W, d_out, out_cap, d_out_offs, nullptr, true, st, d_pos_in);
    if (rc) return rc;
    return finish_scan(d, W, out_cap, needed);
}

double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

int check_host_offsets(const uint64_t* offs, uint64_t n) {
    for (uint64_t i = 0; i < n; ++i) {
        if (offs[i + 1] < offs[i]) {
            set_error("haystack offsets must be ascending");
            return DACH_INVALID_ARGUMENT;
        }
        if (offs[i + 1] - offs[i] > 0xffffffffull) {
            set_error("a haystack is longer than 4 GiB - 1 (match positions are u32)");
            return DACH_INVALID_ARGUMENT;
        }
    }
    return DACH_OK;
}

struct Slice {
    uint64_t first, last;  // haystacks [first, last)
    uint64_t base;         // matches before this slice
    uint64_t total;
};

// The slices a host-buffer batch (n > 0) goes to the device in: whole haystacks; `mode` is the iterator the device runs.
std::vector<Slice> cut_slices(const dach_dev* d, int mode, const uint64_t* offs, uint64_t n) {
    // Slices of ~slice_mib MiB of text, three in flight: while slice k is scanned, slice k+1 is
    // on its way to the device and the matches of slice k-1 are on their way back.
    uint64_t slice_bytes = (uint64_t)std::max<int64_t>(d->opt_slice_mib, 1) << 20;
    {
        // find_iter / leftmost_find_iter / charwise work on whole haystacks: a slice should bring at least one
        // haystack per lane (find_overlapping slices are cut into segments on the device instead)
        const bool segmentable = !d->charwise && (mode == M_OVERLAPPING || mode == M_NO_SUFFIX) && d->d_crec && d->opt_seg_len >= 0 && d->segmentable;
        const uint64_t lanes = (uint64_t)d->sm_count * 1024, avg = (offs[n] - offs[0]) / n + 1;
        if (!segmentable) slice_bytes = std::min<uint64_t>(std::max(slice_bytes, lanes * avg), 1ull << 30);
    }
    std::vector<Slice> slices;
    // Slice sizes ramp up at the head of the batch and down at its tail (1/8, 1/4, 1/2, 1, ..., 1/2, 1/4,
    // 1/8 of slice_bytes): nothing can be scanned before the first upload lands and nothing overlaps the
    // last scan + download, so those two are kept short.
    const uint64_t batch_end = offs[n];
    for (uint64_t i = 0; i < n;) {
        uint64_t j = i + 1;
        const uint64_t done = offs[i] - offs[0], left = batch_end - offs[i];
        uint64_t want = slice_bytes;
        const size_t k = slices.size();
        if (d->opt_slice_ramp && k < 3) want = std::min(want, slice_bytes >> (3 - k));  // head: 1/8, 1/4, 1/2
        if (d->opt_slice_ramp && left < 2 * slice_bytes) want = std::min(want, std::max<uint64_t>(left / 3, slice_bytes >> 3));  // tail: shrinking
        (void)done;
        want = std::max<uint64_t>(want, 1u << 20);
        const uint64_t lim = offs[i] + want;
        if (j < n && offs[j + 1] <= lim) {  // largest j with offs[j] <= lim
            uint64_t lo = j, hi = n;
            while (lo < hi) {
                const uint64_t mid = (lo + hi + 1) / 2;
                if (offs[mid] <= lim)
                    lo = mid;
                else
                    hi = mid - 1;
            }
            j = lo;
        }
        slices.push_back({i, j, 0, 0});
        i = j;
    }
    return slices;
}

// Uploads haystacks [first, last) of a host batch into W's text and offsets buffers on W's stream once the slot's
// previous work is done (the wait is added to *t_reuse).
bool slice_h2d(dach_dev* d, Workspace& W, const uint8_t* text, const uint64_t* offs, uint64_t first, uint64_t last, double* t_reuse) {
    const uint64_t tb = offs[last] - offs[first], ns = last - first;
    const double t0 = now_ms();
    if (!cuda_ok(cudaStreamSynchronize(W.stream), "slot reuse")) return false;
    *t_reuse += now_ms() - t0;
    if (!ensure(W.text, tb + 32) || !ensure(W.offs, (ns + 1) * 8) || !ensure(W.out_offs, (ns + 1) * 8)) return false;
    if (tb && !cuda_ok(cudaMemcpyAsync(W.text.p, text + offs[first], tb, cudaMemcpyHostToDevice, W.stream), "H2D text"))
        return false;
    // The offsets go through a pinned staging buffer: an async copy from pageable memory first waits
    // for everything queued in the stream (here: the 64 MiB text upload) and blocks the host meanwhile,
    // which starves the whole pipeline.  (The slot's stream was synchronised above, so the buffer is free.)
    const void* offs_src = offs + first;
    const size_t ob = (ns + 1) * 8;
    if (W.offs_stage_bytes < ob) {
        if (W.offs_stage) cudaFreeHost(W.offs_stage);
        W.offs_stage = nullptr;
        W.offs_stage_bytes = 0;
        void* q = nullptr;
        if (cudaMallocHost(&q, ob + ob / 2) == cudaSuccess) {
            W.offs_stage = q;
            W.offs_stage_bytes = ob + ob / 2;
        } else {
            cudaGetLastError();  // no staging: copy from the caller's memory directly
        }
    }
    if (W.offs_stage) {
        memcpy(W.offs_stage, offs_src, ob);
        offs_src = W.offs_stage;
    }
    if (!cuda_ok(cudaMemcpyAsync(W.offs.p, offs_src, ob, cudaMemcpyHostToDevice, W.stream), "H2D offsets"))
        return false;
    d->last_h2d += tb + (ns + 1) * 8;
    return true;
}

int scan_batch_host_impl(dach_dev* d, int mode, const uint8_t* text, const uint64_t* offs, uint64_t n,
                         dach_match* out, uint64_t out_cap, uint64_t* out_offs, uint64_t* needed) {
    if (!d || !offs || !out_offs || (out_cap && !out)) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    int rc = check_mode(d, mode);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(d->mu);
    DeviceGuard g(d->device);
    if (!g.ok) return DACH_CUDA_ERROR;
    d->last_h2d = d->last_d2h = 0;
    if (n == 0) {
        out_offs[0] = 0;
        if (needed) *needed = 0;
        return DACH_OK;
    }
    rc = check_host_offsets(offs, n);
    if (rc) return rc;
    // whatever is still queued on the slots' streams reads the caller's text or writes the caller's buffers:
    // no exit from here on may leave it in flight
    struct Drain {
        dach_dev* d;
        ~Drain() {
            for (Workspace& w : d->slot)
                if (w.stream) cudaStreamSynchronize(w.stream);
        }
    } drain_on_exit{d};
    std::vector<Slice> slices = cut_slices(d, mode, offs, n);
    for (Workspace& w : d->slot)
        if (!w.init(true)) return DACH_CUDA_ERROR;
    // every slot's previous work must be finished before its buffers are reused
    bool overflow = false, refused = false;
    uint64_t base = 0;
    const bool trace = getenv("DACH_DEBUG") != nullptr;
    double t_reuse = 0, t_scan = 0, t_final = 0, gpu_ms = 0;
    auto now = now_ms;
    const double t_begin = now();
    auto issue_h2d = [&](size_t k) -> bool {
        return slice_h2d(d, d->slot[k % dach_dev::kSlots], text, offs, slices[k].first, slices[k].last, &t_reuse);
    };
    // The copy engine must never wait for the host: the host blocks in scan_locked() until slice k is
    // scanned, so the uploads of the next TWO slices are queued before that (with one slice ahead the
    // H2D engine idles for the length of every scan).
    if (!issue_h2d(0)) return DACH_CUDA_ERROR;
    if (slices.size() > 1 && !issue_h2d(1)) return DACH_CUDA_ERROR;
    for (size_t k = 0; k < slices.size(); ++k) {
        if (k + 2 < slices.size() && !issue_h2d(k + 2)) return DACH_CUDA_ERROR;
        Workspace& W = d->slot[k % dach_dev::kSlots];
        Slice& s = slices[k];
        const uint64_t tb = offs[s.last] - offs[s.first], ns = s.last - s.first;
        s.base = base;
        // device-side capacity of this slice: what is left of the caller's buffer, bounded by a
        // generous per-slice estimate that grows if a slice overflows it
        uint64_t cap = std::max<uint64_t>(std::max<uint64_t>(tb / 4, 4096), W.out.bytes > 16 ? (W.out.bytes - 16) / 12 : 0);
        const double t_s0 = now();
        for (;;) {
            if (!ensure(W.out, cap * 12 + 16)) return DACH_CUDA_ERROR;
            uint64_t total = 0;
            const uint8_t* d_text = static_cast<const uint8_t*>(W.text.p) - offs[s.first];
            rc = scan_locked(d, W, mode, d_text, static_cast<const uint8_t*>(W.text.p), static_cast<const uint8_t*>(W.text.p) + tb, tb, static_cast<const uint64_t*>(W.offs.p), ns,
                             static_cast<dach_match*>(W.out.p), cap, static_cast<uint64_t*>(W.out_offs.p), &total, W.stream);
            s.total = total;
            if (rc == DACH_OUTPUT_OVERFLOW && total > cap) {
                cap = total;
                continue;
            }
            break;
        }
        t_scan += now() - t_s0;
        gpu_ms += d->last_total_ms;
        // a haystack past 2^32 matches: nothing is copied back, the other slices are still counted for *needed
        if (rc == DACH_INVALID_ARGUMENT && W.refused) refused = true;
        else if (rc != DACH_OK && rc != DACH_OUTPUT_OVERFLOW) return rc;
        if (refused || base + s.total > out_cap) overflow = true;
        if (!overflow) {
            // the slice's final offset is the next slice's first one: only the last slice copies it
            const uint64_t no = (k + 1 == slices.size()) ? ns + 1 : ns;
            if (!cuda_ok(cudaMemcpyAsync(out_offs + s.first, W.out_offs.p, no * 8, cudaMemcpyDeviceToHost, W.stream), "D2H offsets"))
                return DACH_CUDA_ERROR;
            if (s.total && !cuda_ok(cudaMemcpyAsync(out + base, W.out.p, s.total * 12, cudaMemcpyDeviceToHost, W.stream), "D2H matches"))
                return DACH_CUDA_ERROR;
            d->last_d2h += (ns + 1) * 8 + s.total * 12;
        }
        base += s.total;
    }
    const double t_f0 = now();
    for (Workspace& w : d->slot)
        if (!cuda_ok(cudaStreamSynchronize(w.stream), "D2H")) return DACH_CUDA_ERROR;
    t_final = now() - t_f0;
    if (trace)
        fprintf(stderr, "dach_scan_batch_host: %zu slices, %.2f ms total: waiting for slot reuse %.2f, in scan_locked %.2f, final D2H wait %.2f; kernels %.2f ms\n",
                slices.size(), now() - t_begin, t_reuse, t_scan, t_final, gpu_ms);
    if (needed) *needed = base;
    if (refused) {
        char buf[256];
        snprintf(buf, sizeof(buf), "a haystack yields 2^32 or more matches (batch total %llu): its match list cannot be placed; "
                 "count it with dach_count_batch_host / dach_hist_batch_host instead", (unsigned long long)base);
        set_error(buf);
        return DACH_INVALID_ARGUMENT;
    }
    if (overflow) {
        set_error("output capacity too small");
        return DACH_OUTPUT_OVERFLOW;
    }
    // slice-relative offsets -> batch offsets (slice k's last entry is slice k+1's first)
    for (size_t k = slices.size(); k-- > 0;) {
        const Slice& s = slices[k];
        const uint64_t hi = (k + 1 == slices.size()) ? s.last + 1 : s.last;
        for (uint64_t i = s.first; i < hi; ++i) out_offs[i] += s.base;
    }
    return DACH_OK;
}

// DF: set i (0: (haystack, slot) pairs, 1: (haystack, key) pairs) as the kernels see it
DfSet df_set(dach_dev* d, int i) {
    DfSet S;
    S.keys = static_cast<unsigned long long*>(d->df_tab[i].p);
    S.list = static_cast<uint32_t*>(d->df_list[i].p);
    S.n = static_cast<unsigned int*>(d->df_n.p) + i;
    S.mask = d->df_mask;
    S.limit = d->df_limit;
    return S;
}

// ---- COUNT / FIRST / HIST / DF: the scan of a batch and its results on one stream.  No synchronisation. -----------
// rk = RK_COUNT: d_counts (n x u64); RK_FIRST: d_first (n tuples), d_found (n x u8); RK_HIST: added into d_hist by
// `key` (DACH_KEY_OUTPUT / DACH_KEY_VALUE; the caller has checked its size); RK_DF: one window (df_windows), added
// into d_hist by `key` unless W.pinned->ctrl.overflow is set once W.ev_placed has completed.  The total (matches, or haystacks with a
// match) lands in W.pinned->total_rk once W.ev_placed has completed.  No block pool, no offsets, no gather: options
// kernel = 1, 2, 4 run StdMachine3 here (kernel = 0: the lane-per-haystack kernels).
// d_state_io (stream chunks, dach_dev_*_stream): haystack i is the next chunk of stream i, resumed in and leaving its
// state there as in enqueue_scan; FIRST then runs the caller's iterator to each chunk's last byte (RK_FIRST_STREAM)
// and adds d_pos (or nothing) to its positions.  Stream chunks are never cut into segments.
// rk = RK_MASK: d_masked (in the text's coordinates, like d_text) receives [text_lo, text_end) of the text, then `fill`
// over every match; no post-pass.
int enqueue_rk(dach_dev* d, Workspace& W, int rk, int mode, const uint8_t* d_text, const uint8_t* text_lo, const uint8_t* text_end,
               uint64_t text_bytes, const uint64_t* d_offs, uint64_t n, uint64_t* d_counts, dach_match* d_first, uint8_t* d_found,
               cudaStream_t st, int key = 0, uint64_t* d_hist = nullptr, uint32_t* d_state_io = nullptr, const uint32_t* d_pos = nullptr,
               uint8_t* d_masked = nullptr, uint8_t fill = 0) {
    if (n > 0xfffffff0ull) {
        set_error("too many haystacks in one batch (max 2^32-16)");
        return DACH_INVALID_ARGUMENT;
    }
    if (W.job_open) cudaStreamWaitEvent(st, W.ev_placed, 0);
    if (!ensure(W.ctrl, sizeof(ScanCtrl)) || !ensure(W.total_rk, 8)) return DACH_CUDA_ERROR;
    if (!cuda_ok(cudaMemsetAsync(W.ctrl.p, 0, sizeof(ScanCtrl), st), "memset ctrl") ||
        !cuda_ok(cudaMemsetAsync(W.total_rk.p, 0, 8, st), "memset total"))
        return DACH_CUDA_ERROR;
    cudaEventRecord(W.ev[0], st);
    cudaEventRecord(W.ev[3], st);
    unsigned long long* total = static_cast<unsigned long long*>(W.total_rk.p);
    // MASK: the copy runs after the offsets check (it writes nothing if that fails) and before the scan
    auto mask_copy = [&]() {
        const uint64_t bytes = (uint64_t)(text_end - text_lo);
        if (rk != RK_MASK || bytes == 0) return;
        const uint64_t blocks = std::min<uint64_t>((bytes / 16 + 256) / 256, 16ull * d->sm_count);
        k_mask_copy<<<(unsigned)blocks, 256, 0, st>>>(text_lo, d_masked + (text_lo - d_text), bytes, static_cast<const ScanCtrl*>(W.ctrl.p));
        ++d->launches;
    };
    if (n > 0) {
        int threads = (int)std::min<int64_t>(std::max<int64_t>(d->opt_threads, 32), kMaxThreads);
        threads = (threads / 32) * 32;
        const int ctas_per_sm = (int)std::min<int64_t>(std::max<int64_t>(d->opt_ctas_per_sm, 1), 2048 / threads);
        const int free_sms = (int)std::min<int64_t>(std::max<int64_t>(d->opt_reserve_sms, 0), d->sm_count - 1);
        const int grid = (d->sm_count - free_sms) * ctas_per_sm;
        // the first event of a haystack is the same for all three Standard iterators: FIRST runs find_overlapping
        // (not on a stream: the state carried after a find match is not the find_overlapping one)
        const int mmode = (rk == RK_FIRST && mode != M_LEFTMOST && !d_state_io) ? M_OVERLAPPING : mode;
        const bool v1 = d->opt_kernel >= 1 && d->d_crec && !(mmode == M_FIND && d->root_opos != 0);
        const bool cw_machine = v1 && d->charwise;
        const bool lm_machine = v1 && !d->charwise && mmode == M_LEFTMOST;
        const bool std3 = v1 && !d->charwise && mmode != M_LEFTMOST && d->root_base != 0;
        const bool machine = cw_machine || lm_machine || std3;
        if (d_state_io && !std3 && !cw_machine) {  // as enqueue_scan
            set_error("stream chunks need a Standard lane machine (find / find_overlapping, at most 2^24 states, bytewise: "
                      "BASE(ROOT) != 0, no empty pattern for find)");
            return DACH_INVALID_ARGUMENT;
        }
        // segments as in enqueue_scan (no tail-only cutting; a chunk of a stream resumes in a given state: it stays one item)
        bool seg = std3 && !d_state_io && (mmode == M_OVERLAPPING || mmode == M_NO_SUFFIX) && d->opt_seg_len >= 0 && d->segmentable;
        uint32_t seg_len = 0;
        uint64_t n_items_max = n;
        if (seg) {
            const uint64_t lanes = (uint64_t)grid * threads;
            const uint64_t warm = d->max_pattern_len ? d->max_pattern_len - 1 : 0;
            uint64_t want = d->opt_seg_len > 0 ? (uint64_t)d->opt_seg_len : std::max(text_bytes / (2 * lanes) + 1, std::max<uint64_t>(256, 8 * warm));
            want = (want + 255) & ~uint64_t(255);
            if (want >= text_bytes || want >= (1ull << 31)) {
                seg = false;
            } else {
                seg_len = (uint32_t)want;
                n_items_max = n + text_bytes / seg_len + 1;
                if (n_items_max > 0xfffffff0ull) seg = false, n_items_max = n;
            }
        }
        const uint64_t n_tiles = (n + kScanTile - 1) / kScanTile;
        if ((rk == RK_COUNT || rk == RK_FIRST) && !ensure(W.items_rk, n_items_max * (rk == RK_FIRST ? 16 : 8))) return DACH_CUDA_ERROR;
        if (seg && (!ensure(W.tiles, n_tiles * 8) || !ensure(W.nseg, n * 4) || !ensure(W.seg_first, (n + 1) * 8) ||
                    !ensure(W.item_hay, n_items_max * 4) || !ensure(W.item_beg, n_items_max * 4) || !ensure(W.n_items_dev, 8)))
            return DACH_CUDA_ERROR;
        ScanParams P = image_params(d, d_text, text_lo, text_end, d_offs, n);
        P.ctrl = static_cast<ScanCtrl*>(W.ctrl.p);
        P.item_count = static_cast<unsigned long long*>(W.items_rk.p);
        P.item_first = static_cast<uint4*>(W.items_rk.p);
        P.state_io = d_state_io;
        uint32_t hist_k = 0;
        if (rk == RK_HIST) {
            if (machine) hist_k = (uint32_t)std::min<int64_t>(std::max<int64_t>(d->opt_hist_smem, 0), std::min<int64_t>(d->n_cslots, 16384));
            if ((machine && !ensure(W.slot_hist, (size_t)d->n_cslots * 8)) || !ensure(W.rec_hist, (size_t)d->n_outputs * 8))
                return DACH_CUDA_ERROR;
            if ((machine && !cuda_ok(cudaMemsetAsync(W.slot_hist.p, 0, (size_t)d->n_cslots * 8, st), "memset slot counts")) ||
                !cuda_ok(cudaMemsetAsync(W.rec_hist.p, 0, (size_t)d->n_outputs * 8, st), "memset record counts"))
                return DACH_CUDA_ERROR;
            P.slot_hist = static_cast<unsigned long long*>(W.slot_hist.p);
            P.rec_hist = static_cast<unsigned long long*>(W.rec_hist.p);
            P.hist_smem = hist_k;
        }
        if (rk == RK_DF) {  // the sets are empty here (df_prepare, then k_df_clear after every window)
            P.df_key_value = key == DACH_KEY_VALUE;
            P.df_slots = df_set(d, 0);
            P.df_keys = df_set(d, 1);
        }
        P.mask_out = d_masked;
        P.mask_fill = fill;
        const size_t smem = plan_smem(d, P, machine, std3, threads, ctas_per_sm, 1, hist_k);
        k_check_offsets<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_offs, n, (uint64_t)(text_end - d_text), P.ctrl);
        ++d->launches;
        mask_copy();
        if (seg) enqueue_seg_table(d, W, d_offs, n, seg_len, 0, P, st);
        cudaEventRecord(W.ev[3], st);
        const int which = std3 ? 3 : machine ? 1 : 0;
        const int t = machine ? std::min(threads, 1024) : threads;
        if (!cuda_ok(rk == RK_COUNT  ? launch_rk<RK_COUNT>(which, d->charwise, mmode, P, grid, t, smem, st)
                     : rk == RK_HIST ? launch_rk<RK_HIST>(which, d->charwise, mmode, P, grid, t, smem, st)
                     : rk == RK_DF   ? launch_rk<RK_DF>(which, d->charwise, mmode, P, grid, t, smem, st)
                     : rk == RK_MASK ? launch_rk<RK_MASK>(which, d->charwise, mmode, P, grid, t, smem, st)
                     : d_state_io    ? launch_first_stream(d->charwise, mmode, P, grid, t, smem, st)
                                     : launch_rk<RK_FIRST>(which, d->charwise, mmode, P, grid, t, smem, st),
                     "k_scan launch"))
            return DACH_CUDA_ERROR;
        cudaEventRecord(W.ev[1], st);
        const unsigned long long* seg_first = seg ? static_cast<const unsigned long long*>(W.seg_first.p) : nullptr;
        if (rk == RK_HIST) {
            // lane machines: slot counts -> head records; an event of find_overlapping reports the head's whole list
            if (machine) {
                k_hist_heads<<<(unsigned)std::max<uint64_t>(1, std::min<uint64_t>((d->n_cslots + 255) / 256, 8 * d->sm_count)), 256, 0, st>>>(
                    P.slot_hist, d->d_opos, d->n_cslots, P.rec_hist);
                ++d->launches;
            }
            const unsigned fb = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((d->n_outputs + 255) / 256, 8 * d->sm_count));
            unsigned long long* hist = reinterpret_cast<unsigned long long*>(d_hist);
            if (machine && mmode == M_OVERLAPPING)
                k_hist_fold<true><<<fb, 256, 0, st>>>(P.rec_hist, d->d_outputs, d->n_outputs, key, hist, total);
            else
                k_hist_fold<false><<<fb, 256, 0, st>>>(P.rec_hist, d->d_outputs, d->n_outputs, key, hist, total);
            ++d->launches;
        } else if (rk == RK_DF) {
            // lane machines: (haystack, slot) -> (haystack, key); then the window's pairs into d_hist (the call's
            // accumulator) unless it overflowed, and both sets emptied for the next window
            const unsigned fb = (unsigned)(8 * d->sm_count);
            if (machine && mmode == M_OVERLAPPING)
                k_df_expand<true><<<fb, 256, 0, st>>>(P);
            else if (machine)
                k_df_expand<false><<<fb, 256, 0, st>>>(P);
            k_df_add<<<fb, 256, 0, st>>>(P.df_keys, P.ctrl, reinterpret_cast<unsigned long long*>(d_hist), total);
            k_df_clear<<<fb, 256, 0, st>>>(P.df_slots, P.df_keys);
            d->launches += machine ? 3 : 2;
            if (!cuda_ok(cudaMemsetAsync(d->df_n.p, 0, 8, st), "memset pair counts")) return DACH_CUDA_ERROR;
        } else if (rk == RK_COUNT)
            k_count_hay<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(seg_first, P.item_count, n, reinterpret_cast<unsigned long long*>(d_counts), total, P.ctrl);
        else if (rk == RK_MASK) {
        } else if (d_state_io)
            k_first_stream<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(P.item_first, n, d_pos, reinterpret_cast<uint32_t*>(d_first), d_found, total, P.ctrl);
        else
            k_first_hay<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(seg_first, P.item_first, n, reinterpret_cast<uint32_t*>(d_first), d_found, total, P.ctrl);
        if (rk == RK_COUNT || rk == RK_FIRST) d->launches += 2;  // the scan and k_count_hay / k_first_hay
        else ++d->launches;                                    // the scan
        if (!cuda_ok(cudaGetLastError(), "kernel launch")) return DACH_CUDA_ERROR;
    } else {
        if (rk == RK_MASK) {  // no haystack: every byte is outside one
            mask_copy();
            if (!cuda_ok(cudaGetLastError(), "kernel launch")) return DACH_CUDA_ERROR;
        }
        cudaEventRecord(W.ev[1], st);
    }
    cudaEventRecord(W.ev[2], st);
    cudaMemcpyAsync(&W.pinned->total_rk, total, 8, cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(&W.pinned->ctrl, W.ctrl.p, sizeof(ScanCtrl), cudaMemcpyDeviceToHost, st);
    cudaEventRecord(W.ev_placed, st);
    return DACH_OK;
}

// wait for enqueue_rk's work, report.  d == nullptr (jobs): the handle's timings are left to its synchronous calls.
int finish_rk(dach_dev* d, Workspace& W, uint64_t* total) {
    if (!cuda_ok(cudaEventSynchronize(W.ev_placed), "scan pipeline")) return DACH_CUDA_ERROR;
    float ms = 0;
    if (d && cudaEventElapsedTime(&ms, W.ev[3], W.ev[1]) == cudaSuccess) d->last_scan_ms = ms;
    if (d && cudaEventElapsedTime(&ms, W.ev[0], W.ev[2]) == cudaSuccess) d->last_total_ms = ms;
    if (W.pinned->ctrl.bad_offsets) {
        set_error("haystack offsets must be ascending and inside text_bytes, and no haystack may reach 4 GiB (match positions are u32)");
        return DACH_INVALID_ARGUMENT;
    }
    if (total) *total = W.pinned->total_rk;
    return DACH_OK;
}

// COUNT / FIRST of a host-buffer batch: the slices of dach_scan_batch_host; only the per-haystack results come back
int rk_batch_host_impl(dach_dev* d, int rk, int mode, const uint8_t* text, const uint64_t* offs, uint64_t n, uint64_t* counts,
                       dach_match* first, uint8_t* found, uint64_t* total) {
    if (!d || !offs || (n && (rk == RK_COUNT ? !counts : (!first || !found)))) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    int rc = check_mode(d, mode);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(d->mu);
    DeviceGuard g(d->device);
    if (!g.ok) return DACH_CUDA_ERROR;
    d->last_h2d = d->last_d2h = 0;
    if (total) *total = 0;
    if (n == 0) return DACH_OK;
    rc = check_host_offsets(offs, n);
    if (rc) return rc;
    struct Drain {  // no exit may leave copies of the caller's buffers in flight
        dach_dev* d;
        ~Drain() {
            for (Workspace& w : d->slot)
                if (w.stream) cudaStreamSynchronize(w.stream);
        }
    } drain_on_exit{d};
    const std::vector<Slice> slices = cut_slices(d, (rk == RK_FIRST && mode != M_LEFTMOST) ? M_OVERLAPPING : mode, offs, n);
    for (Workspace& w : d->slot)
        if (!w.init(true)) return DACH_CUDA_ERROR;
    double t_reuse = 0;
    auto issue_h2d = [&](size_t k) -> bool {
        return slice_h2d(d, d->slot[k % dach_dev::kSlots], text, offs, slices[k].first, slices[k].last, &t_reuse);
    };
    if (!issue_h2d(0)) return DACH_CUDA_ERROR;
    if (slices.size() > 1 && !issue_h2d(1)) return DACH_CUDA_ERROR;
    uint64_t sum = 0;
    for (size_t k = 0; k < slices.size(); ++k) {
        if (k + 2 < slices.size() && !issue_h2d(k + 2)) return DACH_CUDA_ERROR;
        Workspace& W = d->slot[k % dach_dev::kSlots];
        const Slice& s = slices[k];
        const uint64_t tb = offs[s.last] - offs[s.first], ns = s.last - s.first;
        if (!ensure(W.out, ns * sizeof(dach_match) + 16)) return DACH_CUDA_ERROR;
        const uint8_t* d_text = static_cast<const uint8_t*>(W.text.p) - offs[s.first];
        // COUNT: counts in W.out; FIRST: tuples in W.out, found flags in W.out_offs
        rc = enqueue_rk(d, W, rk, mode, d_text, static_cast<const uint8_t*>(W.text.p), static_cast<const uint8_t*>(W.text.p) + tb, tb,
                        static_cast<const uint64_t*>(W.offs.p), ns, static_cast<uint64_t*>(W.out.p), static_cast<dach_match*>(W.out.p),
                        static_cast<uint8_t*>(W.out_offs.p), W.stream);
        uint64_t t = 0;
        if (!rc) rc = finish_rk(d, W, &t);
        if (rc) return rc;
        sum += t;
        if (rk == RK_COUNT) {
            if (!cuda_ok(cudaMemcpyAsync(counts + s.first, W.out.p, ns * 8, cudaMemcpyDeviceToHost, W.stream), "D2H counts"))
                return DACH_CUDA_ERROR;
            d->last_d2h += ns * 8;
        } else {
            if (!cuda_ok(cudaMemcpyAsync(first + s.first, W.out.p, ns * sizeof(dach_match), cudaMemcpyDeviceToHost, W.stream), "D2H first") ||
                !cuda_ok(cudaMemcpyAsync(found + s.first, W.out_offs.p, ns, cudaMemcpyDeviceToHost, W.stream), "D2H found"))
                return DACH_CUDA_ERROR;
            d->last_d2h += ns * (sizeof(dach_match) + 1);
        }
    }
    for (Workspace& w : d->slot)
        if (!cuda_ok(cudaStreamSynchronize(w.stream), "D2H")) return DACH_CUDA_ERROR;
    if (total) *total = sum;
    return DACH_OK;
}

// MASK: the fill byte of a charwise automaton keeps UTF-8 valid, and the masked buffer does not overlap the text (a lane
// that has not read its bytes yet would see another lane's fill: spans reach back into the segment before theirs)
int check_mask(const dach_dev* d, const uint8_t* text, uint64_t text_bytes, uint8_t fill, const uint8_t* out) {
    if (d->charwise && fill >= 0x80) {
        set_error("the fill byte of a charwise automaton must be below 0x80 (the masked text stays valid UTF-8)");
        return DACH_INVALID_ARGUMENT;
    }
    if (text_bytes && (uintptr_t)out < (uintptr_t)text + text_bytes && (uintptr_t)text < (uintptr_t)out + text_bytes) {
        set_error("the masked buffer overlaps the text (masking in place is not supported)");
        return DACH_INVALID_ARGUMENT;
    }
    return DACH_OK;
}

// MASK of a host-buffer batch: the slices of dach_scan_batch_host; each slice's masked bytes come back into out
int mask_batch_host_impl(dach_dev* d, int mode, const uint8_t* text, const uint64_t* offs, uint64_t n, uint8_t fill, uint8_t* out) {
    if (!d || !offs || (offs[n] && (!text || !out))) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    int rc = check_mask(d, text, offs[n], fill, out);
    if (rc) return rc;
    rc = check_mode(d, mode);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(d->mu);
    DeviceGuard g(d->device);
    if (!g.ok) return DACH_CUDA_ERROR;
    d->last_h2d = d->last_d2h = 0;
    if (n == 0) {
        if (offs[0]) memcpy(out, text, offs[0]);
        return DACH_OK;
    }
    rc = check_host_offsets(offs, n);
    if (rc) return rc;
    struct Drain {  // no exit may leave copies of the caller's buffers in flight
        dach_dev* d;
        ~Drain() {
            for (Workspace& w : d->slot)
                if (w.stream) cudaStreamSynchronize(w.stream);
        }
    } drain_on_exit{d};
    const std::vector<Slice> slices = cut_slices(d, mode, offs, n);
    for (Workspace& w : d->slot)
        if (!w.init(true)) return DACH_CUDA_ERROR;
    if (offs[0]) memcpy(out, text, offs[0]);  // bytes before the first haystack
    double t_reuse = 0;
    auto issue_h2d = [&](size_t k) -> bool {
        return slice_h2d(d, d->slot[k % dach_dev::kSlots], text, offs, slices[k].first, slices[k].last, &t_reuse);
    };
    if (!issue_h2d(0)) return DACH_CUDA_ERROR;
    if (slices.size() > 1 && !issue_h2d(1)) return DACH_CUDA_ERROR;
    for (size_t k = 0; k < slices.size(); ++k) {
        if (k + 2 < slices.size() && !issue_h2d(k + 2)) return DACH_CUDA_ERROR;
        Workspace& W = d->slot[k % dach_dev::kSlots];
        const Slice& s = slices[k];
        const uint64_t tb = offs[s.last] - offs[s.first], ns = s.last - s.first;
        if (!ensure(W.out, tb + 16)) return DACH_CUDA_ERROR;
        const uint8_t* d_text = static_cast<const uint8_t*>(W.text.p) - offs[s.first];
        rc = enqueue_rk(d, W, RK_MASK, mode, d_text, static_cast<const uint8_t*>(W.text.p), static_cast<const uint8_t*>(W.text.p) + tb, tb,
                        static_cast<const uint64_t*>(W.offs.p), ns, nullptr, nullptr, nullptr, W.stream, 0, nullptr, nullptr, nullptr,
                        static_cast<uint8_t*>(W.out.p) - offs[s.first], fill);
        if (!rc) rc = finish_rk(d, W, nullptr);
        if (rc) return rc;
        if (tb && !cuda_ok(cudaMemcpyAsync(out + offs[s.first], W.out.p, tb, cudaMemcpyDeviceToHost, W.stream), "D2H masked text"))
            return DACH_CUDA_ERROR;
        d->last_d2h += tb;
    }
    for (Workspace& w : d->slot)
        if (!cuda_ok(cudaStreamSynchronize(w.stream), "D2H")) return DACH_CUDA_ERROR;
    return DACH_OK;
}

// HIST: the key and the size of the caller's histogram, decided before anything is launched
int check_hist(const dach_dev* d, int key, uint64_t n_hist) {
    if (key != DACH_KEY_OUTPUT && key != DACH_KEY_VALUE) {
        set_error("unknown histogram key");
        return DACH_INVALID_ARGUMENT;
    }
    if (key == DACH_KEY_OUTPUT ? n_hist < d->n_outputs : (d->n_outputs && n_hist <= d->max_value)) {
        set_error(key == DACH_KEY_OUTPUT ? "n_hist is below the number of output records"
                                         : "n_hist must exceed the largest pattern value");
        return DACH_INVALID_ARGUMENT;
    }
    return DACH_OK;
}

// HIST of a host-buffer batch: the slices of dach_scan_batch_host add into one device histogram, which comes back once
// and is added into the caller's
int hist_batch_host_impl(dach_dev* d, int mode, int key, const uint8_t* text, const uint64_t* offs, uint64_t n, uint64_t* hist,
                         uint64_t n_hist, uint64_t* total) {
    if (!d || !offs || (n_hist && !hist)) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    int rc = check_hist(d, key, n_hist);
    if (rc) return rc;
    rc = check_mode(d, mode);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(d->mu);
    DeviceGuard g(d->device);
    if (!g.ok) return DACH_CUDA_ERROR;
    d->last_h2d = d->last_d2h = 0;
    if (total) *total = 0;
    if (n == 0) return DACH_OK;
    rc = check_host_offsets(offs, n);
    if (rc) return rc;
    struct Drain {  // no exit may leave copies of the caller's buffers in flight
        dach_dev* d;
        ~Drain() {
            for (Workspace& w : d->slot)
                if (w.stream) cudaStreamSynchronize(w.stream);
        }
    } drain_on_exit{d};
    const std::vector<Slice> slices = cut_slices(d, mode, offs, n);
    for (Workspace& w : d->slot)
        if (!w.init(true)) return DACH_CUDA_ERROR;
    // the batch's histogram: zeroed before any slice adds into it (the slices run on the slots' streams)
    DevBuf& acc = d->slot[0].hist_acc;
    if (!ensure(acc, n_hist * 8) || !cuda_ok(cudaMemsetAsync(acc.p, 0, n_hist * 8, d->slot[0].stream), "memset histogram") ||
        !cuda_ok(cudaStreamSynchronize(d->slot[0].stream), "memset histogram"))
        return DACH_CUDA_ERROR;
    double t_reuse = 0;
    auto issue_h2d = [&](size_t k) -> bool {
        return slice_h2d(d, d->slot[k % dach_dev::kSlots], text, offs, slices[k].first, slices[k].last, &t_reuse);
    };
    if (!issue_h2d(0)) return DACH_CUDA_ERROR;
    if (slices.size() > 1 && !issue_h2d(1)) return DACH_CUDA_ERROR;
    uint64_t sum = 0;
    for (size_t k = 0; k < slices.size(); ++k) {
        if (k + 2 < slices.size() && !issue_h2d(k + 2)) return DACH_CUDA_ERROR;
        Workspace& W = d->slot[k % dach_dev::kSlots];
        const Slice& s = slices[k];
        const uint64_t tb = offs[s.last] - offs[s.first], ns = s.last - s.first;
        const uint8_t* d_text = static_cast<const uint8_t*>(W.text.p) - offs[s.first];
        rc = enqueue_rk(d, W, RK_HIST, mode, d_text, static_cast<const uint8_t*>(W.text.p), static_cast<const uint8_t*>(W.text.p) + tb, tb,
                        static_cast<const uint64_t*>(W.offs.p), ns, nullptr, nullptr, nullptr, W.stream, key, static_cast<uint64_t*>(acc.p));
        uint64_t t = 0;
        if (!rc) rc = finish_rk(d, W, &t);
        if (rc) return rc;
        sum += t;
    }
    for (Workspace& w : d->slot)
        if (!cuda_ok(cudaStreamSynchronize(w.stream), "scan")) return DACH_CUDA_ERROR;
    std::vector<uint64_t> h(n_hist);
    if (n_hist && !cuda_ok(cudaMemcpy(h.data(), acc.p, n_hist * 8, cudaMemcpyDeviceToHost), "D2H histogram")) return DACH_CUDA_ERROR;
    d->last_d2h = n_hist * 8;
    for (uint64_t i = 0; i < n_hist; ++i) hist[i] += h[i];
    if (total) *total = sum;
    return DACH_OK;
}

// ---- DF ---------------------------------------------------------------------------------------------------------
// Both pair sets sized by option df_pairs and empty, and the call's accumulator (n_df x u64) zeroed, on stream st
int df_prepare(dach_dev* d, uint64_t n_df, cudaStream_t st) {
    const uint64_t limit = std::min<uint64_t>(std::max<uint64_t>({(uint64_t)std::max<int64_t>(d->opt_df_pairs, 1), d->n_cslots, d->n_outputs}), 1ull << 30);
    uint64_t cap = 2;
    while (cap < 2 * limit) cap <<= 1;
    if (cap - 1 != d->df_mask || !d->df_tab[0].p) d->df_clean = false;
    d->df_mask = (uint32_t)(cap - 1);
    d->df_limit = (uint32_t)limit;
    if (!ensure(d->df_acc, n_df * 8) || !cuda_ok(cudaMemsetAsync(d->df_acc.p, 0, n_df * 8, st), "memset document frequencies"))
        return DACH_CUDA_ERROR;
    if (!d->df_clean) {
        for (int i = 0; i < 2; ++i)
            if (!ensure(d->df_tab[i], cap * 8) || !ensure(d->df_list[i], cap * 4) ||
                !cuda_ok(cudaMemsetAsync(d->df_tab[i].p, 0xff, cap * 8, st), "memset pair set"))
                return DACH_CUDA_ERROR;
        if (!ensure(d->df_n, 8) || !cuda_ok(cudaMemsetAsync(d->df_n.p, 0, 8, st), "memset pair counts")) return DACH_CUDA_ERROR;
        d->df_clean = true;
    }
    return cuda_ok(cudaStreamSynchronize(st), "prepare pair sets") ? DACH_OK : DACH_CUDA_ERROR;
}

// DF of haystacks [first, last) of a batch whose host offsets are `offs` and whose device offsets from haystack
// `first` on are d_offs, on W / st: windows of at most *win haystacks, each scanned, expanded and -- unless it
// overflowed -- added into d->df_acc before the next is enqueued.  A window that overflows is scanned again as two
// halves, and *win keeps the smaller size for the rest of the call.  A window of one haystack cannot overflow: it
// holds at most n_cslots distinct states and n_outputs distinct keys, and df_limit is at least both.
int df_windows(dach_dev* d, Workspace& W, int mode, int key, const uint8_t* d_text, const uint8_t* text_lo, const uint8_t* text_end,
               const uint64_t* d_offs, const uint64_t* offs, uint64_t first, uint64_t last, cudaStream_t st, uint64_t* win, uint64_t* sum) {
    for (uint64_t a = first; a < last;) {
        const uint64_t b = last - a <= *win ? last : a + *win;
        d->df_clean = false;
        int rc = enqueue_rk(d, W, RK_DF, mode, d_text, text_lo, text_end, offs[b] - offs[a], d_offs + (a - first), b - a, nullptr, nullptr,
                            nullptr, st, key, static_cast<uint64_t*>(d->df_acc.p));
        if (rc) return rc;
        d->df_clean = true;  // k_df_clear and the counters' reset are enqueued
        uint64_t t = 0;
        rc = finish_rk(d, W, &t);
        if (rc) return rc;
        if (W.pinned->ctrl.overflow) {
            if (b - a == 1) {
                set_error("document frequencies: one haystack overflowed the pair sets");
                return DACH_CUDA_ERROR;
            }
            *win = (b - a + 1) / 2;
            ++d->last_df_rescans;
            continue;
        }
        ++d->last_df_windows;
        *sum += t;
        a = b;
    }
    return DACH_OK;
}

// DF of a device batch: the offsets come to the host once (8 B per haystack) to be checked and cut into the slices of
// dach_scan_batch_host; the windows add into d->df_acc, which reaches d_df only when all of them are done
int df_batch_dev_impl(dach_dev* d, int mode, int key, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                      uint64_t* d_df, uint64_t n_df, uint64_t* total, cudaStream_t st) {
    std::lock_guard<std::mutex> lk(d->mu);
    DeviceGuard g(d->device);
    if (!g.ok) return DACH_CUDA_ERROR;
    d->last_h2d = d->last_d2h = 0;
    d->last_df_windows = d->last_df_rescans = 0;
    if (total) *total = 0;
    if (n == 0) return DACH_OK;
    if (n > 0xfffffff0ull) {
        set_error("too many haystacks in one batch (max 2^32-16)");
        return DACH_INVALID_ARGUMENT;
    }
    std::vector<uint64_t> offs(n + 1);
    if (!cuda_ok(cudaMemcpyAsync(offs.data(), d_offs, (n + 1) * 8, cudaMemcpyDeviceToHost, st), "D2H offsets") ||
        !cuda_ok(cudaStreamSynchronize(st), "D2H offsets"))
        return DACH_CUDA_ERROR;
    d->last_d2h = (n + 1) * 8;
    int rc = check_host_offsets(offs.data(), n);
    if (rc) return rc;
    if (offs[n] > text_bytes) {
        set_error("haystack offsets must be inside text_bytes");
        return DACH_INVALID_ARGUMENT;
    }
    rc = df_prepare(d, n_df, st);
    if (rc) return rc;
    const std::vector<Slice> slices = cut_slices(d, mode, offs.data(), n);
    uint64_t win = ~0ull, sum = 0;
    for (const Slice& s : slices) {
        rc = df_windows(d, d->ws, mode, key, d_text, d_text, d_text + text_bytes, d_offs + s.first, offs.data(), s.first, s.last, st, &win, &sum);
        if (rc) return rc;
    }
    if (n_df) {
        k_df_commit<<<(unsigned)std::min<uint64_t>((n_df + 255) / 256, 8 * d->sm_count), 256, 0, st>>>(
            static_cast<const unsigned long long*>(d->df_acc.p), reinterpret_cast<unsigned long long*>(d_df), n_df);
        ++d->launches;
        if (!cuda_ok(cudaGetLastError(), "kernel launch") || !cuda_ok(cudaStreamSynchronize(st), "add document frequencies"))
            return DACH_CUDA_ERROR;
    }
    if (total) *total = sum;
    return DACH_OK;
}

// DF of a host-buffer batch: the slices of dach_scan_batch_host, each cut into windows; d->df_acc comes back once and
// is added into the caller's
int df_batch_host_impl(dach_dev* d, int mode, int key, const uint8_t* text, const uint64_t* offs, uint64_t n, uint64_t* df, uint64_t n_df,
                       uint64_t* total) {
    if (!d || !offs || (n_df && !df)) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    int rc = check_hist(d, key, n_df);
    if (rc) return rc;
    rc = check_mode(d, mode);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(d->mu);
    DeviceGuard g(d->device);
    if (!g.ok) return DACH_CUDA_ERROR;
    d->last_h2d = d->last_d2h = 0;
    d->last_df_windows = d->last_df_rescans = 0;
    if (total) *total = 0;
    if (n == 0) return DACH_OK;
    rc = check_host_offsets(offs, n);
    if (rc) return rc;
    struct Drain {  // no exit may leave copies of the caller's buffers in flight
        dach_dev* d;
        ~Drain() {
            for (Workspace& w : d->slot)
                if (w.stream) cudaStreamSynchronize(w.stream);
        }
    } drain_on_exit{d};
    const std::vector<Slice> slices = cut_slices(d, mode, offs, n);
    for (Workspace& w : d->slot)
        if (!w.init(true)) return DACH_CUDA_ERROR;
    rc = df_prepare(d, n_df, d->slot[0].stream);
    if (rc) return rc;
    double t_reuse = 0;
    auto issue_h2d = [&](size_t k) -> bool {
        return slice_h2d(d, d->slot[k % dach_dev::kSlots], text, offs, slices[k].first, slices[k].last, &t_reuse);
    };
    if (!issue_h2d(0)) return DACH_CUDA_ERROR;
    if (slices.size() > 1 && !issue_h2d(1)) return DACH_CUDA_ERROR;
    uint64_t win = ~0ull, sum = 0;
    for (size_t k = 0; k < slices.size(); ++k) {
        if (k + 2 < slices.size() && !issue_h2d(k + 2)) return DACH_CUDA_ERROR;
        Workspace& W = d->slot[k % dach_dev::kSlots];
        const Slice& s = slices[k];
        const uint64_t tb = offs[s.last] - offs[s.first];
        const uint8_t* d_text = static_cast<const uint8_t*>(W.text.p) - offs[s.first];
        rc = df_windows(d, W, mode, key, d_text, static_cast<const uint8_t*>(W.text.p), static_cast<const uint8_t*>(W.text.p) + tb,
                        static_cast<const uint64_t*>(W.offs.p), offs, s.first, s.last, W.stream, &win, &sum);
        if (rc) return rc;
    }
    for (Workspace& w : d->slot)
        if (!cuda_ok(cudaStreamSynchronize(w.stream), "scan")) return DACH_CUDA_ERROR;
    std::vector<uint64_t> h(n_df);
    if (n_df && !cuda_ok(cudaMemcpy(h.data(), d->df_acc.p, n_df * 8, cudaMemcpyDeviceToHost), "D2H document frequencies"))
        return DACH_CUDA_ERROR;
    d->last_d2h = n_df * 8;
    for (uint64_t i = 0; i < n_df; ++i) df[i] += h[i];
    if (total) *total = sum;
    return DACH_OK;
}

// maps every exception to a status: nothing may unwind through the C ABI
template <class F>
int guarded(F&& f) {
    try {
        return f();
    } catch (const std::bad_alloc&) {
        set_error("out of memory");
        return DACH_AUTOMATON_SCALE;
    } catch (const std::exception& e) {
        set_error(std::string("internal error: ") + e.what());
        return DACH_INVALID_ARGUMENT;
    } catch (...) {
        set_error("internal error");
        return DACH_INVALID_ARGUMENT;
    }
}

}  // namespace

extern "C" {

int dach_dev_upload(const dach_pma* pma, int device, dach_dev** out) {
    if (!out) return DACH_INVALID_ARGUMENT;
    *out = nullptr;
    if (!pma) {
        set_error("null automaton");
        return DACH_INVALID_ARGUMENT;
    }
    return guarded([&]() -> int {
        HostImage img;
        if (const char* e = getenv("DACH_HOT_SLOTS")) img.want_hot_slots = (uint32_t)strtoul(e, nullptr, 10);  // layout experiments
        const int rc = build_image(pma, &img);
        if (rc) return rc;
        int ndev = 0;
        if (!cuda_ok(cudaGetDeviceCount(&ndev), "cudaGetDeviceCount")) return DACH_CUDA_ERROR;
        if (device < 0 || device >= ndev) {
            set_error("no such CUDA device");
            return DACH_CUDA_ERROR;
        }
        DeviceGuard g(device);
        if (!g.ok) return DACH_CUDA_ERROR;
        std::unique_ptr<dach_dev> d(new dach_dev());
        d->device = device;
        d->charwise = img.charwise;
        d->match_kind = img.match_kind;
        d->n_slots = img.n_slots;
        d->root_opos = img.root_opos;
        d->max_pattern_len = img.max_pattern_len;
        d->segmentable = img.segmentable;
        d->mapper_len = (uint32_t)img.mapper.size();
        d->n_outputs = (uint32_t)(img.outputs.size() / 4);
        for (uint32_t i = 0; i < d->n_outputs; ++i) d->max_value = std::max(d->max_value, img.outputs[(size_t)i * 4]);
        d->n_cslots = (uint32_t)img.opos_tab.size();
        cudaDeviceProp prop;
        if (!cuda_ok(cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties")) return DACH_CUDA_ERROR;
        d->sm_count = prop.multiProcessorCount;
        d->smem_optin = prop.sharedMemPerBlockOptin;
        // one allocation for the whole image, 512-byte aligned parts
        constexpr int kParts = 9;
        const std::vector<uint32_t>* parts[kParts] = {&img.rec, &img.outputs, &img.root_table, &img.mapper, &img.crec, &img.opos_tab,
                                                       &img.new_of_old, &img.old_of_new, &img.pairs};
        size_t part_off[kParts], total = 0;
        for (int i = 0; i < kParts; ++i) {
            part_off[i] = total;
            total += (std::max<size_t>(parts[i]->size() * 4, 16) + 511) & ~size_t(511);
            d->image_bytes += parts[i]->size() * 4;
        }
        bool ok = cuda_ok(cudaMalloc(&d->image_base, total), "cudaMalloc image");
        d->image_alloc = total;
        for (int i = 0; ok && i < kParts; ++i)
            if (!parts[i]->empty())
                ok = cuda_ok(cudaMemcpy(static_cast<char*>(d->image_base) + part_off[i], parts[i]->data(), parts[i]->size() * 4,
                                        cudaMemcpyHostToDevice),
                             "upload image");
        if (ok) {
            char* b = static_cast<char*>(d->image_base);
            d->d_rec = reinterpret_cast<uint4*>(b + part_off[0]);
            d->d_outputs = reinterpret_cast<uint4*>(b + part_off[1]);
            if (!img.pairs.empty()) d->d_pairs = reinterpret_cast<uint4*>(b + part_off[8]);
            d->d_root = reinterpret_cast<uint32_t*>(b + part_off[2]);
            d->d_mapper = reinterpret_cast<uint32_t*>(b + part_off[3]);
            if (!img.crec.empty()) {
                d->d_crec = reinterpret_cast<uint4*>(b + part_off[4]);
                d->d_opos = reinterpret_cast<uint32_t*>(b + part_off[5]);
                if (img.hot_slots) {  // the compact image is renumbered: stream chunks translate state ids
                    d->d_id_in = reinterpret_cast<uint32_t*>(b + part_off[6]);
                    d->d_id_out = reinterpret_cast<uint32_t*>(b + part_off[7]);
                }
                d->hot_slots = img.hot_slots;
            }
            d->root_base = img.root_base;
        }
        ok = ok && install_policies((int)d->opt_l2_hints) && d->ws.init(false);
        if (!ok) {
            dach_dev_free(d.release());
            return DACH_CUDA_ERROR;
        }
        *out = d.release();
        return DACH_OK;
    });
}

void dach_dev_free(dach_dev* d) {
    if (!d || --d->refs > 0) return;  // jobs of this device are still alive: the last dach_job_free releases it
    DeviceGuard g(d->device);
    cudaFree(d->image_base);
    if (d->ev_ref) cudaEventDestroy(d->ev_ref);
    d->ws.release();
    for (Workspace& w : d->slot) w.release();
    for (DevBuf* b : {&d->df_tab[0], &d->df_tab[1], &d->df_list[0], &d->df_list[1], &d->df_n, &d->df_acc})
        if (b->p) cudaFree(b->p);
    delete d;
}

size_t dach_dev_image_bytes(const dach_dev* d) { return d ? d->image_bytes : 0; }

int dach_dev_scan_batch(dach_dev* d, int mode, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n,
                        uint64_t text_bytes, dach_match* d_out, uint64_t out_cap, uint64_t* d_out_offs,
                        uint64_t* needed, void* stream) {
    if (!d || !d_offs || !d_out_offs || (out_cap && !d_out)) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    const int rc = check_mode(d, mode);
    if (rc) return rc;
    return guarded([&]() -> int {
        std::lock_guard<std::mutex> lk(d->mu);
        DeviceGuard g(d->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        return scan_locked(d, d->ws, mode, d_text, d_text, d_text + text_bytes, text_bytes, d_offs, n, d_out, out_cap, d_out_offs, needed,
                           static_cast<cudaStream_t>(stream));
    });
}

int dach_dev_scan_stream(dach_dev* d, int mode, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                         uint32_t* d_state, const uint32_t* d_pos, dach_match* d_out, uint64_t out_cap, uint64_t* d_out_offs,
                         uint64_t* needed, void* stream) {
    if (!d || !d_offs || !d_out_offs || !d_state || (out_cap && !d_out)) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    if (mode != DACH_FIND && mode != DACH_FIND_OVERLAPPING) {
        set_error("stream chunks: mode must be DACH_FIND or DACH_FIND_OVERLAPPING (the crate's two steppers)");
        return DACH_INVALID_ARGUMENT;
    }
    const int rc = check_mode(d, mode);
    if (rc) return rc;
    return guarded([&]() -> int {
        std::lock_guard<std::mutex> lk(d->mu);
        DeviceGuard g(d->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        return scan_locked(d, d->ws, mode, d_text, d_text, d_text + text_bytes, text_bytes, d_offs, n, d_out, out_cap, d_out_offs, needed,
                           static_cast<cudaStream_t>(stream), d_state, d_pos);
    });
}

}  // extern "C"

namespace {
// COUNT / FIRST / HIST of stream chunks: the mode checks of dach_dev_scan_stream, then one enqueue_rk with the state
int rk_stream(dach_dev* d, int rk, int mode, int key, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
              uint32_t* d_state, const uint32_t* d_pos, uint64_t* d_counts, dach_match* d_first, uint8_t* d_found, uint64_t* d_hist,
              uint64_t* total, void* stream) {
    if (mode != DACH_FIND && mode != DACH_FIND_OVERLAPPING) {
        set_error("stream chunks: mode must be DACH_FIND or DACH_FIND_OVERLAPPING (the crate's two steppers)");
        return DACH_INVALID_ARGUMENT;
    }
    const int rc = check_mode(d, mode);
    if (rc) return rc;
    return guarded([&]() -> int {
        std::lock_guard<std::mutex> lk(d->mu);
        DeviceGuard g(d->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        const int r = enqueue_rk(d, d->ws, rk, mode, d_text, d_text, d_text + text_bytes, text_bytes, d_offs, n, d_counts, d_first, d_found,
                                 static_cast<cudaStream_t>(stream), key, d_hist, d_state, d_pos);
        return r ? r : finish_rk(d, d->ws, total);
    });
}
}  // namespace

extern "C" {

int dach_dev_count_stream(dach_dev* d, int mode, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                          uint32_t* d_state, uint64_t* d_counts, uint64_t* total, void* stream) {
    if (!d || !d_offs || !d_state || (n && !d_counts)) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    return rk_stream(d, RK_COUNT, mode, 0, d_text, d_offs, n, text_bytes, d_state, nullptr, d_counts, nullptr, nullptr, nullptr, total, stream);
}

int dach_dev_first_stream(dach_dev* d, int mode, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                          uint32_t* d_state, const uint32_t* d_pos, dach_match* d_first, uint8_t* d_found, uint64_t* n_found, void* stream) {
    if (!d || !d_offs || !d_state || (n && (!d_first || !d_found))) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    return rk_stream(d, RK_FIRST, mode, 0, d_text, d_offs, n, text_bytes, d_state, d_pos, nullptr, d_first, d_found, nullptr, n_found, stream);
}

int dach_dev_hist_stream(dach_dev* d, int mode, int key, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                         uint32_t* d_state, uint64_t* d_hist, uint64_t n_hist, uint64_t* total, void* stream) {
    if (!d || !d_offs || !d_state || (n_hist && !d_hist)) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    const int rc = check_hist(d, key, n_hist);
    if (rc) return rc;
    return rk_stream(d, RK_HIST, mode, key, d_text, d_offs, n, text_bytes, d_state, nullptr, nullptr, nullptr, nullptr, d_hist, total, stream);
}

int dach_scan_batch_host(dach_dev* d, int mode, const uint8_t* text, const uint64_t* offs, uint64_t n,
                         dach_match* out, uint64_t out_cap, uint64_t* out_offs, uint64_t* needed) {
    return guarded([&]() -> int { return scan_batch_host_impl(d, mode, text, offs, n, out, out_cap, out_offs, needed); });
}

int dach_dev_count_batch(dach_dev* d, int mode, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                         uint64_t* d_counts, uint64_t* total, void* stream) {
    if (!d || !d_offs || (n && !d_counts)) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    const int rc = check_mode(d, mode);
    if (rc) return rc;
    return guarded([&]() -> int {
        std::lock_guard<std::mutex> lk(d->mu);
        DeviceGuard g(d->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        const int r = enqueue_rk(d, d->ws, RK_COUNT, mode, d_text, d_text, d_text + text_bytes, text_bytes, d_offs, n, d_counts, nullptr,
                                 nullptr, static_cast<cudaStream_t>(stream));
        return r ? r : finish_rk(d, d->ws, total);
    });
}

int dach_count_batch_host(dach_dev* d, int mode, const uint8_t* text, const uint64_t* offs, uint64_t n, uint64_t* counts, uint64_t* total) {
    return guarded([&]() -> int { return rk_batch_host_impl(d, RK_COUNT, mode, text, offs, n, counts, nullptr, nullptr, total); });
}

int dach_dev_first_batch(dach_dev* d, int mode, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                         dach_match* d_first, uint8_t* d_found, uint64_t* n_found, void* stream) {
    if (!d || !d_offs || (n && (!d_first || !d_found))) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    const int rc = check_mode(d, mode);
    if (rc) return rc;
    return guarded([&]() -> int {
        std::lock_guard<std::mutex> lk(d->mu);
        DeviceGuard g(d->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        const int r = enqueue_rk(d, d->ws, RK_FIRST, mode, d_text, d_text, d_text + text_bytes, text_bytes, d_offs, n, nullptr, d_first,
                                 d_found, static_cast<cudaStream_t>(stream));
        return r ? r : finish_rk(d, d->ws, n_found);
    });
}

int dach_first_batch_host(dach_dev* d, int mode, const uint8_t* text, const uint64_t* offs, uint64_t n, dach_match* first, uint8_t* found,
                          uint64_t* n_found) {
    return guarded([&]() -> int { return rk_batch_host_impl(d, RK_FIRST, mode, text, offs, n, nullptr, first, found, n_found); });
}

int dach_dev_hist_batch(dach_dev* d, int mode, int key, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                        uint64_t* d_hist, uint64_t n_hist, uint64_t* total, void* stream) {
    if (!d || !d_offs || (n_hist && !d_hist)) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    int rc = check_hist(d, key, n_hist);
    if (rc) return rc;
    rc = check_mode(d, mode);
    if (rc) return rc;
    return guarded([&]() -> int {
        std::lock_guard<std::mutex> lk(d->mu);
        DeviceGuard g(d->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        const int r = enqueue_rk(d, d->ws, RK_HIST, mode, d_text, d_text, d_text + text_bytes, text_bytes, d_offs, n, nullptr, nullptr,
                                 nullptr, static_cast<cudaStream_t>(stream), key, d_hist);
        return r ? r : finish_rk(d, d->ws, total);
    });
}

int dach_hist_batch_host(dach_dev* d, int mode, int key, const uint8_t* text, const uint64_t* offs, uint64_t n, uint64_t* hist,
                         uint64_t n_hist, uint64_t* total) {
    return guarded([&]() -> int { return hist_batch_host_impl(d, mode, key, text, offs, n, hist, n_hist, total); });
}

int dach_dev_df_batch(dach_dev* d, int mode, int key, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                      uint64_t* d_df, uint64_t n_df, uint64_t* total, void* stream) {
    if (!d || !d_offs || (n_df && !d_df)) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    int rc = check_hist(d, key, n_df);
    if (rc) return rc;
    rc = check_mode(d, mode);
    if (rc) return rc;
    return guarded([&]() -> int {
        return df_batch_dev_impl(d, mode, key, d_text, d_offs, n, text_bytes, d_df, n_df, total, static_cast<cudaStream_t>(stream));
    });
}

int dach_df_batch_host(dach_dev* d, int mode, int key, const uint8_t* text, const uint64_t* offs, uint64_t n, uint64_t* df,
                       uint64_t n_df, uint64_t* total) {
    return guarded([&]() -> int { return df_batch_host_impl(d, mode, key, text, offs, n, df, n_df, total); });
}

int dach_dev_last_df_windows(const dach_dev* d, uint64_t* windows, uint64_t* rescans) {
    if (!d) return DACH_INVALID_ARGUMENT;
    if (windows) *windows = d->last_df_windows;
    if (rescans) *rescans = d->last_df_rescans;
    return DACH_OK;
}

int dach_dev_mask_batch(dach_dev* d, int mode, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                        uint8_t fill, uint8_t* d_out, void* stream) {
    if (!d || !d_offs || (text_bytes && (!d_text || !d_out))) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    int rc = check_mask(d, d_text, text_bytes, fill, d_out);
    if (rc) return rc;
    rc = check_mode(d, mode);
    if (rc) return rc;
    return guarded([&]() -> int {
        std::lock_guard<std::mutex> lk(d->mu);
        DeviceGuard g(d->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        const int r = enqueue_rk(d, d->ws, RK_MASK, mode, d_text, d_text, d_text + text_bytes, text_bytes, d_offs, n, nullptr, nullptr,
                                 nullptr, static_cast<cudaStream_t>(stream), 0, nullptr, nullptr, nullptr, d_out, fill);
        return r ? r : finish_rk(d, d->ws, nullptr);
    });
}

int dach_mask_batch_host(dach_dev* d, int mode, const uint8_t* text, const uint64_t* offs, uint64_t n, uint8_t fill, uint8_t* out) {
    return guarded([&]() -> int { return mask_batch_host_impl(d, mode, text, offs, n, fill, out); });
}

}  // extern "C"

namespace {
// time zero of dach_job_times: recorded on `stream` by the handle's first job operation
// (tried again by the next job operation if the event cannot be created)
void job_time_zero(dach_dev* d, cudaStream_t stream) {
    std::lock_guard<std::mutex> lk(d->ev_ref_mu);
    if (d->ev_ref) return;
    if (cudaEventCreate(&d->ev_ref) == cudaSuccess) cudaEventRecord(d->ev_ref, stream);
    else d->ev_ref = nullptr;
}

// COUNT / FIRST / HIST / MASK on a job: the mode check of the synchronous call (the caller has made the others), then
// enqueue_rk on the job's workspace, ordered after the job's previous operation; dach_job_wait reports it.  No handle
// mutex and no handle-wide state: the job's own workspace, events and pinned block only.
int job_rk(dach_job* j, int rk, int mode, int key, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
           uint64_t* d_counts, dach_match* d_first, uint8_t* d_found, uint64_t* d_hist, uint8_t* d_masked, uint8_t fill, void* stream) {
    int rc = check_mode(j->d, mode);
    if (rc) return rc;
    if (n > 0xfffffff0ull) {  // enqueue_rk's check, made here so that nothing at all is recorded on the stream
        set_error("too many haystacks in one batch (max 2^32-16)");
        return DACH_INVALID_ARGUMENT;
    }
    if (j->unplaced) {
        set_error("the job's scan has not been placed (dach_job_place comes before the job's next operation)");
        return DACH_INVALID_ARGUMENT;
    }
    return guarded([&]() -> int {
        DeviceGuard g(j->d->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        const cudaStream_t st = static_cast<cudaStream_t>(stream);
        job_time_zero(j->d, st);
        const int r = enqueue_rk(j->d, j->W, rk, mode, d_text, d_text, d_text + text_bytes, text_bytes, d_offs, n, d_counts, d_first,
                                 d_found, st, key, d_hist, nullptr, nullptr, d_masked, fill);
        if (r) return r;
        j->W.job_open = true;  // the job's next operation waits for W.ev_placed
        j->rk = rk;
        return DACH_OK;
    });
}
}  // namespace

extern "C" {

// ---- asynchronous jobs ------------------------------------------------------------------------------

int dach_job_create(dach_dev* d, dach_job** out) {
    if (!d || !out) return DACH_INVALID_ARGUMENT;
    *out = nullptr;
    return guarded([&]() -> int {
        DeviceGuard g(d->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        std::unique_ptr<dach_job> j(new dach_job());
        j->d = d;
        if (!j->W.init(false)) {
            j->W.release();
            return DACH_CUDA_ERROR;
        }
        ++d->refs;
        *out = j.release();
        return DACH_OK;
    });
}

void dach_job_free(dach_job* j) {
    if (!j) return;
    dach_dev* d = j->d;
    {
        DeviceGuard g(d->device);
        if (j->W.job_open) cudaEventSynchronize(j->W.ev_placed);
        j->W.release();
    }
    delete j;
    dach_dev_free(d);  // this job's reference (frees the device if its owner let go first)
}

int dach_job_scan(dach_job* j, int mode, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                  uint64_t cap_matches, void* stream) {
    if (!j || !d_offs) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    const int rc = check_mode(j->d, mode);
    if (rc) return rc;
    return guarded([&]() -> int {
        DeviceGuard g(j->d->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        job_time_zero(j->d, static_cast<cudaStream_t>(stream));
        const int r = enqueue_scan(j->d, j->W, mode, d_text, d_text, d_text + text_bytes, text_bytes, d_offs, n, cap_matches,
                                   static_cast<cudaStream_t>(stream));
        if (!r) {
            j->rk = RK_MATCHES;
            j->unplaced = true;
        }
        return r;
    });
}

int dach_job_place(dach_job* j, dach_match* d_out, uint64_t out_cap, uint64_t* d_out_offs, const uint64_t* d_base, void* stream) {
    if (!j || !d_out_offs || (out_cap && !d_out)) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    if (j->rk != RK_MATCHES) {
        set_error("no scan to place: the job's last operation was a count, first-match, histogram or mask");
        return DACH_INVALID_ARGUMENT;
    }
    return guarded([&]() -> int {
        DeviceGuard g(j->d->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        j->out_cap = out_cap;
        const int r = enqueue_place(j->d, j->W, d_out, out_cap, d_out_offs, reinterpret_cast<const unsigned long long*>(d_base), true,
                                    static_cast<cudaStream_t>(stream));
        if (!r) j->unplaced = false;
        return r;
    });
}

int dach_job_count(dach_job* j, int mode, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                   uint64_t* d_counts, void* stream) {
    if (!j || !d_offs || (n && !d_counts)) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    return job_rk(j, RK_COUNT, mode, 0, d_text, d_offs, n, text_bytes, d_counts, nullptr, nullptr, nullptr, nullptr, 0, stream);
}

int dach_job_first(dach_job* j, int mode, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                   dach_match* d_first, uint8_t* d_found, void* stream) {
    if (!j || !d_offs || (n && (!d_first || !d_found))) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    return job_rk(j, RK_FIRST, mode, 0, d_text, d_offs, n, text_bytes, nullptr, d_first, d_found, nullptr, nullptr, 0, stream);
}

int dach_job_hist(dach_job* j, int mode, int key, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes,
                  uint64_t* d_hist, uint64_t n_hist, void* stream) {
    if (!j || !d_offs || (n_hist && !d_hist)) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    const int rc = check_hist(j->d, key, n_hist);
    if (rc) return rc;
    return job_rk(j, RK_HIST, mode, key, d_text, d_offs, n, text_bytes, nullptr, nullptr, nullptr, d_hist, nullptr, 0, stream);
}

int dach_job_mask(dach_job* j, int mode, const uint8_t* d_text, const uint64_t* d_offs, uint64_t n, uint64_t text_bytes, uint8_t fill,
                  uint8_t* d_out, void* stream) {
    if (!j || !d_offs || (text_bytes && (!d_text || !d_out))) {
        set_error("null argument");
        return DACH_INVALID_ARGUMENT;
    }
    const int rc = check_mask(j->d, d_text, text_bytes, fill, d_out);
    if (rc) return rc;
    return job_rk(j, RK_MASK, mode, 0, d_text, d_offs, n, text_bytes, nullptr, nullptr, nullptr, nullptr, d_out, fill, stream);
}

int dach_job_wait(dach_job* j, uint64_t* needed) {
    if (!j) return DACH_INVALID_ARGUMENT;
    if (j->unplaced) {  // the last placement's report would be stale
        set_error("dach_job_wait: the job's scan has not been placed yet");
        return DACH_INVALID_ARGUMENT;
    }
    if (j->rk != RK_MATCHES)  // a reduction: *needed = its total (0 for MASK, whose total stays at its zero)
        return guarded([&]() -> int {
            DeviceGuard g(j->d->device);
            if (!g.ok) return DACH_CUDA_ERROR;
            return finish_rk(nullptr, j->W, needed);
        });
    if (!j->W.job_placed) {
        set_error("dach_job_wait: nothing has been placed yet");
        return DACH_INVALID_ARGUMENT;
    }
    return guarded([&]() -> int {
        DeviceGuard g(j->d->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        return finish_scan(j->d, j->W, j->out_cap, needed);
    });
}

double dach_job_scan_kernel_ms(const dach_job* j) {
    float ms = 0;
    if (j && cudaEventElapsedTime(&ms, j->W.ev[3], j->W.ev[1]) == cudaSuccess) return ms;
    cudaGetLastError();
    return 0;
}

// ms since the handle's first job operation of {scan kernel start, scan kernel end, peer push start, peer push end} of the
// job's last step (the last two are 0 without a peer push, and after a reduction): the timeline of a pipelined run
int dach_job_times(const dach_job* j, double out[4]) {
    if (!j || !out || !j->d->ev_ref) return DACH_INVALID_ARGUMENT;
    cudaEvent_t evs[4] = {j->W.ev[3], j->W.ev[1], j->W.ev_push[0], j->W.ev_push[1]};
    for (int i = 0; i < 4; ++i) {
        float ms = 0;
        out[i] = (i < 2 || j->rk == RK_MATCHES) && cudaEventElapsedTime(&ms, j->d->ev_ref, evs[i]) == cudaSuccess ? ms : 0.0;
    }
    cudaGetLastError();
    return DACH_OK;
}

double dach_job_push_ms(const dach_job* j) {
    float ms = 0;
    if (j && j->rk == RK_MATCHES && cudaEventElapsedTime(&ms, j->W.ev_push[0], j->W.ev_push[1]) == cudaSuccess) return ms;
    cudaGetLastError();
    return 0;
}

// ---- shard groups -----------------------------------------------------------------------------------

struct dach_group {
    int rank = 0, world = 1, device = 0;
    uint64_t match_cap = 0, n_total = 0;
    GroupCtl* ctl = nullptr;       // this rank's control block
    dach_match* out = nullptr;     // the gathering rank's dense match buffer (peer-mapped on the other ranks)
    uint64_t* offs = nullptr;      // ... and its n_total + 1 offsets
    GroupPeers peers;
    void* ipc_opened[3 * kMaxRanks];
    int n_ipc = 0;
    unsigned long long step = 0;
    GroupCtl* pinned = nullptr;    // host copy of the control block (finish)
    unsigned long long* h_vals = nullptr;  // pinned: {base, total, overflow flag} of the step being placed
    bool connected = false;
    bool push_dma = true;  // packed tuples leave through a copy engine (the rank's host learns base and count first)
};

namespace {
struct GroupHandle {
    uint64_t pid;
    int32_t device, rank;
    uint64_t ctl_ptr, out_ptr, offs_ptr;
    cudaIpcMemHandle_t ctl, out, offs;
};
static_assert(sizeof(GroupHandle) <= DACH_GROUP_HANDLE_BYTES, "DACH_GROUP_HANDLE_BYTES too small");
}  // namespace

int dach_group_create(int rank, int world, int device, uint64_t match_cap, uint64_t n_haystacks_total, dach_group** out) {
    if (!out) return DACH_INVALID_ARGUMENT;
    *out = nullptr;
    if (world < 1 || world > kMaxRanks || rank < 0 || rank >= world) {
        set_error("shard group: rank / world out of range (at most 16 ranks)");
        return DACH_INVALID_ARGUMENT;
    }
    return guarded([&]() -> int {
        DeviceGuard g(device);
        if (!g.ok) return DACH_CUDA_ERROR;
        std::unique_ptr<dach_group> G(new dach_group());
        G->rank = rank;
        G->world = world;
        G->device = device;
        G->match_cap = match_cap;
        G->n_total = n_haystacks_total;
        memset(&G->peers, 0, sizeof(G->peers));
        bool ok = cuda_ok(cudaMalloc(reinterpret_cast<void**>(&G->ctl), sizeof(GroupCtl)), "cudaMalloc group control") &&
                  cuda_ok(cudaMemset(G->ctl, 0, sizeof(GroupCtl)), "memset group control") &&
                  cuda_ok(cudaMallocHost(reinterpret_cast<void**>(&G->pinned), sizeof(GroupCtl)), "cudaMallocHost") &&
                  cuda_ok(cudaMallocHost(reinterpret_cast<void**>(&G->h_vals), 64), "cudaMallocHost");
        if (const char* e = getenv("DACH_GROUP_PUSH")) G->push_dma = strcmp(e, "sm") != 0;  // "sm": k_push instead of the copy engine
        if (ok && rank == 0)
            ok = cuda_ok(cudaMalloc(reinterpret_cast<void**>(&G->out), std::max<uint64_t>(match_cap, 1) * sizeof(dach_match)), "cudaMalloc gathered matches") &&
                 cuda_ok(cudaMalloc(reinterpret_cast<void**>(&G->offs), (n_haystacks_total + 1) * 8), "cudaMalloc gathered offsets");
        if (!ok) {
            dach_group_free(G.release());
            return DACH_CUDA_ERROR;
        }
        *out = G.release();
        return DACH_OK;
    });
}

int dach_group_export(const dach_group* G, void* handle) {
    if (!G || !handle) return DACH_INVALID_ARGUMENT;
    DeviceGuard g(G->device);
    if (!g.ok) return DACH_CUDA_ERROR;
    GroupHandle h;
    memset(&h, 0, sizeof(h));
    h.pid = (uint64_t)getpid();
    h.device = G->device;
    h.rank = G->rank;
    h.ctl_ptr = (uint64_t)(uintptr_t)G->ctl;
    if (!cuda_ok(cudaIpcGetMemHandle(&h.ctl, G->ctl), "cudaIpcGetMemHandle")) return DACH_CUDA_ERROR;
    if (G->rank == 0) {
        h.out_ptr = (uint64_t)(uintptr_t)G->out;
        h.offs_ptr = (uint64_t)(uintptr_t)G->offs;
        if (!cuda_ok(cudaIpcGetMemHandle(&h.out, G->out), "cudaIpcGetMemHandle") ||
            !cuda_ok(cudaIpcGetMemHandle(&h.offs, G->offs), "cudaIpcGetMemHandle"))
            return DACH_CUDA_ERROR;
    }
    memset(handle, 0, DACH_GROUP_HANDLE_BYTES);
    memcpy(handle, &h, sizeof(h));
    return DACH_OK;
}

int dach_group_connect(dach_group* G, const void* handles) {
    if (!G || !handles) return DACH_INVALID_ARGUMENT;
    return guarded([&]() -> int {
        DeviceGuard g(G->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        const uint64_t me = (uint64_t)getpid();
        auto map = [&](const GroupHandle& h, uint64_t raw, const cudaIpcMemHandle_t& ipc, void** out) -> bool {
            if (h.pid == me) {  // same process: the pointer itself, peer access between the two devices
                if (h.device != G->device) {
                    int can = 0;
                    cudaDeviceCanAccessPeer(&can, G->device, h.device);
                    if (!can) {
                        set_error("shard group: no peer access between the devices");
                        return false;
                    }
                    const cudaError_t e = cudaDeviceEnablePeerAccess(h.device, 0);
                    if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return cuda_ok(e, "cudaDeviceEnablePeerAccess");
                    cudaGetLastError();
                }
                *out = reinterpret_cast<void*>((uintptr_t)raw);
                return true;
            }
            void* p = nullptr;
            if (!cuda_ok(cudaIpcOpenMemHandle(&p, ipc, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle")) return false;
            G->ipc_opened[G->n_ipc++] = p;
            *out = p;
            return true;
        };
        for (int j = 0; j < G->world; ++j) {
            GroupHandle h;
            memcpy(&h, static_cast<const char*>(handles) + (size_t)j * DACH_GROUP_HANDLE_BYTES, sizeof(h));
            if (h.rank != j) {
                set_error("shard group: handles must be in rank order");
                return DACH_INVALID_ARGUMENT;
            }
            if (j == G->rank) {
                G->peers.ctl[j] = G->ctl;
            } else {
                void* p = nullptr;
                if (!map(h, h.ctl_ptr, h.ctl, &p)) return DACH_CUDA_ERROR;
                G->peers.ctl[j] = static_cast<GroupCtl*>(p);
            }
            if (j == 0 && G->rank != 0) {
                void *po = nullptr, *pf = nullptr;
                if (!map(h, h.out_ptr, h.out, &po) || !map(h, h.offs_ptr, h.offs, &pf)) return DACH_CUDA_ERROR;
                G->out = static_cast<dach_match*>(po);
                G->offs = static_cast<uint64_t*>(pf);
            }
        }
        G->connected = true;
        return DACH_OK;
    });
}

int dach_group_place(dach_group* G, dach_job* j, uint64_t hay_base, int last, void* stream) {
    if (!G || !j || !G->connected) {
        set_error("shard group: not connected");
        return DACH_INVALID_ARGUMENT;
    }
    if (j->rk != RK_MATCHES) {
        set_error("no scan to place: the job's last operation was a count, first-match, histogram or mask");
        return DACH_INVALID_ARGUMENT;
    }
    if (hay_base + j->W.job_n > G->n_total) {
        set_error("shard group: haystack range outside the gathered batch");
        return DACH_INVALID_ARGUMENT;
    }
    return guarded([&]() -> int {
        DeviceGuard g(G->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        cudaStream_t st = static_cast<cudaStream_t>(stream);
        Workspace& W = j->W;
        if (!W.job_open) {
            set_error("no scan to place");
            return DACH_INVALID_ARGUMENT;
        }
        const unsigned long long step = ++G->step;
        if (st != W.job_stream) cudaStreamWaitEvent(st, W.ev_scanned, 0);
        // calling for step s says the result of step s-1 has been consumed: its buffers are free again
        if (G->rank == 0 && step > 1) k_group_release<<<1, kMaxRanks, 0, st>>>(G->peers, G->world, step - 1);
        const unsigned long long* total = static_cast<const unsigned long long*>(W.item_offs.p) + W.job_items;
        k_group_publish<<<1, kMaxRanks, 0, st>>>(G->peers, G->world, G->rank, step, total, static_cast<const ScanCtrl*>(W.ctrl.p));
        k_group_wait_base<<<1, 1, 0, st>>>(G->ctl, G->rank, step);
        j->d->launches += 3;
        j->out_cap = G->match_cap;
        const bool staged = G->rank != 0, dma = staged && G->push_dma;
        uint64_t h_base = 0, h_total = 0;
        bool over = false;
        if (dma) {
            // The rank's host learns its base and count (blocks until the rank's scan is done, the lower ranks have
            // published and rank 0 has released the previous result).  Callers that pipeline steps enqueue the next
            // scan BEFORE this call so that the scan stream stays fed.
            cudaMemcpyAsync(&G->h_vals[0], &G->ctl->base[step & 1], 8, cudaMemcpyDeviceToHost, st);
            cudaMemcpyAsync(&G->h_vals[1], total, 8, cudaMemcpyDeviceToHost, st);
            cudaMemcpyAsync(&G->h_vals[2], W.ctrl.p, sizeof(ScanCtrl), cudaMemcpyDeviceToHost, st);
            if (!cuda_ok(cudaStreamSynchronize(st), "shard group: base")) return DACH_CUDA_ERROR;
            h_base = G->h_vals[0];
            h_total = G->h_vals[1];
            // the job's pool or its packed copy was too small for this shard: nothing valid to send (the rank's count
            // is published all the same, so the other ranks' bases stay right and nobody waits for this one)
            over = reinterpret_cast<const ScanCtrl*>(&G->h_vals[2])->overflow != 0 || h_total > W.job_cap;
            if (over) h_total = 0;
        }
        const int rc = enqueue_place(j->d, W, G->out, G->match_cap, G->offs + hay_base, &G->ctl->base[step & 1], last != 0, st, nullptr,
                                     staged, dma, h_base, h_total);
        if (rc) return rc;
        j->unplaced = false;
        k_group_signal_done<<<1, 1, 0, st>>>(G->peers.ctl[0], G->rank, step);
        ++j->d->launches;
        if (!cuda_ok(cudaGetLastError(), "shard group kernels")) return DACH_CUDA_ERROR;
        cudaEventRecord(W.ev_placed, st);  // the job's buffers are free once the done signal is out
        if (over) {
            char buf[200];
            snprintf(buf, sizeof(buf), "shard group: the job's capacity (%llu matches) is too small for this shard (needed %llu)",
                     (unsigned long long)W.job_cap, (unsigned long long)G->h_vals[1]);
            set_error(buf);
            return DACH_OUTPUT_OVERFLOW;
        }
        return DACH_OK;
    });
}

int dach_group_finish(dach_group* G, uint64_t* total, void* stream) {
    if (!G || !G->connected) return DACH_INVALID_ARGUMENT;
    return guarded([&]() -> int {
        DeviceGuard g(G->device);
        if (!g.ok) return DACH_CUDA_ERROR;
        cudaStream_t st = static_cast<cudaStream_t>(stream);
        if (G->rank == 0 && G->step) k_group_wait_all<<<1, 1, 0, st>>>(G->ctl, G->world, G->step);
        cudaMemcpyAsync(G->pinned, G->ctl, sizeof(GroupCtl), cudaMemcpyDeviceToHost, st);
        if (!cuda_ok(cudaStreamSynchronize(st), "shard group finish")) return DACH_CUDA_ERROR;
        if (G->pinned->error) {
            set_error("shard group: a rank did not arrive within 20 s");
            return DACH_CUDA_ERROR;
        }
        const uint64_t sum = G->rank == 0 ? G->pinned->sum[G->step & 1] : 0;
        if (total) *total = sum;
        if (G->rank == 0 && sum > G->match_cap) {
            set_error("shard group: gathered matches exceed the capacity of the result buffer");
            return DACH_OUTPUT_OVERFLOW;
        }
        return DACH_OK;
    });
}

int dach_group_result(const dach_group* G, dach_match** d_out, uint64_t** d_offs) {
    if (!G || G->rank != 0) {
        set_error("shard group: only the gathering rank (0) holds the result");
        return DACH_INVALID_ARGUMENT;
    }
    if (d_out) *d_out = G->out;
    if (d_offs) *d_offs = G->offs;
    return DACH_OK;
}

void dach_group_free(dach_group* G) {
    if (!G) return;
    DeviceGuard g(G->device);
    cudaDeviceSynchronize();
    for (int i = 0; i < G->n_ipc; ++i) cudaIpcCloseMemHandle(G->ipc_opened[i]);
    if (G->rank == 0) {
        cudaFree(G->out);
        cudaFree(G->offs);
    }
    cudaFree(G->ctl);
    if (G->pinned) cudaFreeHost(G->pinned);
    if (G->h_vals) cudaFreeHost(G->h_vals);
    delete G;
}

uint64_t dach_dev_kernel_launches(const dach_dev* d) { return d ? d->launches.load() : 0; }
double dach_dev_last_scan_kernel_ms(const dach_dev* d) { return d ? d->last_scan_ms : 0; }
double dach_dev_last_total_ms(const dach_dev* d) { return d ? d->last_total_ms : 0; }
uint64_t dach_dev_last_h2d_bytes(const dach_dev* d) { return d ? d->last_h2d : 0; }
uint64_t dach_dev_last_d2h_bytes(const dach_dev* d) { return d ? d->last_d2h : 0; }

int dach_dev_set_option(dach_dev* d, const char* name, int64_t value) {
    if (!d || !name) return DACH_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> lk(d->mu);
    const std::string k(name);
    if (k == "hot_records")
        d->opt_hot_records = value;
    else if (k == "threads")
        d->opt_threads = value;
    else if (k == "ctas_per_sm")
        d->opt_ctas_per_sm = value;
    else if (k == "kernel")
        d->opt_kernel = value;
    else if (k == "slice_mib")
        d->opt_slice_mib = value;
    else if (k == "seg_len")
        d->opt_seg_len = value;
    else if (k == "slice_ramp")
        d->opt_slice_ramp = value;
    else if (k == "tail_seg")
        d->opt_tail_seg = value;
    else if (k == "gather_ordered")
        d->opt_gather_ordered = value;
    else if (k == "gather_u")
        d->opt_gather_u = value;
    else if (k == "reserve_sms")
        d->opt_reserve_sms = value;
    else if (k == "smem_pad_kib")
        d->opt_smem_pad_kib = value;
    else if (k == "hot_entries")
        d->opt_hot_entries = value;
    else if (k == "event_queue")
        d->opt_event_queue = value;
    else if (k == "expand_desc")
        d->opt_expand_desc = value;
    else if (k == "expand_u")
        d->opt_expand_u = value;
    else if (k == "hist_smem")
        d->opt_hist_smem = value;
    else if (k == "df_pairs")
        d->opt_df_pairs = value;
    else if (k == "l2_hints") {
        d->opt_l2_hints = value;
        DeviceGuard g(d->device);
        if (!g.ok || !install_policies((int)value)) return DACH_CUDA_ERROR;  // device-wide: all handles on this device
    } else {
        set_error("unknown option " + k);
        return DACH_INVALID_ARGUMENT;
    }
    return DACH_OK;
}

}  // extern "C"
