//! `extern "C"` declarations of libdaachorse_b200 (include/daachorse_b200.h, ABI version 2).
//! Not compiled in this repository (it builds without a Rust toolchain).
#![allow(non_camel_case_types)]
use core::ffi::{c_char, c_void};

#[repr(C)]
#[derive(Clone, Copy, Debug, Default, PartialEq, Eq)]
pub struct DachMatch {
    pub start: u32,
    pub end: u32,
    pub value: u32,
}

#[repr(C)]
pub struct DachPma {
    _private: [u8; 0],
}
#[repr(C)]
pub struct DachDev {
    _private: [u8; 0],
}
#[repr(C)]
pub struct DachJob {
    _private: [u8; 0],
}
#[repr(C)]
pub struct DachGroup {
    _private: [u8; 0],
}
pub const DACH_GROUP_HANDLE_BYTES: usize = 256;

// status codes
pub const DACH_OK: i32 = 0;
pub const DACH_INVALID_ARGUMENT: i32 = 1;
pub const DACH_AUTOMATON_SCALE: i32 = 2;
pub const DACH_INVALID_CONVERSION: i32 = 3;
pub const DACH_INVALID_AUTOMATON: i32 = 4;
pub const DACH_MATCH_KIND_MISMATCH: i32 = 5;
pub const DACH_OUTPUT_OVERFLOW: i32 = 6;
pub const DACH_CUDA_ERROR: i32 = 7;

// scan modes == the iterator being reproduced
pub const DACH_FIND: i32 = 0; // find_iter                       src/bytewise.rs:190
pub const DACH_FIND_OVERLAPPING: i32 = 1; // find_overlapping_iter           src/bytewise.rs:292
pub const DACH_FIND_OVERLAPPING_NO_SUFFIX: i32 = 2; // find_overlapping_no_suffix_iter src/bytewise.rs:410
pub const DACH_LEFTMOST_FIND: i32 = 3; // leftmost_find_iter              src/bytewise.rs:547

#[link(name = "daachorse_b200")]
extern "C" {
    pub fn dach_abi_version() -> i32;
    pub fn dach_last_error() -> *const c_char;

    /// Parses the crate's own `serialize()` bytes (src/bytewise.rs:801-820, src/charwise.rs:831-848)
    /// with the validation of `deserialize()` (src/bytewise.rs:892-962, src/charwise.rs:912-950).
    pub fn dach_pma_deserialize(src: *const u8, len: usize, charwise: i32, out: *mut *mut DachPma,
                                consumed: *mut usize) -> i32;
    pub fn dach_pma_free(pma: *mut DachPma);

    pub fn dach_dev_upload(pma: *const DachPma, device: i32, out: *mut *mut DachDev) -> i32;
    pub fn dach_dev_free(dev: *mut DachDev);

    /// Host buffers in, host buffers out.
    pub fn dach_scan_batch_host(dev: *mut DachDev, mode: i32, text: *const u8, offs: *const u64, n: u64,
                                out: *mut DachMatch, out_cap: u64, out_offs: *mut u64, needed: *mut u64) -> i32;
    /// Device-resident buffers.
    pub fn dach_dev_scan_batch(dev: *mut DachDev, mode: i32, d_text: *const u8, d_offs: *const u64, n: u64,
                               text_bytes: u64, d_out: *mut DachMatch, out_cap: u64, d_out_offs: *mut u64,
                               needed: *mut u64, stream: *mut c_void) -> i32;
    /// Batch form of find_stepper() / find_overlapping_stepper() (src/bytewise.rs:627-729): haystack i is
    /// the next chunk of stream i; d_state (n x u32, in/out) is the stepper's state_id, d_pos (n x u32 or
    /// null) its pos at the chunk's first byte.
    pub fn dach_dev_scan_stream(dev: *mut DachDev, mode: i32, d_text: *const u8, d_offs: *const u64, n: u64,
                                text_bytes: u64, d_state: *mut u32, d_pos: *const u32, d_out: *mut DachMatch,
                                out_cap: u64, d_out_offs: *mut u64, needed: *mut u64, stream: *mut c_void) -> i32;

    /// Asynchronous two-phase scans with their own workspace: scan and place only enqueue, wait blocks.
    pub fn dach_job_create(dev: *mut DachDev, out: *mut *mut DachJob) -> i32;
    pub fn dach_job_free(job: *mut DachJob);
    pub fn dach_job_scan(job: *mut DachJob, mode: i32, d_text: *const u8, d_offs: *const u64, n: u64, text_bytes: u64,
                         cap_matches: u64, stream: *mut c_void) -> i32;
    pub fn dach_job_place(job: *mut DachJob, d_out: *mut DachMatch, out_cap: u64, d_out_offs: *mut u64, d_base: *const u64,
                          stream: *mut c_void) -> i32;
    pub fn dach_job_wait(job: *mut DachJob, needed: *mut u64) -> i32;

    /// Shard groups: every rank's placement stores its matches into rank 0's dense buffer over NVLink peer memory.
    pub fn dach_group_create(rank: i32, world: i32, device: i32, match_cap: u64, n_haystacks_total: u64,
                             out: *mut *mut DachGroup) -> i32;
    pub fn dach_group_export(group: *const DachGroup, handle: *mut c_void) -> i32;
    pub fn dach_group_connect(group: *mut DachGroup, handles: *const c_void) -> i32;
    pub fn dach_group_place(group: *mut DachGroup, job: *mut DachJob, hay_base: u64, last: i32, stream: *mut c_void) -> i32;
    pub fn dach_group_finish(group: *mut DachGroup, total: *mut u64, stream: *mut c_void) -> i32;
    pub fn dach_group_result(group: *const DachGroup, d_out: *mut *mut DachMatch, d_offs: *mut *mut u64) -> i32;
    pub fn dach_group_free(group: *mut DachGroup);
}
