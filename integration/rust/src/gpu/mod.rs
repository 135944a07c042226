//! `daachorse::gpu`: drop-in twins of the crate's automata whose scans run on an H100.  Same type names, same
//! constructors (`new`, `with_values`), same iterator methods and `MatchKind` gating; construction stays in the crate,
//! the serialized automaton crosses the FFI once, haystacks are scanned by libdaachorse_b200.
//! Not compiled in this repository (it builds without a Rust toolchain).
//!
//! Needs two one-line accessors in the crate, `pub(crate) fn match_kind(&self) -> MatchKind { self.match_kind }`
//! in src/bytewise.rs and src/charwise.rs (the field is private to those modules); `Match`'s fields and
//! `MatchKind::is_standard / is_leftmost` are visible here because this module hangs off the crate root.
pub mod ffi;

use crate::{Match, MatchKind};
use core::ffi::CStr;

#[derive(Debug)]
pub struct GpuError {
    pub code: i32,
    pub message: String,
}

fn last_error() -> String {
    unsafe { CStr::from_ptr(ffi::dach_last_error()) }.to_string_lossy().into_owned()
}

fn check(code: i32) -> Result<(), GpuError> {
    if code == ffi::DACH_OK {
        Ok(())
    } else {
        Err(GpuError { code, message: last_error() })
    }
}

/// Matches of a batch: `matches[offsets[i]..offsets[i + 1]]` belong to haystack i, in the order the
/// crate's iterator yields them.
pub struct BatchMatches {
    pub matches: Vec<Match<u32>>,
    pub offsets: Vec<u64>,
}

struct Device {
    dev: *mut ffi::DachDev,
}
impl Drop for Device {
    fn drop(&mut self) {
        unsafe { ffi::dach_dev_free(self.dev) }
    }
}

fn upload(bytes: &[u8], charwise: bool, device: i32) -> Result<Device, GpuError> {
    let (mut h, mut used, mut dev) = (core::ptr::null_mut(), 0usize, core::ptr::null_mut());
    check(unsafe { ffi::dach_pma_deserialize(bytes.as_ptr(), bytes.len(), charwise as i32, &mut h, &mut used) })?;
    let rc = unsafe { ffi::dach_dev_upload(h, device, &mut dev) };
    unsafe { ffi::dach_pma_free(h) };
    check(rc)?;
    Ok(Device { dev })
}

fn scan<P: AsRef<[u8]>>(dev: &Device, mode: i32, haystacks: &[P]) -> Result<BatchMatches, GpuError> {
    let mut text = Vec::new();
    let mut offs = Vec::with_capacity(haystacks.len() + 1);
    offs.push(0u64);
    for h in haystacks {
        text.extend_from_slice(h.as_ref());
        offs.push(text.len() as u64);
    }
    let mut out_offs = vec![0u64; haystacks.len() + 1];
    let mut cap = (text.len() / 8).max(1024) as u64;
    loop {
        let mut out = vec![ffi::DachMatch::default(); cap as usize];
        let mut needed = 0u64;
        let rc = unsafe {
            ffi::dach_scan_batch_host(dev.dev, mode, text.as_ptr(), offs.as_ptr(), haystacks.len() as u64,
                                      out.as_mut_ptr(), cap, out_offs.as_mut_ptr(), &mut needed)
        };
        match rc {
            ffi::DACH_OK => {
                out.truncate(needed as usize);
                // Match { length, end, value } (src/lib.rs:287-320): length = end - start
                let matches = out
                    .iter()
                    .map(|t| Match { length: (t.end - t.start) as usize, end: t.end as usize, value: t.value })
                    .collect();
                return Ok(BatchMatches { matches, offsets: out_offs });
            }
            ffi::DACH_OUTPUT_OVERFLOW => cap = needed, // eager API: retry with the exact size
            ffi::DACH_MATCH_KIND_MISMATCH => panic!("Error: match_kind mismatch"), // src/bytewise.rs:194-197
            _ => return Err(GpuError { code: rc, message: last_error() }),
        }
    }
}

/// Drop-in for `daachorse::DoubleArrayAhoCorasick<u32>`: same constructors, same iterator methods, same
/// `MatchKind` gating -- `use daachorse::gpu::DoubleArrayAhoCorasick;` is the whole switch.  Construction runs the
/// crate's own builder (src/bytewise/builder.rs) on the host; the serialized automaton crosses the FFI once.
/// The iterator methods scan eagerly on the device and then yield the crate's `Match` sequence; the `*_batch`
/// methods are the throughput interface (many haystacks per call).
pub struct DoubleArrayAhoCorasick {
    pma: crate::DoubleArrayAhoCorasick<u32>,
    dev: Device,
}

impl DoubleArrayAhoCorasick {
    /// src/bytewise.rs:103
    pub fn new<I, P>(patterns: I) -> crate::errors::Result<Self>
    where
        I: IntoIterator<Item = P>,
        P: AsRef<[u8]>,
    {
        Self::from_pma(crate::DoubleArrayAhoCorasick::new(patterns)?, 0)
    }
    /// src/bytewise.rs:145
    pub fn with_values<I, P>(patvals: I) -> crate::errors::Result<Self>
    where
        I: IntoIterator<Item = (P, u32)>,
        P: AsRef<[u8]>,
    {
        Self::from_pma(crate::DoubleArrayAhoCorasick::with_values(patvals)?, 0)
    }
    /// From an automaton any builder of the crate made (`DoubleArrayAhoCorasickBuilder::new().match_kind(..)`),
    /// on CUDA device `device`.
    pub fn from_pma(pma: crate::DoubleArrayAhoCorasick<u32>, device: i32) -> crate::errors::Result<Self> {
        let dev = upload(&pma.serialize(), false, device).map_err(|e| crate::errors::DaachorseError::invalid_argument("gpu", ">=", e.code as isize))?;
        Ok(Self { pma, dev })
    }
    pub fn match_kind(&self) -> MatchKind {
        self.pma.match_kind()
    }
    pub fn heap_bytes(&self) -> usize {
        self.pma.heap_bytes()
    }
    pub fn num_states(&self) -> usize {
        self.pma.num_states()
    }

    fn one<P: AsRef<[u8]>>(&self, mode: i32, haystack: P) -> std::vec::IntoIter<Match<u32>> {
        scan(&self.dev, mode, &[haystack]).expect("GPU scan failed").matches.into_iter()
    }
    /// src/bytewise.rs:190
    pub fn find_iter<P: AsRef<[u8]>>(&self, haystack: P) -> impl Iterator<Item = Match<u32>> {
        assert!(self.match_kind().is_standard(), "Error: match_kind must be standard.");
        self.one(ffi::DACH_FIND, haystack)
    }
    /// src/bytewise.rs:292
    pub fn find_overlapping_iter<P: AsRef<[u8]>>(&self, haystack: P) -> impl Iterator<Item = Match<u32>> {
        assert!(self.match_kind().is_standard(), "Error: match_kind must be standard.");
        self.one(ffi::DACH_FIND_OVERLAPPING, haystack)
    }
    /// src/bytewise.rs:410
    pub fn find_overlapping_no_suffix_iter<P: AsRef<[u8]>>(&self, haystack: P) -> impl Iterator<Item = Match<u32>> {
        assert!(self.match_kind().is_standard(), "Error: match_kind must be standard.");
        self.one(ffi::DACH_FIND_OVERLAPPING_NO_SUFFIX, haystack)
    }
    /// src/bytewise.rs:547
    pub fn leftmost_find_iter<P: AsRef<[u8]>>(&self, haystack: P) -> impl Iterator<Item = Match<u32>> {
        assert!(self.match_kind().is_leftmost(), "Error: match_kind must be leftmost.");
        self.one(ffi::DACH_LEFTMOST_FIND, haystack)
    }

    /// Batch forms: haystack i's matches are `matches[offsets[i]..offsets[i + 1]]`, in iterator order.
    pub fn find_batch<P: AsRef<[u8]>>(&self, h: &[P]) -> Result<BatchMatches, GpuError> {
        assert!(self.match_kind().is_standard(), "Error: match_kind must be standard.");
        scan(&self.dev, ffi::DACH_FIND, h)
    }
    pub fn find_overlapping_batch<P: AsRef<[u8]>>(&self, h: &[P]) -> Result<BatchMatches, GpuError> {
        assert!(self.match_kind().is_standard(), "Error: match_kind must be standard.");
        scan(&self.dev, ffi::DACH_FIND_OVERLAPPING, h)
    }
    pub fn find_overlapping_no_suffix_batch<P: AsRef<[u8]>>(&self, h: &[P]) -> Result<BatchMatches, GpuError> {
        assert!(self.match_kind().is_standard(), "Error: match_kind must be standard.");
        scan(&self.dev, ffi::DACH_FIND_OVERLAPPING_NO_SUFFIX, h)
    }
    pub fn leftmost_find_batch<P: AsRef<[u8]>>(&self, h: &[P]) -> Result<BatchMatches, GpuError> {
        assert!(self.match_kind().is_leftmost(), "Error: match_kind must be leftmost.");
        scan(&self.dev, ffi::DACH_LEFTMOST_FIND, h)
    }
}

/// Drop-in for `daachorse::CharwiseDoubleArrayAhoCorasick<u32>` (haystacks are `&str`: valid UTF-8).
pub struct CharwiseDoubleArrayAhoCorasick {
    pma: crate::CharwiseDoubleArrayAhoCorasick<u32>,
    dev: Device,
}

impl CharwiseDoubleArrayAhoCorasick {
    /// src/charwise.rs:100
    pub fn new<I, P>(patterns: I) -> crate::errors::Result<Self>
    where
        I: IntoIterator<Item = P>,
        P: AsRef<str>,
    {
        Self::from_pma(crate::CharwiseDoubleArrayAhoCorasick::new(patterns)?, 0)
    }
    /// src/charwise.rs:139
    pub fn with_values<I, P>(patvals: I) -> crate::errors::Result<Self>
    where
        I: IntoIterator<Item = (P, u32)>,
        P: AsRef<str>,
    {
        Self::from_pma(crate::CharwiseDoubleArrayAhoCorasick::with_values(patvals)?, 0)
    }
    pub fn from_pma(pma: crate::CharwiseDoubleArrayAhoCorasick<u32>, device: i32) -> crate::errors::Result<Self> {
        let dev = upload(&pma.serialize(), true, device).map_err(|e| crate::errors::DaachorseError::invalid_argument("gpu", ">=", e.code as isize))?;
        Ok(Self { pma, dev })
    }
    pub fn match_kind(&self) -> MatchKind {
        self.pma.match_kind()
    }
    fn one(&self, mode: i32, haystack: &str) -> std::vec::IntoIter<Match<u32>> {
        scan(&self.dev, mode, &[haystack]).expect("GPU scan failed").matches.into_iter()
    }
    /// src/charwise.rs:184
    pub fn find_iter<P: AsRef<str>>(&self, haystack: P) -> impl Iterator<Item = Match<u32>> {
        assert!(self.match_kind().is_standard(), "Error: match_kind must be standard.");
        self.one(ffi::DACH_FIND, haystack.as_ref())
    }
    /// src/charwise.rs:290
    pub fn find_overlapping_iter<P: AsRef<str>>(&self, haystack: P) -> impl Iterator<Item = Match<u32>> {
        assert!(self.match_kind().is_standard(), "Error: match_kind must be standard.");
        self.one(ffi::DACH_FIND_OVERLAPPING, haystack.as_ref())
    }
    /// src/charwise.rs:412
    pub fn find_overlapping_no_suffix_iter<P: AsRef<str>>(&self, haystack: P) -> impl Iterator<Item = Match<u32>> {
        assert!(self.match_kind().is_standard(), "Error: match_kind must be standard.");
        self.one(ffi::DACH_FIND_OVERLAPPING_NO_SUFFIX, haystack.as_ref())
    }
    /// src/charwise.rs:553
    pub fn leftmost_find_iter<P: AsRef<str>>(&self, haystack: P) -> impl Iterator<Item = Match<u32>> {
        assert!(self.match_kind().is_leftmost(), "Error: match_kind must be leftmost.");
        self.one(ffi::DACH_LEFTMOST_FIND, haystack.as_ref())
    }
    pub fn find_batch(&self, h: &[&str]) -> Result<BatchMatches, GpuError> {
        assert!(self.match_kind().is_standard(), "Error: match_kind must be standard.");
        scan(&self.dev, ffi::DACH_FIND, h)
    }
    pub fn find_overlapping_batch(&self, h: &[&str]) -> Result<BatchMatches, GpuError> {
        assert!(self.match_kind().is_standard(), "Error: match_kind must be standard.");
        scan(&self.dev, ffi::DACH_FIND_OVERLAPPING, h)
    }
    pub fn find_overlapping_no_suffix_batch(&self, h: &[&str]) -> Result<BatchMatches, GpuError> {
        assert!(self.match_kind().is_standard(), "Error: match_kind must be standard.");
        scan(&self.dev, ffi::DACH_FIND_OVERLAPPING_NO_SUFFIX, h)
    }
    pub fn leftmost_find_batch(&self, h: &[&str]) -> Result<BatchMatches, GpuError> {
        assert!(self.match_kind().is_leftmost(), "Error: match_kind must be leftmost.");
        scan(&self.dev, ffi::DACH_LEFTMOST_FIND, h)
    }
}

/// Many streams scanned chunk after chunk: the batch form of `find_overlapping_stepper()`
/// (src/bytewise.rs:660-729).  `state[i]` / `pos[i]` are stream i's `state_id` / `pos` and live in device
/// memory (allocated by the caller's CUDA binding); each call consumes one chunk per stream.
pub struct StreamScanner<'a> {
    pub pma: &'a DoubleArrayAhoCorasick,
}

impl StreamScanner<'_> {
    /// # Safety
    /// All pointers are device pointers of the sizes `dach_dev_scan_stream` documents.
    pub unsafe fn consume_chunks(&self, d_text: *const u8, d_offs: *const u64, n: u64, text_bytes: u64,
                                 d_state: *mut u32, d_pos: *const u32, d_out: *mut ffi::DachMatch, out_cap: u64,
                                 d_out_offs: *mut u64, stream: *mut core::ffi::c_void) -> Result<u64, GpuError> {
        let mut needed = 0u64;
        check(ffi::dach_dev_scan_stream(self.pma.dev.dev, ffi::DACH_FIND_OVERLAPPING, d_text, d_offs, n, text_bytes,
                                        d_state, d_pos, d_out, out_cap, d_out_offs, &mut needed, stream))?;
        Ok(needed)
    }
}
