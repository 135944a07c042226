"""Host-side mirror of the crate's public interface for the scan path.

Names, argument meaning and error behaviour follow daac-tools/daachorse 4.0.0
(file:line relative to the crate root):

    DoubleArrayAhoCorasick            src/bytewise.rs:54-68   (new :103, with_values :145,
        find_iter :190, find_overlapping_iter :292, find_overlapping_no_suffix_iter :410,
        leftmost_find_iter :547, match_kind :747, heap_bytes :764, num_states :785,
        serialize :801, deserialize :868)
    DoubleArrayAhoCorasickBuilder     src/bytewise/builder.rs:21-244
    CharwiseDoubleArrayAhoCorasick    src/charwise.rs:59-65 (same surface + num_elements :796)
    CharwiseDoubleArrayAhoCorasickBuilder  src/charwise/builder.rs
    MatchKind                         src/lib.rs:324-346
    Match                             src/lib.rs:287-320

Construction runs on the host inside libdaachorse_b200.so; every scan runs on the GPU
through the C ABI (include/daachorse_b200.h).  There is no CPU scan path: without a CUDA
device the scan methods raise DaachorseError(CUDA_ERROR).

The crate's iterators are lazy; here an iterator call scans the haystack eagerly on the
device and then yields the same Match sequence.  The ``*_batch`` methods are the
throughput interface (many haystacks per call).

Streams: every ``*_device`` form takes ``stream=`` -- ``None`` (the current stream of the text's
device), a torch stream, or a raw ``cudaStream_t`` handle (int).  A stream other than the current
one is made to wait for the work queued so far on the current stream before each library call, so
the inputs written there and the outputs the wrapper allocates there are ready; the call
synchronises its stream before it returns, so its results may be used on the current stream.
"""
import ctypes as C
import enum
import threading

import numpy as np

from . import _lib

MATCH_DTYPE = np.dtype([("start", "<u4"), ("end", "<u4"), ("value", "<u4")])

FIND, FIND_OVERLAPPING, FIND_OVERLAPPING_NO_SUFFIX, LEFTMOST_FIND = range(4)
HIST_KEYS = {"output": 0, "value": 1}  # dach_hist_key


class MatchKind(enum.IntEnum):
    """src/lib.rs:324-346"""
    Standard = 0
    LeftmostLongest = 1
    LeftmostFirst = 2


class DaachorseError(Exception):
    """Mirror of errors::DaachorseError (src/errors.rs:10-22); ``code`` is the dach_status."""

    NAMES = {1: "InvalidArgument", 2: "AutomatonScale", 3: "InvalidConversion", 4: "InvalidAutomaton",
             5: "MatchKindMismatch", 6: "OutputOverflow", 7: "CudaError"}

    def __init__(self, code, msg=""):
        super().__init__("%s: %s" % (self.NAMES.get(code, code), msg))
        self.code = code


def _check(rc):
    if rc == _lib.OK:
        return
    msg = _lib.last_error()
    if rc == _lib.MATCH_KIND_MISMATCH:
        # the crate panics: assert!(self.match_kind.is_standard(), ...) (src/bytewise.rs:194-197)
        raise AssertionError(msg)
    raise DaachorseError(rc, msg)


class Match:
    """src/lib.rs:287-320: start() / end() / value()."""
    __slots__ = ("_s", "_e", "_v")

    def __init__(self, start, end, value):
        self._s, self._e, self._v = int(start), int(end), int(value)

    def start(self):
        return self._s

    def end(self):
        return self._e

    def value(self):
        return self._v

    def __eq__(self, o):
        return isinstance(o, Match) and (self._s, self._e, self._v) == (o._s, o._e, o._v)

    def __hash__(self):
        return hash((self._s, self._e, self._v))

    def __repr__(self):
        return "Match { start: %d, end: %d, value: %d }" % (self._s, self._e, self._v)


class BatchResult:
    """Matches of a batch: ``matches`` (structured array start/end/value, or an (n,3) torch
    tensor for device-resident scans) and ``offsets`` (n+1) delimiting each haystack's run."""

    def __init__(self, matches, offsets):
        self.matches = matches
        self.offsets = offsets

    def __len__(self):
        return len(self.offsets) - 1

    def triples(self, i):
        lo, hi = int(self.offsets[i]), int(self.offsets[i + 1])
        m = self.matches[lo:hi]
        if isinstance(m, np.ndarray):
            return [(int(a), int(b), int(c)) for a, b, c in zip(m["start"], m["end"], m["value"])]
        return [tuple(int(x) for x in row) for row in m.cpu().tolist()]


def _pack(items, as_str):
    bs = []
    for p in items:
        if isinstance(p, str):
            bs.append(p.encode("utf-8"))
        else:
            if as_str:
                # the charwise crate API takes &str: reject invalid UTF-8 early
                bytes(p).decode("utf-8")
            bs.append(bytes(p))
    offs = np.zeros(len(bs) + 1, dtype=np.uint64)
    if bs:
        offs[1:] = np.cumsum([len(b) for b in bs], dtype=np.uint64)
    blob = np.frombuffer(b"".join(bs), dtype=np.uint8) if bs else np.zeros(0, dtype=np.uint8)
    return blob, offs


def _ptr(a):
    return C.c_void_p(a.ctypes.data) if a.size else None


def _stream_handle(stream, device):
    """The raw cudaStream_t of ``stream``: None = the current stream of ``device``, a torch stream, or a handle."""
    import torch

    if stream is None:
        return torch.cuda.current_stream(device).cuda_stream
    return int(stream.cuda_stream) if hasattr(stream, "cuda_stream") else int(stream)


def _wait_stream(handle, current, device):
    """Stream ``handle`` waits for the work queued so far on ``current``."""
    import torch

    torch.cuda.ExternalStream(handle, device=device).wait_stream(current)


def _ordered_stream(stream, device):
    """``stream`` as a ctypes handle, ordered after the current stream of ``device`` when it is another stream: the
    wrappers allocate and fill on the current stream, and the caller's inputs were written there.  Called right
    before every library call, retries included.  The same stream costs nothing."""
    import torch

    handle = _stream_handle(stream, device)
    current = torch.cuda.current_stream(device)
    if handle != current.cuda_stream:
        _wait_stream(handle, current, device)
    return C.c_void_p(handle)


def _torch_stream(stream, device):
    """``stream`` (None, a torch stream or a raw handle) as a torch stream object, for ``record_stream``."""
    import torch

    if stream is None:
        return torch.cuda.current_stream(device)
    if isinstance(stream, torch.cuda.Stream):
        return stream
    return torch.cuda.ExternalStream(_stream_handle(stream, device), device=device)


class _Automaton:
    """Shared implementation of the two automaton classes."""

    _charwise = False

    def __init__(self, handle):
        self._h = handle
        self._devs = {}
        self._devs_lock = threading.Lock()  # one upload per device, whichever thread calls first

    # -- construction ----------------------------------------------------------------------
    @classmethod
    def _build(cls, patterns, values, match_kind, num_free_blocks):
        L = _lib.load()
        blob, offs = _pack(list(patterns), cls._charwise)
        n = len(offs) - 1
        vals = None
        if values is not None:
            for v in values:
                if not (0 <= int(v) <= 0xFFFFFFFF):
                    # V::try_from(i) failed (src/bytewise/builder.rs:160-165)
                    raise DaachorseError(_lib.INVALID_CONVERSION, "value does not fit u32")
            vals = np.ascontiguousarray(values, dtype=np.uint32)
            if vals.size != n:
                raise DaachorseError(_lib.INVALID_ARGUMENT, "one value per pattern expected")
        h = C.c_void_p()
        f = L.dach_charwise_build if cls._charwise else L.dach_bytewise_build
        _check(f(_ptr(blob), C.c_void_p(offs.ctypes.data), None if vals is None else _ptr(vals), n,
                 int(match_kind), int(num_free_blocks), C.byref(h)))
        return cls(h)

    @classmethod
    def new(cls, patterns):
        """``new(patterns)``: value i is associated with patterns[i]."""
        return cls._build(patterns, None, MatchKind.Standard, 16)

    @classmethod
    def with_values(cls, patvals):
        """``with_values([(pattern, value), ...])``"""
        patvals = list(patvals)
        return cls._build([p for p, _ in patvals], [v for _, v in patvals], MatchKind.Standard, 16)

    @classmethod
    def deserialize(cls, source):
        """Returns (automaton, remaining bytes) like the crate's ``deserialize``."""
        L = _lib.load()
        buf = np.frombuffer(bytes(source), dtype=np.uint8)
        h = C.c_void_p()
        used = C.c_size_t()
        _check(L.dach_pma_deserialize(_ptr(buf), buf.size, int(cls._charwise), C.byref(h), C.byref(used)))
        return cls(h), bytes(source)[used.value:]

    # deserialize_unchecked (src/bytewise.rs:1009) maps to the checked loader on purpose
    deserialize_unchecked = deserialize

    def __del__(self):
        try:
            L = _lib.load()
            for d in self._devs.values():
                L.dach_dev_free(d)
            self._devs = {}
            if self._h:
                L.dach_pma_free(self._h)
                self._h = None
        except Exception:
            pass

    # -- introspection ------------------------------------------------------------------------
    def match_kind(self):
        return MatchKind(_lib.load().dach_pma_match_kind(self._h))

    def heap_bytes(self):
        return _lib.load().dach_pma_heap_bytes(self._h)

    def num_states(self):
        return _lib.load().dach_pma_num_states(self._h)

    def num_elements(self):
        return _lib.load().dach_pma_num_elements(self._h)

    def max_pattern_len(self):
        return _lib.load().dach_pma_max_pattern_len(self._h)

    def outputs(self):
        """The output records as numpy uint32 arrays ``(values, lengths, parents)``: one record per pattern the builder
        kept (duplicates get one each); parent 0 = none, else the parent's 1-based index.  Index i labels bin i of a
        ``key="output"`` histogram."""
        L = _lib.load()
        k = int(L.dach_pma_num_outputs(self._h))
        vals, lens, pars = (np.zeros(max(k, 1), dtype=np.uint32) for _ in range(3))
        _check(L.dach_pma_outputs(self._h, _ptr(vals), _ptr(lens), _ptr(pars), k))
        return vals[:k], lens[:k], pars[:k]

    def _hist_len(self, key):
        if key not in HIST_KEYS:
            raise DaachorseError(_lib.INVALID_ARGUMENT, "key must be 'value' or 'output'")
        vals = self.outputs()[0]
        if key == "output":
            return len(vals)
        return int(vals.max()) + 1 if len(vals) else 0

    def serialize(self):
        L = _lib.load()
        n = L.dach_pma_serialized_bytes(self._h)
        buf = np.zeros(max(n, 1), dtype=np.uint8)
        w = C.c_size_t()
        _check(L.dach_pma_serialize(self._h, C.c_void_p(buf.ctypes.data), n, C.byref(w)))
        return buf[:n].tobytes()

    # -- device ---------------------------------------------------------------------------------
    def device_handle(self, device=None):
        """Uploads the scan image to ``device`` once (default: the current CUDA device), also when several host
        threads make their first call at the same time: they all get the one handle."""
        L = _lib.load()
        if device is None:
            device = _current_device()
        with self._devs_lock:
            d = self._devs.get(device)
            if d is None:
                d = C.c_void_p()
                _check(L.dach_dev_upload(self._h, int(device), C.byref(d)))
                self._devs[device] = d
        return d

    def set_option(self, name, value, device=None):
        _check(_lib.load().dach_dev_set_option(self.device_handle(device), name.encode(), int(value)))

    def stats(self, device=None):
        L = _lib.load()
        d = self.device_handle(device)
        return {"launches": L.dach_dev_kernel_launches(d), "scan_kernel_ms": L.dach_dev_last_scan_kernel_ms(d),
                "total_ms": L.dach_dev_last_total_ms(d), "h2d_bytes": L.dach_dev_last_h2d_bytes(d),
                "d2h_bytes": L.dach_dev_last_d2h_bytes(d), "image_bytes": L.dach_dev_image_bytes(d)}

    def _assert_mode(self, mode):
        lm = self.match_kind() != MatchKind.Standard
        if (mode == LEFTMOST_FIND) != lm:
            raise AssertionError("Error: match_kind must be %s." % ("standard" if lm else "leftmost"))

    # -- batch scans ----------------------------------------------------------------------------
    def scan_batch_host(self, mode, text, offs, out_cap=None, device=None, out=None, out_offs=None):
        """Host buffers in, host buffers out (numpy).  ``text`` uint8, ``offs`` uint64 (n+1).
        ``out`` (MATCH_DTYPE) / ``out_offs`` (uint64, n+1) may be preallocated -- e.g. views of pinned
        memory -- to keep allocation and page faults out of the call."""
        self._assert_mode(mode)
        L = _lib.load()
        d = self.device_handle(device)
        text = np.ascontiguousarray(text, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        n = len(offs) - 1
        if n < 0 or (n > 0 and int(offs.max()) > text.size):
            raise DaachorseError(_lib.INVALID_ARGUMENT, "offsets must hold n + 1 entries and stay inside the text")
        if out is not None and (out.dtype != MATCH_DTYPE or not out.flags.c_contiguous):
            raise DaachorseError(_lib.INVALID_ARGUMENT, "out must be a contiguous MATCH_DTYPE array")
        if out_offs is not None and (out_offs.dtype != np.uint64 or not out_offs.flags.c_contiguous or len(out_offs) < n + 1):
            raise DaachorseError(_lib.INVALID_ARGUMENT, "out_offs must be a contiguous uint64 array of n + 1 entries")
        if out is not None:
            cap = len(out)
        else:
            cap = int(out_cap) if out_cap else max(1024, int(text.size // 8))
        if out_offs is None:
            out_offs = np.empty(n + 1, dtype=np.uint64)
        while True:
            if out is None or len(out) < cap:
                out = np.empty(cap, dtype=MATCH_DTYPE)
            need = C.c_uint64()
            rc = L.dach_scan_batch_host(d, mode, _ptr(text), C.c_void_p(offs.ctypes.data), n,
                                        C.c_void_p(out.ctypes.data), len(out), C.c_void_p(out_offs.ctypes.data),
                                        C.byref(need))
            if rc == _lib.OUTPUT_OVERFLOW:
                if int(need.value) <= len(out):
                    raise DaachorseError(rc, "overflow reported although capacity %d >= needed %d" % (len(out), need.value))
                cap = int(need.value)
                out = None
                continue
            _check(rc)
            return BatchResult(out[: need.value], out_offs[: n + 1])

    def scan_batch_device(self, mode, text, offs, out=None, out_offs=None, stream=None):
        """Device-resident scan.  ``text`` (uint8) and ``offs`` (int64/uint64, n+1) are CUDA torch
        tensors; returns BatchResult with an (total, 3) int32-typed view of u32 triples and an
        int64 offsets tensor, both on the device.  ``out``: optional preallocated (cap, 3) int32.  ``stream``: None, a
        torch stream or a raw handle; another stream than the current one is ordered after the current one (module
        docstring), and the call synchronises it before it returns."""
        import torch

        self._assert_mode(mode)
        L = _lib.load()
        dev = text.device.index if text.device.index is not None else torch.cuda.current_device()
        _check_device_batch(text, offs, dev, out, out_offs)
        d = self.device_handle(dev)
        n = offs.numel() - 1
        if out_offs is None:
            out_offs = torch.empty(n + 1, dtype=torch.int64, device=text.device)
        cap = out.shape[0] if out is not None else max(1024, int(text.numel() // 8))
        while True:
            if out is None or out.shape[0] < cap:
                out = torch.empty((cap, 3), dtype=torch.int32, device=text.device)
            need = C.c_uint64()
            rc = L.dach_dev_scan_batch(d, mode, C.c_void_p(text.data_ptr()), C.c_void_p(offs.data_ptr()), n,
                                       text.numel(), C.c_void_p(out.data_ptr()), out.shape[0],
                                       C.c_void_p(out_offs.data_ptr()), C.byref(need), _ordered_stream(stream, text.device))
            if rc == _lib.OUTPUT_OVERFLOW:
                if int(need.value) <= cap:
                    raise DaachorseError(rc, "overflow reported although capacity %d >= needed %d" % (cap, need.value))
                cap = int(need.value)
                out = None
                continue
            _check(rc)
            return BatchResult(out[: need.value], out_offs)

    def scan_stream_device(self, mode, text, offs, state, pos=None, out=None, out_offs=None, stream=None):
        """Chunks of streams -- the batch form of ``find_stepper()`` / ``find_overlapping_stepper()``
        (src/bytewise.rs:627-729): haystack i is the next chunk of stream i.  ``state`` (CUDA int32/uint32,
        n entries) holds each stream's state id and is updated in place; ``pos`` (optional, n entries) is
        the stream position of each chunk's first byte and is added to the reported positions.  For every
        byte: consume(byte), then matches().  Returns a BatchResult of device tensors.  ``stream`` as in
        ``scan_batch_device``: the copy of ``state`` an overflow retry restarts from is taken on the current stream,
        before the call."""
        import torch

        self._assert_mode(mode)
        L = _lib.load()
        dev = text.device.index if text.device.index is not None else torch.cuda.current_device()
        _check_device_batch(text, offs, dev, out, out_offs, state, pos)
        d = self.device_handle(dev)
        n = offs.numel() - 1
        if out_offs is None:
            out_offs = torch.empty(n + 1, dtype=torch.int64, device=text.device)
        cap = out.shape[0] if out is not None else max(1024, int(text.numel() // 8))
        state_in = state.clone()  # the call advances `state` even when the output overflows
        while True:
            if out is None or out.shape[0] < cap:
                out = torch.empty((cap, 3), dtype=torch.int32, device=text.device)
            need = C.c_uint64()
            rc = L.dach_dev_scan_stream(d, mode, C.c_void_p(text.data_ptr()), C.c_void_p(offs.data_ptr()), n, text.numel(),
                                        C.c_void_p(state.data_ptr()), C.c_void_p(pos.data_ptr()) if pos is not None else None,
                                        C.c_void_p(out.data_ptr()), out.shape[0], C.c_void_p(out_offs.data_ptr()),
                                        C.byref(need), _ordered_stream(stream, text.device))
            if rc == _lib.OUTPUT_OVERFLOW:
                if int(need.value) <= cap:
                    raise DaachorseError(rc, "overflow reported although capacity %d >= needed %d" % (cap, need.value))
                cap = int(need.value)
                out = None
                state.copy_(state_in)
                continue
            _check(rc)
            return BatchResult(out[: need.value], out_offs)

    # -- stream chunks without a match list -------------------------------------------------------
    # ``state`` is read and updated in place exactly as ``scan_stream_device`` does it, so calls of every kind may
    # take turns on one stream.  Nothing can overflow: one call per round, no copy of the state.
    def _stream_args(self, mode, text):
        import torch

        self._assert_mode(mode)
        dev = text.device.index if text.device.index is not None else torch.cuda.current_device()
        return dev, self.device_handle(dev)

    def count_stream_device(self, mode, text, offs, state, out=None, stream=None):
        """Matches per chunk of ``scan_stream_device`` without the matches: an int64 CUDA tensor of n counts
        (``out``: optional preallocated one), ``state`` advanced in place."""
        import torch

        dev, d = self._stream_args(mode, text)
        n = offs.numel() - 1
        if out is None and n >= 0:
            out = torch.empty(n, dtype=torch.int64, device=text.device)
        _check_device_batch(text, offs, dev, state=state, counts=out)
        total = C.c_uint64()
        _check(_lib.load().dach_dev_count_stream(d, mode, C.c_void_p(text.data_ptr()), C.c_void_p(offs.data_ptr()), n, text.numel(),
                                                 C.c_void_p(state.data_ptr()), C.c_void_p(out.data_ptr()), C.byref(total),
                                                 _ordered_stream(stream, text.device)))
        return out

    def first_stream_device(self, mode, text, offs, state, pos=None, out=None, found=None, stream=None):
        """The first match ``scan_stream_device`` reports for each chunk: ``(first, found)`` CUDA tensors as in
        ``first_batch_device``, positions plus ``pos`` (modulo 2^32; chunk-relative without it), ``state`` advanced
        in place.  Every chunk is still scanned to its end."""
        import torch

        dev, d = self._stream_args(mode, text)
        n = offs.numel() - 1
        if out is None and n >= 0:
            out = torch.empty((n, 3), dtype=torch.int32, device=text.device)
        if found is None and n >= 0:
            found = torch.empty(n, dtype=torch.bool, device=text.device)
        _check_device_batch(text, offs, dev, state=state, pos=pos, first=out, found=found)
        nf = C.c_uint64()
        _check(_lib.load().dach_dev_first_stream(d, mode, C.c_void_p(text.data_ptr()), C.c_void_p(offs.data_ptr()), n, text.numel(),
                                                 C.c_void_p(state.data_ptr()), C.c_void_p(pos.data_ptr()) if pos is not None else None,
                                                 C.c_void_p(out.data_ptr()), C.c_void_p(found.data_ptr()), C.byref(nf),
                                                 _ordered_stream(stream, text.device)))
        return out, found

    def pattern_counts_stream_device(self, mode, text, offs, state, key="value", out=None, stream=None):
        """``pattern_counts_device`` on chunks of streams: the histogram of this round's matches of
        ``scan_stream_device``, added into ``out`` if given (zeros otherwise), ``state`` advanced in place.  Summed
        over the rounds it is the histogram of the stepper's matches over the whole streams."""
        import torch

        dev, d = self._stream_args(mode, text)
        need = self._hist_len(key)
        if out is None:
            out = torch.zeros(need, dtype=torch.int64, device=text.device)
        _check_device_batch(text, offs, dev, state=state, hist=out, hist_len=need)
        total = C.c_uint64()
        _check(_lib.load().dach_dev_hist_stream(d, mode, HIST_KEYS[key], C.c_void_p(text.data_ptr()), C.c_void_p(offs.data_ptr()),
                                                offs.numel() - 1, text.numel(), C.c_void_p(state.data_ptr()),
                                                C.c_void_p(out.data_ptr()), out.numel(), C.byref(total),
                                                _ordered_stream(stream, text.device)))
        return out

    # -- counts and first matches (no match list) -------------------------------------------------
    def _host_batch_args(self, mode, text, offs):
        self._assert_mode(mode)
        text = np.ascontiguousarray(text, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        n = len(offs) - 1
        if n < 0 or (n > 0 and int(offs.max()) > text.size):
            raise DaachorseError(_lib.INVALID_ARGUMENT, "offsets must hold n + 1 entries and stay inside the text")
        return text, offs, n

    def count_batch_host(self, mode, text, offs, device=None):
        """Matches per haystack of iterator ``mode``, host buffers in and out: ``(np.uint64[n], total)``.
        counts[i] equals the length of haystack i's run in ``scan_batch_host``; nothing is stored per match."""
        text, offs, n = self._host_batch_args(mode, text, offs)
        L = _lib.load()
        d = self.device_handle(device)
        counts = np.zeros(n, dtype=np.uint64)
        total = C.c_uint64()
        _check(L.dach_count_batch_host(d, mode, _ptr(text), C.c_void_p(offs.ctypes.data), n, _ptr(counts), C.byref(total)))
        return counts, int(total.value)

    def first_batch_host(self, mode, text, offs, device=None):
        """First match of iterator ``mode`` on every haystack: ``(MATCH_DTYPE[n], bool[n])``.  Where there is
        none, found is False and the tuple is all-ones.  The scan of a haystack stops at its first match."""
        text, offs, n = self._host_batch_args(mode, text, offs)
        L = _lib.load()
        d = self.device_handle(device)
        first = np.zeros(n, dtype=MATCH_DTYPE)
        found = np.zeros(n, dtype=np.uint8)
        nf = C.c_uint64()
        _check(L.dach_first_batch_host(d, mode, _ptr(text), C.c_void_p(offs.ctypes.data), n, _ptr(first), _ptr(found), C.byref(nf)))
        return first, found.astype(bool)

    def count_batch_device(self, mode, text, offs, out=None, stream=None):
        """Device-resident form of ``count_batch_host``: ``text`` / ``offs`` as in ``scan_batch_device``;
        returns an int64 CUDA tensor of n counts (``out``: optional preallocated one)."""
        import torch

        self._assert_mode(mode)
        dev = text.device.index if text.device.index is not None else torch.cuda.current_device()
        n = offs.numel() - 1
        if out is None and n >= 0:
            out = torch.empty(n, dtype=torch.int64, device=text.device)
        _check_device_batch(text, offs, dev, counts=out)
        d = self.device_handle(dev)
        total = C.c_uint64()
        _check(_lib.load().dach_dev_count_batch(d, mode, C.c_void_p(text.data_ptr()), C.c_void_p(offs.data_ptr()), n, text.numel(),
                                                C.c_void_p(out.data_ptr()), C.byref(total), _ordered_stream(stream, text.device)))
        return out

    def first_batch_device(self, mode, text, offs, out=None, found=None, stream=None):
        """Device-resident form of ``first_batch_host``: returns ``(first, found)`` CUDA tensors -- (n, 3) int32
        carrying the u32 tuples and a bool (n) (``out`` / ``found``: optional preallocated ones)."""
        import torch

        self._assert_mode(mode)
        dev = text.device.index if text.device.index is not None else torch.cuda.current_device()
        n = offs.numel() - 1
        if out is None and n >= 0:
            out = torch.empty((n, 3), dtype=torch.int32, device=text.device)
        if found is None and n >= 0:
            found = torch.empty(n, dtype=torch.bool, device=text.device)
        _check_device_batch(text, offs, dev, first=out, found=found)
        d = self.device_handle(dev)
        nf = C.c_uint64()
        _check(_lib.load().dach_dev_first_batch(d, mode, C.c_void_p(text.data_ptr()), C.c_void_p(offs.data_ptr()), n, text.numel(),
                                                C.c_void_p(out.data_ptr()), C.c_void_p(found.data_ptr()), C.byref(nf), _ordered_stream(stream, text.device)))
        return out, found

    def pattern_counts_host(self, mode, text, offs, key="value", out=None, device=None):
        """How often each pattern occurs in the batch, host buffers in and out: ``np.uint64`` histogram, added into
        ``out`` if given (zeros otherwise).  ``key="value"``: bin = the match's value (a bincount of the values of
        ``scan_batch_host``); ``key="output"``: bin = the match's output record (``outputs()``).  No match list."""
        text, offs, n = self._host_batch_args(mode, text, offs)
        L = _lib.load()
        d = self.device_handle(device)
        need = self._hist_len(key)
        if out is None:
            out = np.zeros(need, dtype=np.uint64)
        elif out.dtype != np.uint64 or out.ndim != 1 or not out.flags.c_contiguous or not out.flags.writeable:
            raise DaachorseError(_lib.INVALID_ARGUMENT, "out must be a writable contiguous 1-d uint64 array")
        total = C.c_uint64()
        _check(L.dach_hist_batch_host(d, mode, HIST_KEYS[key], _ptr(text), C.c_void_p(offs.ctypes.data), n, _ptr(out), out.size,
                                      C.byref(total)))
        return out

    def pattern_counts_device(self, mode, text, offs, key="value", out=None, stream=None):
        """Device-resident form of ``pattern_counts_host``: ``text`` / ``offs`` as in ``scan_batch_device``; returns the
        int64 CUDA histogram, added into ``out`` if given (zeros otherwise) -- calls on consecutive batches accumulate
        a corpus on the device."""
        import torch

        self._assert_mode(mode)
        dev = text.device.index if text.device.index is not None else torch.cuda.current_device()
        need = self._hist_len(key)
        if out is None:
            out = torch.zeros(need, dtype=torch.int64, device=text.device)
        _check_device_batch(text, offs, dev, hist=out, hist_len=need)
        d = self.device_handle(dev)
        total = C.c_uint64()
        _check(_lib.load().dach_dev_hist_batch(d, mode, HIST_KEYS[key], C.c_void_p(text.data_ptr()), C.c_void_p(offs.data_ptr()),
                                               offs.numel() - 1, text.numel(), C.c_void_p(out.data_ptr()), out.numel(),
                                               C.byref(total), _ordered_stream(stream, text.device)))
        return out

    def doc_counts_host(self, mode, text, offs, key="value", out=None, device=None):
        """In how many haystacks of the batch each pattern occurs (document frequency), host buffers in and out:
        ``np.uint64`` counts, added into ``out`` if given (zeros otherwise).  Bin k counts the haystacks with at least
        one match of key k -- keys as in ``pattern_counts_host``.  No match list; on an error ``out`` is unchanged."""
        text, offs, n = self._host_batch_args(mode, text, offs)
        need = self._hist_len(key)
        if out is None:
            out = np.zeros(need, dtype=np.uint64)
        elif out.dtype != np.uint64 or out.ndim != 1 or not out.flags.c_contiguous or not out.flags.writeable:
            raise DaachorseError(_lib.INVALID_ARGUMENT, "out must be a writable contiguous 1-d uint64 array")
        L = _lib.load()
        d = self.device_handle(device)
        total = C.c_uint64()
        _check(L.dach_df_batch_host(d, mode, HIST_KEYS[key], _ptr(text), C.c_void_p(offs.ctypes.data), n, _ptr(out), out.size,
                                    C.byref(total)))
        return out

    def doc_counts_device(self, mode, text, offs, key="value", out=None, stream=None):
        """Device-resident form of ``doc_counts_host``: ``text`` / ``offs`` as in ``scan_batch_device``; returns the
        int64 CUDA counts, added into ``out`` if given (zeros otherwise) -- calls on consecutive batches accumulate a
        corpus on the device."""
        import torch

        self._assert_mode(mode)
        dev = text.device.index if text.device.index is not None else torch.cuda.current_device()
        need = self._hist_len(key)
        if out is None:
            out = torch.zeros(need, dtype=torch.int64, device=text.device)
        _check_device_batch(text, offs, dev, hist=out, hist_len=need)
        d = self.device_handle(dev)
        total = C.c_uint64()
        _check(_lib.load().dach_dev_df_batch(d, mode, HIST_KEYS[key], C.c_void_p(text.data_ptr()), C.c_void_p(offs.data_ptr()),
                                             offs.numel() - 1, text.numel(), C.c_void_p(out.data_ptr()), out.numel(),
                                             C.byref(total), _ordered_stream(stream, text.device)))
        return out

    def last_doc_windows(self, device=None):
        """``(windows, rescans)`` of the last ``doc_counts_*`` call on this device: the windows the batch was scanned
        in, and how many of them overflowed the pair sets (option ``df_pairs``) and were scanned again as halves."""
        w, r = C.c_uint64(), C.c_uint64()
        _check(_lib.load().dach_dev_last_df_windows(self.device_handle(device), C.byref(w), C.byref(r)))
        return w.value, r.value

    # -- masked text (no match list) ----------------------------------------------------------------
    def _fill_byte(self, fill):
        if isinstance(fill, (bytes, str)) and len(fill) == 1:
            fill = ord(fill)
        if isinstance(fill, bool) or not isinstance(fill, (int, np.integer)) or not 0 <= int(fill) <= 255:
            raise DaachorseError(_lib.INVALID_ARGUMENT, "fill must be one byte (an int in 0..255)")
        if self._charwise and fill >= 0x80:
            raise DaachorseError(_lib.INVALID_ARGUMENT, "the fill of a charwise automaton must be ASCII (below 0x80)")
        return int(fill)

    def mask_batch_host(self, mode, text, offs, fill=ord("*"), out=None, device=None):
        """``text`` with every byte a match of iterator ``mode`` covers set to ``fill``, host buffers in and out:
        ``np.uint8`` of ``text``'s size (``out``: optional preallocated one).  Bytes outside the haystacks are copied."""
        fill = self._fill_byte(fill)
        text, offs, n = self._host_batch_args(mode, text, offs)
        if int(offs[-1]) > text.size:  # the copy reads text[0, offs[n]) even when n == 0
            raise DaachorseError(_lib.INVALID_ARGUMENT, "offsets must stay inside the text")
        if out is None:
            out = np.empty(text.size, dtype=np.uint8)
        elif out.dtype != np.uint8 or out.ndim != 1 or out.size < text.size or not out.flags.c_contiguous or not out.flags.writeable:
            raise DaachorseError(_lib.INVALID_ARGUMENT, "out must be a writable contiguous 1-d uint8 array of at least text.size bytes")
        if out.size and text.size and np.shares_memory(out, text):
            raise DaachorseError(_lib.INVALID_ARGUMENT, "out must not overlap text (masking in place is not supported)")
        L = _lib.load()
        d = self.device_handle(device)
        _check(L.dach_mask_batch_host(d, mode, _ptr(text), C.c_void_p(offs.ctypes.data), n, fill, _ptr(out)))
        end = int(offs[-1])
        out[end:text.size] = text[end:]
        return out

    def mask_batch_device(self, mode, text, offs, fill=ord("*"), out=None, stream=None):
        """Device-resident form of ``mask_batch_host``: ``text`` / ``offs`` as in ``scan_batch_device``; returns a uint8
        CUDA tensor of ``text``'s size (``out``: optional preallocated one, which must not overlap ``text``)."""
        import torch

        fill = self._fill_byte(fill)
        self._assert_mode(mode)
        dev = text.device.index if text.device.index is not None else torch.cuda.current_device()
        if out is None:
            out = torch.empty(text.numel(), dtype=torch.uint8, device=text.device)
        _check_device_batch(text, offs, dev, masked=out)
        d = self.device_handle(dev)
        _check(_lib.load().dach_dev_mask_batch(d, mode, C.c_void_p(text.data_ptr()), C.c_void_p(offs.data_ptr()), offs.numel() - 1,
                                               text.numel(), fill, C.c_void_p(out.data_ptr()), _ordered_stream(stream, text.device)))
        return out

    def mask_batch(self, haystacks, fill=b"*", mode=None):
        """Every haystack with the bytes its matches cover replaced by ``fill``: a list of ``bytes``, or of ``str`` for
        a charwise automaton (whose fill must be ASCII); ``mode=None`` as in ``count_batch``."""
        haystacks = list(haystacks)
        fill = self._fill_byte(fill)
        blob, offs = _pack(haystacks, self._charwise)
        masked = self.mask_batch_host(self._default_mode(mode), blob, offs, fill=fill).tobytes()
        res = [masked[int(offs[i]):int(offs[i + 1])] for i in range(len(haystacks))]
        return [r.decode("utf-8") for r in res] if self._charwise else res

    def value_doc_counts_batch(self, haystacks, mode=None):
        """Haystacks containing each value: ``np.uint64[max value + 1]`` (for ``new`` automata: per pattern);
        ``mode=None`` as in ``count_batch``."""
        blob, offs = _pack(list(haystacks), self._charwise)
        return self.doc_counts_host(self._default_mode(mode), blob, offs, key="value")

    def value_counts_batch(self, haystacks, mode=None):
        """Occurrences per value over all haystacks: ``np.uint64[max value + 1]`` (for ``new`` automata: per pattern);
        ``mode=None`` as in ``count_batch``."""
        blob, offs = _pack(list(haystacks), self._charwise)
        return self.pattern_counts_host(self._default_mode(mode), blob, offs, key="value")

    def _default_mode(self, mode):
        if mode is not None:
            return mode
        return FIND_OVERLAPPING if self.match_kind() == MatchKind.Standard else LEFTMOST_FIND

    def count_batch(self, haystacks, mode=None):
        """Matches per haystack (np.uint64[n]); ``mode=None``: find_overlapping for Standard automata,
        leftmost_find for leftmost ones."""
        blob, offs = _pack(list(haystacks), self._charwise)
        return self.count_batch_host(self._default_mode(mode), blob, offs)[0]

    def first_match_batch(self, haystacks):
        """``[Match | None]``: what ``find_iter(h).next()`` (Standard) or ``leftmost_find_iter(h).next()`` gives."""
        blob, offs = _pack(list(haystacks), self._charwise)
        first, found = self.first_batch_host(self._default_mode(None), blob, offs)
        return [Match(m["start"], m["end"], m["value"]) if f else None for m, f in zip(first, found)]

    def is_match_batch(self, haystacks):
        """np.bool_[n]: does haystack i contain any pattern (the empty pattern included)."""
        blob, offs = _pack(list(haystacks), self._charwise)
        return self.first_batch_host(self._default_mode(None), blob, offs)[1]

    def is_match(self, haystack):
        return bool(self.is_match_batch([haystack])[0])

    def job(self, device=None):
        """An asynchronous scan with its own workspace (dach_job_*): ``scan`` and ``place`` only enqueue work,
        ``wait`` blocks.  Several jobs of one automaton overlap across streams and host threads."""
        return Job(self, device)

    def _batch(self, mode, haystacks):
        blob, offs = _pack(list(haystacks), self._charwise)
        return self.scan_batch_host(mode, blob, offs)

    def find_batch(self, haystacks):
        return self._batch(FIND, haystacks)

    def find_overlapping_batch(self, haystacks):
        return self._batch(FIND_OVERLAPPING, haystacks)

    def find_overlapping_no_suffix_batch(self, haystacks):
        return self._batch(FIND_OVERLAPPING_NO_SUFFIX, haystacks)

    def leftmost_find_batch(self, haystacks):
        return self._batch(LEFTMOST_FIND, haystacks)

    # -- the crate's iterator surface ---------------------------------------------------------------
    def _iter(self, mode, haystack):
        self._assert_mode(mode)  # the crate asserts when the iterator is created
        r = self._batch(mode, [haystack])
        m = r.matches
        return iter([Match(a, b, c) for a, b, c in zip(m["start"], m["end"], m["value"])])

    def find_iter(self, haystack):
        return self._iter(FIND, haystack)

    def find_overlapping_iter(self, haystack):
        return self._iter(FIND_OVERLAPPING, haystack)

    def find_overlapping_no_suffix_iter(self, haystack):
        return self._iter(FIND_OVERLAPPING_NO_SUFFIX, haystack)

    def leftmost_find_iter(self, haystack):
        return self._iter(LEFTMOST_FIND, haystack)


class Job:
    """dach_job: one in-flight scan of device-resident buffers (include/daachorse_b200.h, "asynchronous scans").
    ``scan`` and ``place`` only enqueue work and keep the tensors they are given alive in stream order; inputs written
    on another stream than the one they are enqueued on must be ordered by the caller first."""

    def __init__(self, pma, device=None):
        import torch

        self._pma = pma
        self._dev = torch.cuda.current_device() if device is None else int(device)
        self._h = C.c_void_p()
        _check(_lib.load().dach_job_create(pma.device_handle(self._dev), C.byref(self._h)))
        self._keep = None

    def __del__(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            _lib.load().dach_job_free(self._h)
            self._h = C.c_void_p()

    @staticmethod
    def _stream(stream, device):
        import torch

        if stream is None:
            return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        return C.c_void_p(stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream))

    def scan(self, mode, text, offs, cap_matches, stream=None):
        """Enqueue the scan of ``text`` (uint8 CUDA tensor) / ``offs`` (int64, n+1) on ``stream`` (None, a torch
        stream or a raw handle).  The next ``scan`` may be enqueued before ``wait``, and the caller may drop its
        references at once: both tensors are recorded on ``stream`` (``record_stream``), so the caching allocator
        hands their memory out again only after the scan has read it.  Unlike the ``*_device`` forms this does not
        wait for the current stream: as with torch's own streams, inputs written on another stream are the caller's to
        order (``stream.wait_stream(...)``)."""
        self._pma._assert_mode(mode)
        _check_device_batch(text, offs, self._dev)
        ts = _torch_stream(stream, text.device)
        text.record_stream(ts)
        offs.record_stream(ts)
        self._keep = (text, offs)  # the kernels read them after this call returns
        _check(_lib.load().dach_job_scan(self._h, mode, C.c_void_p(text.data_ptr()), C.c_void_p(offs.data_ptr()),
                                         offs.numel() - 1, text.numel(), int(cap_matches), C.c_void_p(ts.cuda_stream)))

    def place(self, out, out_offs, base=None, stream=None):
        """Enqueue the gather into ``out`` ((cap, 3) int32) / ``out_offs`` (int64, n+1); ``base``: optional
        1-element int64 CUDA tensor, index of the first match in ``out``.  ``out``, ``out_offs`` and ``base`` are
        recorded on ``stream`` as ``scan`` records its inputs; ``base``, too, is the caller's to order if it was
        written on another stream."""
        _check_device_batch(self._keep[0], self._keep[1], out.device.index, out, out_offs)
        if base is not None and (not base.is_cuda or base.dtype not in (torch_int64(),) or base.numel() < 1):
            raise DaachorseError(_lib.INVALID_ARGUMENT, "base must be a 1-element int64 CUDA tensor")
        ts = _torch_stream(stream, out.device)
        for t in (out, out_offs, base):
            if t is not None:
                t.record_stream(ts)
        self._out = (out, out_offs, base)
        _check(_lib.load().dach_job_place(self._h, C.c_void_p(out.data_ptr()), out.shape[0], C.c_void_p(out_offs.data_ptr()),
                                          C.c_void_p(base.data_ptr()) if base is not None else None,
                                          C.c_void_p(ts.cuda_stream)))

    # -- reductions: count_batch_device ... mask_batch_device on the job ---------------------------------------------
    # Each enqueues on ``stream`` and returns the output tensors at once; they hold the results once ``wait`` returns or
    # on ``stream`` after the call.  Inputs and outputs are recorded on ``stream`` as ``scan`` records its inputs, and
    # inputs written on another stream are the caller's to order.  Outputs the wrapper creates are allocated on
    # ``stream``, so the histogram's zeros come before the scan with no wait between streams.
    def _enqueue(self, fn, head, text, offs, tail, ts, tensors):
        """dach_job_<fn>(job, *head, text, offs, n, text_bytes, *tail, stream) after recording ``tensors`` on ``ts``."""
        for t in (text, offs) + tensors:
            t.record_stream(ts)
        _check(getattr(_lib.load(), "dach_job_" + fn)(self._h, *head, C.c_void_p(text.data_ptr()), C.c_void_p(offs.data_ptr()),
                                                      offs.numel() - 1, text.numel(), *tail, C.c_void_p(ts.cuda_stream)))

    def count(self, mode, text, offs, out=None, stream=None):
        """``count_batch_device`` on the job: the int64 counts (``out``: optional preallocated one); ``wait`` returns
        their sum."""
        import torch

        self._pma._assert_mode(mode)
        _check_device_batch(text, offs, self._dev, counts=out)
        ts = _torch_stream(stream, text.device)
        if out is None:
            with torch.cuda.stream(ts):
                out = torch.empty(offs.numel() - 1, dtype=torch.int64, device=text.device)
        self._enqueue("count", (mode,), text, offs, (C.c_void_p(out.data_ptr()),), ts, (out,))
        return out

    def first(self, mode, text, offs, out=None, found=None, stream=None):
        """``first_batch_device`` on the job: ``(first, found)``; ``wait`` returns the number of haystacks with a match."""
        import torch

        self._pma._assert_mode(mode)
        _check_device_batch(text, offs, self._dev, first=out, found=found)
        ts = _torch_stream(stream, text.device)
        n = offs.numel() - 1
        with torch.cuda.stream(ts):
            if out is None:
                out = torch.empty((n, 3), dtype=torch.int32, device=text.device)
            if found is None:
                found = torch.empty(n, dtype=torch.bool, device=text.device)
        self._enqueue("first", (mode,), text, offs, (C.c_void_p(out.data_ptr()), C.c_void_p(found.data_ptr())), ts, (out, found))
        return out, found

    def pattern_counts(self, mode, text, offs, key="value", out=None, stream=None):
        """``pattern_counts_device`` on the job: the int64 histogram, added into ``out`` if given (zeros otherwise).
        Jobs may add into one histogram at the same time; ``wait`` returns the number of matches this call added."""
        import torch

        self._pma._assert_mode(mode)
        need = self._pma._hist_len(key)
        _check_device_batch(text, offs, self._dev, hist=out, hist_len=need)
        ts = _torch_stream(stream, text.device)
        if out is None:
            with torch.cuda.stream(ts):
                out = torch.zeros(need, dtype=torch.int64, device=text.device)
        self._enqueue("hist", (mode, HIST_KEYS[key]), text, offs, (C.c_void_p(out.data_ptr()), out.numel()), ts, (out,))
        return out

    def mask(self, mode, text, offs, fill=ord("*"), out=None, stream=None):
        """``mask_batch_device`` on the job: a uint8 tensor of ``text``'s size (``out``: optional preallocated one, which
        must not overlap ``text``); ``wait`` returns 0."""
        import torch

        fill = self._pma._fill_byte(fill)
        self._pma._assert_mode(mode)
        _check_device_batch(text, offs, self._dev, masked=out)
        ts = _torch_stream(stream, text.device)
        if out is None:
            with torch.cuda.stream(ts):
                out = torch.empty(text.numel(), dtype=torch.uint8, device=text.device)
        self._enqueue("mask", (mode,), text, offs, (fill, C.c_void_p(out.data_ptr())), ts, (out,))
        return out

    def wait(self):
        """Block until the job's last operation is done.  Returns the number of matches after ``place`` (raises on
        overflow), the total of the synchronous twin after a reduction (counts' sum, haystacks with a match, matches
        added into the histogram; 0 for ``mask``); bad offsets raise INVALID_ARGUMENT and leave the outputs as they were."""
        need = C.c_uint64()
        _check(_lib.load().dach_job_wait(self._h, C.byref(need)))
        return int(need.value)

    def scan_kernel_ms(self):
        return _lib.load().dach_job_scan_kernel_ms(self._h)

    def push_ms(self):
        return _lib.load().dach_job_push_ms(self._h)

    def times(self):
        """ms since the automaton's first job scan on this device: (scan start, scan end, push start, push end)."""
        buf = (C.c_double * 4)()
        _check(_lib.load().dach_job_times(self._h, C.byref(buf)))
        return tuple(float(x) for x in buf)


def torch_int64():
    import torch

    return torch.int64


def _check_device_batch(text, offs, dev_index, out=None, out_offs=None, state=None, pos=None, counts=None, first=None,
                        found=None, hist=None, hist_len=0, masked=None):
    """Raw pointers cross the C ABI: a wrong dtype, stride or device would be silent garbage or a device fault."""
    import torch

    def bad(msg):
        raise DaachorseError(_lib.INVALID_ARGUMENT, msg)

    n = offs.numel() - 1
    if n < 0:
        bad("offs must hold n + 1 entries")
    for name, t, dtypes in (("text", text, (torch.uint8,)), ("offs", offs, (torch.int64, torch.uint64)),
                            ("out", out, (torch.int32, torch.uint32)), ("out_offs", out_offs, (torch.int64, torch.uint64)),
                            ("state", state, (torch.int32, torch.uint32)), ("pos", pos, (torch.int32, torch.uint32)),
                            ("counts", counts, (torch.int64, torch.uint64)), ("first", first, (torch.int32, torch.uint32)),
                            ("found", found, (torch.bool, torch.uint8)), ("hist", hist, (torch.int64,)),
                            ("masked", masked, (torch.uint8,))):
        if t is None:
            continue
        if not t.is_cuda or t.device.index != dev_index:
            bad("%s must be a CUDA tensor on cuda:%d" % (name, dev_index))
        if t.dtype not in dtypes:
            bad("%s has dtype %s, expected one of %s" % (name, t.dtype, dtypes))
        if not t.is_contiguous():
            bad("%s must be contiguous" % name)
    if out is not None and (out.dim() != 2 or out.shape[1] != 3):
        bad("out must have shape (capacity, 3)")
    if out_offs is not None and out_offs.numel() < n + 1:
        bad("out_offs must hold n + 1 entries")
    for name, t in (("state", state), ("pos", pos), ("counts", counts), ("found", found)):
        if t is not None and t.numel() != n:
            bad("%s must hold n entries" % name)
    if first is not None and (first.dim() != 2 or first.shape[0] != n or first.shape[1] != 3):
        bad("first must have shape (n, 3)")
    if hist is not None and (hist.dim() != 1 or hist.numel() < hist_len):
        bad("hist must be 1-d with at least %d entries" % hist_len)
    if masked is not None:
        if masked.numel() < text.numel():
            bad("the masked output must hold at least text.numel() bytes")
        a, b = text.data_ptr(), masked.data_ptr()
        if text.numel() and a < b + text.numel() and b < a + text.numel():
            bad("the masked output must not overlap text (masking in place is not supported)")


def _current_device():
    try:
        import torch

        if torch.cuda.is_available():
            return torch.cuda.current_device()
    except Exception:
        pass
    return 0


class DoubleArrayAhoCorasick(_Automaton):
    """Byte-wise double-array Aho-Corasick automaton (src/bytewise.rs:54-68)."""
    _charwise = False


class CharwiseDoubleArrayAhoCorasick(_Automaton):
    """Char-wise double-array Aho-Corasick automaton (src/charwise.rs:59-65)."""
    _charwise = True


class _Builder:
    _cls = None

    def __init__(self):
        self._kind = MatchKind.Standard
        self._nfb = 16  # src/bytewise/builder.rs:61

    @classmethod
    def new(cls):
        return cls()

    def match_kind(self, kind):
        self._kind = MatchKind(kind)
        return self

    def num_free_blocks(self, n):
        assert n >= 1  # src/bytewise/builder.rs:113
        self._nfb = int(n)
        return self

    def build(self, patterns):
        return self._cls._build(patterns, None, self._kind, self._nfb)

    def build_with_values(self, patvals):
        patvals = list(patvals)
        return self._cls._build([p for p, _ in patvals], [v for _, v in patvals], self._kind, self._nfb)


class DoubleArrayAhoCorasickBuilder(_Builder):
    """src/bytewise/builder.rs:21-244"""
    _cls = DoubleArrayAhoCorasick


class CharwiseDoubleArrayAhoCorasickBuilder(_Builder):
    """src/charwise/builder.rs"""
    _cls = CharwiseDoubleArrayAhoCorasick
