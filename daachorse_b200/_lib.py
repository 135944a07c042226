"""ctypes loader of libdaachorse_b200.so (the C ABI declared in include/daachorse_b200.h).

The library is built in-tree by ``__graft_entry__.build()`` / ``make -C daachorse_b200/csrc``.
There is no fallback: if the shared object is missing the import fails loudly.
"""
import ctypes as C
import os

_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DACH_LIB") or os.path.join(_DIR, "libdaachorse_b200.so")  # DACH_LIB: experiment builds

(OK, INVALID_ARGUMENT, AUTOMATON_SCALE, INVALID_CONVERSION, INVALID_AUTOMATON, MATCH_KIND_MISMATCH,
 OUTPUT_OVERFLOW, CUDA_ERROR) = range(8)

# every symbol include/daachorse_b200.h declares (tests check the .so exports all of them)
SYMBOLS = [
    "dach_bytewise_build", "dach_charwise_build", "dach_pma_deserialize", "dach_pma_serialized_bytes",
    "dach_pma_serialize", "dach_pma_match_kind", "dach_pma_num_states", "dach_pma_heap_bytes",
    "dach_pma_num_elements", "dach_pma_is_charwise", "dach_pma_max_pattern_len", "dach_pma_num_outputs",
    "dach_pma_outputs", "dach_pma_free",
    "dach_dev_upload", "dach_dev_free", "dach_dev_image_bytes", "dach_dev_scan_batch", "dach_dev_scan_stream",
    "dach_dev_count_stream", "dach_dev_first_stream", "dach_dev_hist_stream", "dach_scan_batch_host", "dach_dev_count_batch", "dach_count_batch_host", "dach_dev_first_batch", "dach_first_batch_host",
    "dach_dev_hist_batch", "dach_hist_batch_host", "dach_dev_df_batch", "dach_df_batch_host", "dach_dev_last_df_windows",
    "dach_dev_mask_batch", "dach_mask_batch_host", "dach_dev_kernel_launches", "dach_dev_last_scan_kernel_ms",
    "dach_dev_last_total_ms", "dach_dev_last_h2d_bytes", "dach_dev_last_d2h_bytes",
    "dach_dev_set_option", "dach_last_error", "dach_abi_version",
    "dach_job_create", "dach_job_free", "dach_job_scan", "dach_job_place", "dach_job_count", "dach_job_first",
    "dach_job_hist", "dach_job_mask", "dach_job_wait", "dach_job_scan_kernel_ms", "dach_job_push_ms", "dach_job_times",
    "dach_group_create", "dach_group_export", "dach_group_connect", "dach_group_place", "dach_group_finish",
    "dach_group_result", "dach_group_free",
]
GROUP_HANDLE_BYTES = 256

_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "daachorse_b200: %s is missing -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C daachorse_b200/csrc`; there is no CPU fallback." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    pp = C.POINTER(vp)
    L.dach_abi_version.restype = C.c_int
    L.dach_last_error.restype = C.c_char_p
    for f in (L.dach_bytewise_build, L.dach_charwise_build):
        f.argtypes = [vp, vp, vp, C.c_uint32, C.c_uint8, C.c_uint32, pp]
        f.restype = C.c_int
    L.dach_pma_deserialize.argtypes = [vp, C.c_size_t, C.c_int, pp, C.POINTER(C.c_size_t)]
    L.dach_pma_deserialize.restype = C.c_int
    L.dach_pma_serialized_bytes.argtypes = [vp]
    L.dach_pma_serialized_bytes.restype = C.c_size_t
    L.dach_pma_serialize.argtypes = [vp, vp, C.c_size_t, C.POINTER(C.c_size_t)]
    L.dach_pma_serialize.restype = C.c_int
    for name, rt in (("dach_pma_match_kind", C.c_uint8), ("dach_pma_num_states", C.c_uint32),
                     ("dach_pma_heap_bytes", C.c_size_t), ("dach_pma_num_elements", C.c_size_t),
                     ("dach_pma_is_charwise", C.c_int), ("dach_pma_max_pattern_len", C.c_uint32),
                     ("dach_pma_num_outputs", C.c_uint32)):
        getattr(L, name).argtypes = [vp]
        getattr(L, name).restype = rt
    L.dach_pma_outputs.argtypes = [vp, vp, vp, vp, C.c_uint32]
    L.dach_pma_outputs.restype = C.c_int
    L.dach_pma_free.argtypes = [vp]
    L.dach_pma_free.restype = None
    L.dach_dev_upload.argtypes = [vp, C.c_int, pp]
    L.dach_dev_upload.restype = C.c_int
    L.dach_dev_free.argtypes = [vp]
    L.dach_dev_free.restype = None
    L.dach_dev_image_bytes.argtypes = [vp]
    L.dach_dev_image_bytes.restype = C.c_size_t
    L.dach_dev_scan_batch.argtypes = [vp, C.c_int, vp, vp, C.c_uint64, C.c_uint64, vp, C.c_uint64, vp,
                                      C.POINTER(C.c_uint64), vp]
    L.dach_dev_scan_batch.restype = C.c_int
    L.dach_dev_scan_stream.argtypes = [vp, C.c_int, vp, vp, C.c_uint64, C.c_uint64, vp, vp, vp, C.c_uint64, vp,
                                       C.POINTER(C.c_uint64), vp]
    L.dach_dev_scan_stream.restype = C.c_int
    L.dach_dev_count_stream.argtypes = [vp, C.c_int, vp, vp, C.c_uint64, C.c_uint64, vp, vp, C.POINTER(C.c_uint64), vp]
    L.dach_dev_first_stream.argtypes = [vp, C.c_int, vp, vp, C.c_uint64, C.c_uint64, vp, vp, vp, vp, C.POINTER(C.c_uint64), vp]
    L.dach_dev_hist_stream.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_uint64, C.c_uint64, vp, vp, C.c_uint64,
                                       C.POINTER(C.c_uint64), vp]
    for name in ("dach_dev_count_stream", "dach_dev_first_stream", "dach_dev_hist_stream"):
        getattr(L, name).restype = C.c_int
    L.dach_scan_batch_host.argtypes = [vp, C.c_int, vp, vp, C.c_uint64, vp, C.c_uint64, vp,
                                       C.POINTER(C.c_uint64)]
    L.dach_scan_batch_host.restype = C.c_int
    L.dach_dev_count_batch.argtypes = [vp, C.c_int, vp, vp, C.c_uint64, C.c_uint64, vp, C.POINTER(C.c_uint64), vp]
    L.dach_count_batch_host.argtypes = [vp, C.c_int, vp, vp, C.c_uint64, vp, C.POINTER(C.c_uint64)]
    L.dach_dev_first_batch.argtypes = [vp, C.c_int, vp, vp, C.c_uint64, C.c_uint64, vp, vp, C.POINTER(C.c_uint64), vp]
    L.dach_first_batch_host.argtypes = [vp, C.c_int, vp, vp, C.c_uint64, vp, vp, C.POINTER(C.c_uint64)]
    L.dach_dev_hist_batch.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_uint64, C.c_uint64, vp, C.c_uint64, C.POINTER(C.c_uint64), vp]
    L.dach_hist_batch_host.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_uint64, vp, C.c_uint64, C.POINTER(C.c_uint64)]
    L.dach_dev_df_batch.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_uint64, C.c_uint64, vp, C.c_uint64, C.POINTER(C.c_uint64), vp]
    L.dach_df_batch_host.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_uint64, vp, C.c_uint64, C.POINTER(C.c_uint64)]
    L.dach_dev_last_df_windows.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.dach_dev_mask_batch.argtypes = [vp, C.c_int, vp, vp, C.c_uint64, C.c_uint64, C.c_uint8, vp, vp]
    L.dach_mask_batch_host.argtypes = [vp, C.c_int, vp, vp, C.c_uint64, C.c_uint8, vp]
    for name in ("dach_dev_count_batch", "dach_count_batch_host", "dach_dev_first_batch", "dach_first_batch_host",
                 "dach_dev_hist_batch", "dach_hist_batch_host", "dach_dev_df_batch", "dach_df_batch_host", "dach_dev_last_df_windows",
                 "dach_dev_mask_batch", "dach_mask_batch_host"):
        getattr(L, name).restype = C.c_int
    L.dach_dev_kernel_launches.argtypes = [vp]
    L.dach_dev_kernel_launches.restype = C.c_uint64
    for name in ("dach_dev_last_scan_kernel_ms", "dach_dev_last_total_ms"):
        getattr(L, name).argtypes = [vp]
        getattr(L, name).restype = C.c_double
    for name in ("dach_dev_last_h2d_bytes", "dach_dev_last_d2h_bytes"):
        getattr(L, name).argtypes = [vp]
        getattr(L, name).restype = C.c_uint64
    L.dach_dev_set_option.argtypes = [vp, C.c_char_p, C.c_int64]
    L.dach_dev_set_option.restype = C.c_int
    u64 = C.c_uint64
    L.dach_job_create.argtypes = [vp, pp]
    L.dach_job_free.argtypes = [vp]
    L.dach_job_free.restype = None
    L.dach_job_scan.argtypes = [vp, C.c_int, vp, vp, u64, u64, u64, vp]
    L.dach_job_place.argtypes = [vp, vp, u64, vp, vp, vp]
    L.dach_job_count.argtypes = [vp, C.c_int, vp, vp, u64, u64, vp, vp]
    L.dach_job_first.argtypes = [vp, C.c_int, vp, vp, u64, u64, vp, vp, vp]
    L.dach_job_hist.argtypes = [vp, C.c_int, C.c_int, vp, vp, u64, u64, vp, u64, vp]
    L.dach_job_mask.argtypes = [vp, C.c_int, vp, vp, u64, u64, C.c_uint8, vp, vp]
    L.dach_job_wait.argtypes = [vp, C.POINTER(u64)]
    L.dach_job_scan_kernel_ms.argtypes = [vp]
    L.dach_job_scan_kernel_ms.restype = C.c_double
    L.dach_job_push_ms.argtypes = [vp]
    L.dach_job_push_ms.restype = C.c_double
    L.dach_job_times.argtypes = [vp, C.POINTER(C.c_double * 4)]
    L.dach_job_times.restype = C.c_int
    L.dach_group_create.argtypes = [C.c_int, C.c_int, C.c_int, u64, u64, pp]
    L.dach_group_export.argtypes = [vp, vp]
    L.dach_group_connect.argtypes = [vp, vp]
    L.dach_group_place.argtypes = [vp, vp, u64, C.c_int, vp]
    L.dach_group_finish.argtypes = [vp, C.POINTER(u64), vp]
    L.dach_group_result.argtypes = [vp, pp, pp]
    L.dach_group_free.argtypes = [vp]
    L.dach_group_free.restype = None
    for name in ("dach_job_create", "dach_job_scan", "dach_job_place", "dach_job_count", "dach_job_first", "dach_job_hist",
                 "dach_job_mask", "dach_job_wait", "dach_group_create", "dach_group_export",
                 "dach_group_connect", "dach_group_place", "dach_group_finish", "dach_group_result"):
        getattr(L, name).restype = C.c_int
    if L.dach_abi_version() != 2:
        raise ImportError("daachorse_b200: ABI version mismatch")
    _lib = L
    return L


def last_error():
    return load().dach_last_error().decode("utf-8", "replace")
