"""ctypes binding of libfxg.so -- the C-ABI declared in include/fxg.h.

This is the only place the package touches native code.  There is no CPU fallback: if the
library is missing or no CUDA device is usable, the compute entry points raise.
"""
import ctypes as C
import os
import re

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("FXG_LIB_PATH") or os.path.join(_HERE, "libfxg.so")     # override: A/B builds only
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "fxg.h")

FASTA_ROW = np.dtype([("boff", "<i8"), ("blen", "<i8"), ("slen", "<i8"), ("llen", "<i8"),
                      ("dlen", "<i4"), ("nlen", "<i4"), ("elen", "u1"), ("norm", "u1"),
                      ("pad", "u1", (6,))])
FASTQ_ROW = np.dtype([("soff", "<i8"), ("qoff", "<i8"), ("rlen", "<i8"),
                      ("dlen", "<i4"), ("nlen", "<i4")])

FXG_OK, FXG_ENODEV, FXG_ECUDA, FXG_EINVAL, FXG_ENOMEM, FXG_ECAP, FXG_EIO, FXG_EFORMAT = 0, -1, -2, -3, -4, -5, -6, -7
SCAN_FULL_NAME = 1
X_UPPER, X_REVERSE, X_COMPLEMENT, X_RAW, X_WHOLE = 1, 2, 4, 8, 16


class ScanStats(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("n_lines", C.c_int64), ("total_len", C.c_int64),
                ("end_position", C.c_int64), ("lead_lines", C.c_int64), ("lead_bytes", C.c_int64),
                ("lead_llen", C.c_int64), ("reserved", C.c_int64)]


class ShardInfo(C.Structure):
    """fxg_shard_info: what one shard tells the others (the struct of the one small all-gather)"""
    _fields_ = [("n_rows", C.c_int64), ("n_lines", C.c_int64), ("bytes", C.c_int64), ("base_offset", C.c_int64),
                ("end_position", C.c_int64), ("edge_n", C.c_int64), ("edge_off", C.c_int64 * 3),
                ("edge_len", C.c_int64 * 3), ("reserved", C.c_int64 * 4)]


SHARD_INFO = np.dtype([("n_rows", "<i8"), ("n_lines", "<i8"), ("bytes", "<i8"), ("base_offset", "<i8"),
                       ("end_position", "<i8"), ("edge_n", "<i8"), ("edge_off", "<i8", (3,)), ("edge_len", "<i8", (3,)),
                       ("reserved", "<i8", (4,))])
COMM_ID_BYTES = 128


class GzIndex(C.Structure):
    _fields_ = [("compressed_size", C.c_int64), ("uncompressed_size", C.c_int64), ("spacing", C.c_uint32),
                ("window_size", C.c_uint32), ("npoints", C.c_int64), ("cmp_offset", C.c_void_p),
                ("uncmp_offset", C.c_void_p), ("bits", C.c_void_p), ("has_data", C.c_void_p), ("windows", C.c_void_p)]


class FastqMeta(C.Structure):
    _fields_ = [(k, C.c_int64) for k in ("a", "c", "g", "t", "n", "maxlen", "minlen", "minqs", "maxqs", "phred")]


COMP_ROW = np.dtype([("seqid", "<i8"), ("abc", "<i8"), ("num", "<i8")])
SEARCH_HIT = np.dtype([("query", "<i8"), ("start", "<i8"), ("minus", "<i4"), ("mismatches", "<i4")])   # fxg_search_hit

SEARCH_PIECE, SEARCH_MAX_PATTERN = 4096, 1024                     # FXG_SEARCH_PIECE, FXG_SEARCH_MAX_PATTERN
SEARCH_PLUS, SEARCH_MINUS = 1, 2
SEARCH_ALL, SEARCH_FIRST = 0, 1


class FxgError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libfxg error %d: %s" % (code, msg))
        self.code = code


class NoDeviceError(FxgError):
    pass


vp, i64, i32, u64 = C.c_void_p, C.c_int64, C.c_int, C.c_uint64
P = C.POINTER

# name -> (restype, argtypes); every symbol declared in include/fxg.h
SIGNATURES = {
    "fxg_abi_version": (i32, []),
    "fxg_last_error": (C.c_char_p, []),
    "fxg_device_count": (i32, []),
    "fxg_ctx_create": (i32, [i32, P(vp)]),
    "fxg_ctx_destroy": (None, [vp]),
    "fxg_ctx_set_stream": (i32, [vp, vp]),
    "fxg_ctx_sync": (i32, [vp]),
    "fxg_ctx_sm_count": (i32, [vp]),
    "fxg_profile_enable": (i32, [vp, i32]),
    "fxg_profile_last_ms": (i32, [vp, i32, P(C.c_float)]),
    "fxg_ctx_launch_count": (i64, [vp]),
    "fxg_host_alloc": (i32, [i64, P(vp)]),
    "fxg_host_free": (None, [vp]),
    "fxg_file_alloc": (i32, [vp, i64, P(vp)]),
    "fxg_file_upload": (i32, [vp, vp, i64, vp, i64]),
    "fxg_file_from_host": (i32, [vp, vp, i64, P(vp)]),
    "fxg_file_from_path": (i32, [vp, C.c_char_p, P(vp)]),
    "fxg_file_wrap": (i32, [vp, vp, i64, i64, P(vp)]),
    "fxg_file_download": (i32, [vp, vp, i64, vp, i64]),
    "fxg_file_devptr": (vp, [vp]),
    "fxg_file_size": (i64, [vp]),
    "fxg_file_free": (None, [vp]),
    "fxg_pool_trim": (None, []),
    "fxg_fasta_scan": (i32, [vp, vp, i64, i32, P(vp), P(ScanStats)]),
    "fxg_fastq_scan": (i32, [vp, vp, i64, P(vp), P(ScanStats)]),
    "fxg_scan_begin": (i32, [vp, vp, i32, i64, i32, vp]),
    "fxg_shard_exchange": (i32, [vp, vp, vp, vp, i64]),
    "fxg_scan_finish": (i32, [vp, vp, i32, i32, P(vp), P(ScanStats), vp]),
    "fxg_scan_sharded": (i32, [vp, vp, vp, i32, i64, i32, P(vp), P(ScanStats), vp]),
    "fxg_comm_unique_id": (i32, [vp]),
    "fxg_comm_create": (i32, [vp, vp, i32, i32, P(vp)]),
    "fxg_comm_nranks": (i32, [vp]),
    "fxg_comm_rank": (i32, [vp]),
    "fxg_comm_uses_p2p": (i32, [vp]),
    "fxg_comm_check": (i32, [vp]),
    "fxg_comm_destroy": (None, [vp]),
    "fxg_split_point_dev": (i32, [vp, vp, i64, i32, P(i64)]),
    "fxg_split_point_path": (i32, [C.c_char_p, i64, i32, P(i64), P(i64)]),
    "fxg_file_from_path_range": (i32, [vp, C.c_char_p, i64, i64, P(vp)]),
    "fxg_file_slice": (i32, [vp, vp, i64, i64, P(vp)]),
    "fxg_rows_download": (i32, [vp, vp, i64, i32, vp]),
    "fxg_rows_upload": (i32, [vp, vp, i64, i32, P(vp)]),
    "fxg_dev_free": (None, [vp]),
    "fxg_fasta_build_index_host": (i32, [vp, vp, i64, i32, vp, i64, P(ScanStats)]),
    "fxg_fastq_build_index_host": (i32, [vp, vp, i64, vp, i64, P(ScanStats)]),
    "fxg_extract_plan_dev": (i32, [vp, vp, vp, i64, vp, P(i64)]),
    "fxg_extract_dev": (i32, [vp, vp, vp, i64, vp, vp, vp, vp, i64, vp, vp, vp]),
    "fxg_extract_host": (i32, [vp, vp, vp, i64, vp, vp, vp, vp, i64, vp, vp, i64, vp]),
    "fxg_extract_one_host": (i32, [vp, vp, vp, i64, i64, i64, i64, i32, vp, i64]),
    "fxg_composition_host": (i32, [vp, vp, vp, i64, vp, vp, vp, vp, i64, vp]),
    "fxg_search_host": (i32, [vp, vp, vp, i64, vp, vp, vp, i32, i64, vp, i32, i32, i32, P(vp), P(i64)]),
    "fxg_search_reads_host": (i32, [vp, vp, vp, i64, vp, i32, i32, P(vp), P(i64)]),
    "fxg_search_approx_host": (i32, [vp, vp, vp, i64, vp, vp, vp, i32, i64, vp, i32, i32, i32, P(vp), P(i64)]),
    "fxg_search_reads_approx_host": (i32, [vp, vp, vp, i64, vp, i32, i32, i32, P(vp), P(i64)]),
    "fxg_reads_dev": (i32, [vp, vp, vp, i64, vp, i64, i32, vp, vp, vp, i64, P(i64)]),
    "fxg_reads_host": (i32, [vp, vp, vp, i64, vp, i64, i32, vp, vp, vp, i64]),
    "fxg_read_one_host": (i32, [vp, vp, vp, i64, i64, i32, i32, i64, vp, i64]),
    "fxg_bgzf_members_host": (i32, [vp, i64, vp, vp, i64, P(i64), P(i64)]),
    "fxg_inflate_members_dev": (i32, [vp, vp, vp, vp, i64, vp, i64, vp]),
    "fxg_file_from_bgzf_host": (i32, [vp, vp, i64, P(vp), P(i64)]),
    "fxg_fxi_write_fasta": (i32, [C.c_char_p, vp, i64, vp, vp, i64, vp, vp, i64]),
    "fxg_fxi_write_fastq": (i32, [C.c_char_p, vp, i64, vp, vp, i64, i64, vp, vp]),
    "fxg_gzip_inflate_host": (i32, [vp, i64, C.c_uint32, P(vp)]),
    "fxg_gzip_data": (vp, [vp, P(i64)]),
    "fxg_gzip_index": (i32, [vp, P(GzIndex)]),
    "fxg_gzip_free": (None, [vp]),
    "fxg_file_from_gzip_points_host": (i32, [vp, vp, i64, P(GzIndex), P(vp)]),
    "fxg_fasta_composition": (i32, [vp, vp, vp, i64, i64, P(vp), P(i64), vp]),
    "fxg_fastq_stats": (i32, [vp, vp, vp, i64, i64, i32, P(FastqMeta)]),
    "fxg_free_host": (None, [vp]),
    "fxg_nametab_build": (i32, [vp, vp, i64, P(vp)]),
    "fxg_nametab_find": (i64, [vp, C.c_char_p, i64]),
    "fxg_nametab_lookup": (i32, [vp, vp, vp, i64, vp]),
    "fxg_nametab_free": (None, [vp]),
    "fxg_bgzf_compress_host": (i32, [vp, i64, i32, P(vp), P(i64)]),
    "fxg_synth_fasta_dev": (i32, [vp, u64, vp, vp, i64, i64, i32, vp]),
    "fxg_synth_fastq_dev": (i32, [vp, u64, i64, i64, i32, vp, vp]),
}

_lib = None


def declared_symbols():
    """Function names declared in include/fxg.h (parsed, so the header stays the source of truth)."""
    with open(HEADER_PATH) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return sorted(set(re.findall(r"\b(fxg_[a-z0-9_]+)\s*\(", text)))


def lib():
    """Load libfxg.so; raise loudly if the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FxgError(FXG_ENODEV, "libfxg.so not built (run pyfastx_b200/csrc/build.sh or "
                                       "__graft_entry__.build()); there is no CPU fallback")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc):
    if rc != FXG_OK:
        msg = lib().fxg_last_error().decode("utf-8", "replace")
        raise (NoDeviceError if rc == FXG_ENODEV else FxgError)(rc, msg)
    return rc


def ptr(a):
    """device/host pointer of a numpy array, a torch tensor, an int or None"""
    if a is None:
        return None
    if isinstance(a, int):
        return a
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    raise TypeError("cannot take a pointer of %r" % type(a))
