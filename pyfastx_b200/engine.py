"""numpy-facing wrapper over the C-ABI (one Engine per process and GPU).

Everything here runs on the GPU through libfxg.so; nothing falls back to the CPU.
"""
import ctypes as C
import os
import threading

import numpy as np

from . import _cabi
from ._cabi import FASTA_ROW, FASTQ_ROW, ScanStats, check, lib, ptr

try:
    from . import _fast                     # compiled bridge: per-object getters call the C-ABI without ctypes
except ImportError:                         # pragma: no cover
    _fast = None

_engines = {}
_lock = threading.Lock()


def default_device():
    d = os.environ.get("PYFASTX_B200_DEVICE")
    if d is not None:
        return int(d)
    lr = os.environ.get("LOCAL_RANK")
    return int(lr) if lr is not None else 0


def get_engine(device=None):
    if device is None:
        device = default_device()
    with _lock:
        e = _engines.get(device)
        if e is None:
            e = _engines[device] = Engine(device)
        return e


class DeviceFile:
    """A FASTA/FASTQ byte stream resident in HBM (fxg_file)."""

    def __init__(self, engine, handle):
        self.engine = engine
        self.handle = handle

    @property
    def size(self):
        return lib().fxg_file_size(self.handle)

    @property
    def devptr(self):
        return lib().fxg_file_devptr(self.handle)

    def download(self, offset=0, nbytes=None):
        n = self.size - offset if nbytes is None else nbytes
        out = np.empty(max(n, 0), dtype=np.uint8)
        if n > 0:
            check(lib().fxg_file_download(self.engine.ctx, self.handle, offset, out.ctypes.data, n))
        return out

    def free(self):
        if self.handle:
            lib().fxg_file_free(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class DeviceRows:
    """Index rows resident in HBM (own allocation, independent of the scan scratch)."""

    def __init__(self, engine, devptr, n_rows, dtype):
        self.engine, self.devptr, self.n_rows, self.dtype = engine, devptr, n_rows, dtype

    def free(self):
        if self.devptr:
            lib().fxg_dev_free(self.devptr)
            self.devptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _stats_dict(st):
    return {k: getattr(st, k) for k, _ in ScanStats._fields_ if k != "reserved"}


class Engine:
    def __init__(self, device=0):
        L = lib()
        h = C.c_void_p()
        check(L.fxg_ctx_create(device, C.byref(h)))
        self.ctx = h
        self.device = device
        self.sm_count = L.fxg_ctx_sm_count(h)

    def close(self):
        if getattr(self, "ctx", None):
            lib().fxg_ctx_destroy(self.ctx)
            self.ctx = None

    def set_stream(self, cuda_stream):
        check(lib().fxg_ctx_set_stream(self.ctx, cuda_stream))

    def sync(self):
        check(lib().fxg_ctx_sync(self.ctx))

    # ---- staging --------------------------------------------------------------------------
    def stage_bytes(self, data):
        a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data)
        h = C.c_void_p()
        check(lib().fxg_file_from_host(self.ctx, a.ctypes.data if a.size else None, a.size, C.byref(h)))
        self.sync()
        return DeviceFile(self, h)

    def stage_bgzf(self, data):
        """BGZF bytes (host) -> uncompressed DeviceFile, inflated member-parallel on the GPU (K6).
        Raises FxgError(FXG_EFORMAT) if the stream is plain gzip rather than BGZF."""
        a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data)
        h = C.c_void_p()
        nm = C.c_int64(0)
        check(lib().fxg_file_from_bgzf_host(self.ctx, a.ctypes.data, a.size, C.byref(h), C.byref(nm)))
        f = DeviceFile(self, h)
        f.n_members = nm.value
        return f

    def bgzf_members(self, data):
        """member table of a BGZF byte string (host header walk, no inflation): (cmp_off, ucmp_off), n+1 entries each.
        Raises FxgError(FXG_EFORMAT) for plain gzip."""
        a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data)
        nm, tot = C.c_int64(0), C.c_int64(0)
        check(lib().fxg_bgzf_members_host(a.ctypes.data, a.size, None, None, 0, C.byref(nm), C.byref(tot)))
        co = np.zeros(nm.value + 1, dtype=np.int64)
        uo = np.zeros(nm.value + 1, dtype=np.int64)
        check(lib().fxg_bgzf_members_host(a.ctypes.data, a.size, co.ctypes.data, uo.ctypes.data, nm.value + 1,
                                          C.byref(nm), C.byref(tot)))
        return co, uo

    def gzip_inflate(self, data):
        """generic gzip (one serial deflate stream): ONE zlib pass on the host -> (inflated uint8 view, GzIndex with
        the zran checkpoints, handle).  The handle owns both; keep it until the .fxi is written, then gzip_free."""
        a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data)
        h = C.c_void_p()
        check(lib().fxg_gzip_inflate_host(a.ctypes.data, a.size, 0, C.byref(h)))
        n = C.c_int64(0)
        p = lib().fxg_gzip_data(h, C.byref(n))
        view = np.frombuffer((C.c_uint8 * n.value).from_address(p), dtype=np.uint8) if n.value else np.zeros(0, np.uint8)
        gz = _cabi.GzIndex()
        check(lib().fxg_gzip_index(h, C.byref(gz)))
        return view, gz, h

    def stage_gzip_points(self, data, gz):
        """generic gzip with known checkpoints (fxi.read_gzindex): every checkpoint's segment is inflated by its own GPU
        thread, verified against the gzip trailer (length + CRC-32) -> DeviceFile.  FxgError(FXG_EFORMAT) if the
        checkpoints do not fit the file (then: gzip_inflate)."""
        a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data)
        h = C.c_void_p()
        check(lib().fxg_file_from_gzip_points_host(self.ctx, a.ctypes.data, a.size, C.byref(gz["struct"]), C.byref(h)))
        return DeviceFile(self, h)

    def gzip_free(self, handle):
        lib().fxg_gzip_free(handle)

    def gather_ranges(self, dfile, offsets, lengths):
        """raw byte ranges of the resident file (e.g. record names) -> (packed uint8, offsets[n+1])"""
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        lengths = np.ascontiguousarray(lengths, dtype=np.int64)
        rows = np.zeros(offsets.size, dtype=FASTQ_ROW)
        rows["soff"] = offsets
        rows["qoff"] = offsets
        rows["rlen"] = lengths
        d = self.upload_rows(rows)
        try:
            seq, _, off = self.reads(dfile, d, np.arange(offsets.size, dtype=np.int64), want_qual=False, rlens=lengths)
        finally:
            d.free()
        return seq, off

    def stage_path(self, path):
        h = C.c_void_p()
        check(lib().fxg_file_from_path(self.ctx, os.fsencode(path), C.byref(h)))
        return DeviceFile(self, h)

    def alloc_file(self, nbytes):
        h = C.c_void_p()
        check(lib().fxg_file_alloc(self.ctx, nbytes, C.byref(h)))
        return DeviceFile(self, h)

    def wrap_file(self, devptr, nbytes, capacity):
        h = C.c_void_p()
        check(lib().fxg_file_wrap(self.ctx, devptr, nbytes, capacity, C.byref(h)))
        return DeviceFile(self, h)

    # ---- index scans ------------------------------------------------------------------------
    def fasta_scan_dev(self, dfile, full_name=False, base_offset=0):
        """-> (device pointer to rows in the context scratch, stats dict)"""
        st = ScanStats()
        d_rows = C.c_void_p()
        check(lib().fxg_fasta_scan(self.ctx, dfile.handle, base_offset, _cabi.SCAN_FULL_NAME if full_name else 0,
                                   C.byref(d_rows), C.byref(st)))
        return d_rows.value, _stats_dict(st)

    def fasta_scan(self, dfile, full_name=False, base_offset=0, keep_device_rows=False):
        d_rows, st = self.fasta_scan_dev(dfile, full_name, base_offset)
        rows = np.zeros(st["n_rows"], dtype=FASTA_ROW)
        if st["n_rows"]:
            check(lib().fxg_rows_download(self.ctx, d_rows, st["n_rows"], FASTA_ROW.itemsize, rows.ctypes.data))
        if keep_device_rows:
            return rows, st, self.upload_rows(rows)
        return rows, st

    def fastq_scan_dev(self, dfile, base_offset=0):
        st = ScanStats()
        d_rows = C.c_void_p()
        check(lib().fxg_fastq_scan(self.ctx, dfile.handle, base_offset, C.byref(d_rows), C.byref(st)))
        return d_rows.value, _stats_dict(st)

    def fastq_scan(self, dfile, base_offset=0, keep_device_rows=False, with_tail=False):
        """rows of the complete reads; with_tail also returns the (partial) row of a trailing incomplete record"""
        d_rows, st = self.fastq_scan_dev(dfile, base_offset)
        n = st["n_rows"]
        has_tail = with_tail and st["n_lines"] % 4 != 0
        rows = np.zeros(n + (1 if has_tail else 0), dtype=FASTQ_ROW)
        if rows.size:
            check(lib().fxg_rows_download(self.ctx, d_rows, rows.size, FASTQ_ROW.itemsize, rows.ctypes.data))
        tail = rows[n].copy() if has_tail else np.zeros(1, dtype=FASTQ_ROW)[0]
        rows = rows[:n]
        if keep_device_rows:
            return rows, st, self.upload_rows(rows)
        if with_tail:
            return rows, st, tail
        return rows, st

    # ---- multi-GPU index build: split-phase scan + the one small exchange (SURVEY 8e) --------
    def scan_begin(self, dfile, mode, base_offset=0, full_name=False, d_info=None):
        """phase A (mark + prefix); the shard's fxg_shard_info lands at device pointer d_info (optional)"""
        check(lib().fxg_scan_begin(self.ctx, dfile.handle, mode, base_offset,
                                   _cabi.SCAN_FULL_NAME if full_name else 0, d_info))

    def scan_finish(self, d_all, nranks, rank, row_dtype):
        """phase B + boundary-row merge + the single host sync -> (rows, stats, all shard infos)"""
        st = ScanStats()
        d_rows = C.c_void_p()
        infos = np.zeros(nranks, dtype=_cabi.SHARD_INFO)
        check(lib().fxg_scan_finish(self.ctx, d_all, nranks, rank, C.byref(d_rows), C.byref(st), infos.ctypes.data))
        rows = np.zeros(st.n_rows, dtype=row_dtype)
        if st.n_rows:
            check(lib().fxg_rows_download(self.ctx, d_rows, st.n_rows, row_dtype.itemsize, rows.ctypes.data))
        return rows, _stats_dict(st), infos

    def scan_sharded_dev(self, comm, dfile, mode, base_offset=0, full_name=False):
        """begin -> in-stream exchange (peer-memory mailboxes, or ncclAllGather as fallback) -> finish on this rank; rows stay on the device.
        -> (device pointer to this shard's rows, stats dict, infos of all ranks)"""
        st = ScanStats()
        d_rows = C.c_void_p()
        nranks = lib().fxg_comm_nranks(comm) if comm else 1
        infos = np.zeros(nranks, dtype=_cabi.SHARD_INFO)
        check(lib().fxg_scan_sharded(self.ctx, comm, dfile.handle, mode, base_offset,
                                     _cabi.SCAN_FULL_NAME if full_name else 0, C.byref(d_rows), C.byref(st),
                                     infos.ctypes.data))
        return d_rows.value, _stats_dict(st), infos

    def scan_sharded(self, comm, dfile, mode, base_offset=0, full_name=False):
        d_rows, st, infos = self.scan_sharded_dev(comm, dfile, mode, base_offset, full_name)
        dt = FASTA_ROW if mode == 0 else FASTQ_ROW
        rows = np.zeros(st["n_rows"], dtype=dt)
        if st["n_rows"]:
            check(lib().fxg_rows_download(self.ctx, d_rows, st["n_rows"], dt.itemsize, rows.ctypes.data))
        return rows, st, infos

    def split_point(self, dfile, start, want_header=False):
        """first line start (or FASTA header line start) at or after `start` in a resident buffer"""
        pos = C.c_int64(0)
        check(lib().fxg_split_point_dev(self.ctx, dfile.handle, int(start), 1 if want_header else 0, C.byref(pos)))
        return pos.value

    def slice_file(self, dfile, begin, end):
        h = C.c_void_p()
        check(lib().fxg_file_slice(self.ctx, dfile.handle, int(begin), int(end), C.byref(h)))
        return DeviceFile(self, h)

    def stage_path_range(self, path, begin, end):
        h = C.c_void_p()
        check(lib().fxg_file_from_path_range(self.ctx, os.fsencode(path), int(begin), int(end), C.byref(h)))
        return DeviceFile(self, h)

    # ---- full-index statistics (K7) ----------------------------------------------------------------
    def fasta_composition(self, dfile, drows, base_offset=0):
        """per-record composition of the resident file -> (COMP_ROW array in (seqid, letter) order, total[128])"""
        out = C.c_void_p()
        n = C.c_int64(0)
        total = np.zeros(128, dtype=np.int64)
        check(lib().fxg_fasta_composition(self.ctx, dfile.handle, drows.devptr, drows.n_rows, base_offset,
                                          C.byref(out), C.byref(n), total.ctypes.data))
        rows = np.zeros(n.value, dtype=_cabi.COMP_ROW)
        if n.value:
            C.memmove(rows.ctypes.data, out.value, n.value * _cabi.COMP_ROW.itemsize)
        lib().fxg_free_host(out)
        return rows, total

    def fastq_stats(self, dfile, drows, n_rows, base_offset=0, trailing_seq=False):
        """A/C/G/T/N totals, min/max read length and quality, phred guess (reference src/fastq.c:663-795)"""
        m = _cabi.FastqMeta()
        check(lib().fxg_fastq_stats(self.ctx, dfile.handle, drows.devptr, n_rows, base_offset, 1 if trailing_seq else 0,
                                    C.byref(m)))
        return {k: getattr(m, k) for k, _ in _cabi.FastqMeta._fields_}

    def dev_alloc(self, nbytes):
        """small device scratch (gathered shard infos in tests / single-process emulation)"""
        return self.upload_rows(np.zeros(max(int(nbytes), 1), dtype=np.uint8))

    def upload_rows(self, rows):
        rows = np.ascontiguousarray(rows)
        d = C.c_void_p()
        check(lib().fxg_rows_upload(self.ctx, rows.ctypes.data if rows.size else None, rows.size,
                                    rows.dtype.itemsize, C.byref(d)))
        return DeviceRows(self, d.value, rows.size, rows.dtype)

    def fasta_build_index_host(self, data, full_name=False):
        """End-to-end host-buffer form: H2D staging + scan + D2H rows in one C call."""
        a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
        cap = max(1024, a.size // 64)
        while True:
            rows = np.zeros(cap, dtype=FASTA_ROW)
            st = ScanStats()
            rc = lib().fxg_fasta_build_index_host(self.ctx, a.ctypes.data if a.size else None, a.size,
                                                  _cabi.SCAN_FULL_NAME if full_name else 0,
                                                  rows.ctypes.data, cap, C.byref(st))
            if rc == _cabi.FXG_ECAP:
                cap = st.n_rows
                continue
            check(rc)
            return rows[:st.n_rows], _stats_dict(st)

    def fastq_build_index_host(self, data):
        a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
        cap = max(1024, a.size // 64)
        while True:
            rows = np.zeros(cap, dtype=FASTQ_ROW)
            st = ScanStats()
            rc = lib().fxg_fastq_build_index_host(self.ctx, a.ctypes.data if a.size else None, a.size,
                                                  rows.ctypes.data, cap, C.byref(st))
            if rc == _cabi.FXG_ECAP:
                cap = st.n_rows
                continue
            check(rc)
            return rows[:st.n_rows], _stats_dict(st)

    # ---- extraction -------------------------------------------------------------------------
    def extract(self, dfile, drows, row_id, s, e, flags=None, want_acgt=False):
        """Batched (row, s, e, flags) -> (out uint8[total], out_off int64[nq+1], acgt int64[nq,4] | None)"""
        row_id = np.ascontiguousarray(row_id, dtype=np.int64)
        s = np.ascontiguousarray(s, dtype=np.int64)
        e = np.ascontiguousarray(e, dtype=np.int64)
        nq = row_id.size
        fl = None if flags is None else np.ascontiguousarray(flags, dtype=np.int32)
        total = int(np.maximum(e - s, 0).sum())
        out = np.empty(max(total, 1), dtype=np.uint8)
        off = np.zeros(nq + 1, dtype=np.int64)
        acgt = np.zeros((nq, 4), dtype=np.int64) if want_acgt else None
        check(lib().fxg_extract_host(self.ctx, dfile.handle, drows.devptr, drows.n_rows, ptr(row_id), ptr(s), ptr(e),
                                     ptr(fl), nq, ptr(off), ptr(out), out.size, ptr(acgt)))
        return out[:total], off, acgt

    def extract_one(self, dfile, drows, row_id, s, e, flags=0):
        """one query, one kernel launch, one synchronisation -> bytes (the per-object getters)"""
        n = e - s
        if n <= 0:
            return b""
        if _fast is not None:
            return _fast.extract_one(self.ctx.value, dfile.handle.value, drows.devptr, drows.n_rows, row_id, s, e, flags)
        buf = C.create_string_buffer(n)
        check(lib().fxg_extract_one_host(self.ctx, dfile.handle, drows.devptr, drows.n_rows, row_id, s, e, flags, buf, n))
        return buf.raw

    def search(self, dfile, drows, row_id, s, e, flags, pattern, strands=_cabi.SEARCH_PLUS, first=False):
        """Exact pattern search (K8) in the haystacks of the queries (row_id, s, e) -- the bytes extraction returns for
        them -- or, with row_id = s = e = None, in every whole record.  -> SEARCH_HIT array of (query, start, minus) in
        (query, start, minus) order, start relative to s; first=True keeps the first hit of each (query, strand)."""
        pat = bytes(pattern)
        nq, rp, sp, ep, keep = self._queries(drows, row_id, s, e)
        out = C.c_void_p()
        n = C.c_int64(0)
        check(lib().fxg_search_host(self.ctx, dfile.handle, drows.devptr, drows.n_rows, rp, sp, ep, int(flags), nq,
                                    pat, len(pat), int(strands), _cabi.SEARCH_FIRST if first else _cabi.SEARCH_ALL,
                                    C.byref(out), C.byref(n)))
        return self._take_hits(out, n)

    def search_approx(self, dfile, drows, row_id, s, e, flags, pattern, max_mismatches, strands=_cabi.SEARCH_PLUS):
        """Search with mismatches: every start of the queries' haystacks (as for search) within max_mismatches
        substitutions of the pattern (or of its reverse complement on the minus strand).  -> SEARCH_HIT array of
        (query, start, minus, mismatches) in (query, start, minus) order, start relative to s."""
        pat = bytes(pattern)
        nq, rp, sp, ep, keep = self._queries(drows, row_id, s, e)
        out = C.c_void_p()
        n = C.c_int64(0)
        check(lib().fxg_search_approx_host(self.ctx, dfile.handle, drows.devptr, drows.n_rows, rp, sp, ep, int(flags),
                                           nq, pat, len(pat), int(max_mismatches), int(strands), C.byref(out),
                                           C.byref(n)))
        return self._take_hits(out, n, with_mismatches=True)

    @staticmethod
    def _queries(drows, row_id, s, e):
        """(nq, row_id, s, e pointers, the arrays they point into) of a search's queries; None: every whole record"""
        if row_id is None:
            return drows.n_rows, None, None, None, None
        row_id = np.ascontiguousarray(row_id, dtype=np.int64)
        s = np.ascontiguousarray(s, dtype=np.int64)
        e = np.ascontiguousarray(e, dtype=np.int64)
        return row_id.size, ptr(row_id), ptr(s), ptr(e), (row_id, s, e)

    def search_reads(self, dfile, drows, pattern, strands=_cabi.SEARCH_PLUS):
        """Exact pattern search (K8 on reads) in every FASTQ read of drows; a read's haystack is its raw sequence line
        (Read.seq).  -> SEARCH_HIT array of (query = read index, start, minus) in (query, start, minus) order."""
        pat = bytes(pattern)
        out = C.c_void_p()
        n = C.c_int64(0)
        check(lib().fxg_search_reads_host(self.ctx, dfile.handle, drows.devptr, drows.n_rows, pat, len(pat), int(strands),
                                          C.byref(out), C.byref(n)))
        return self._take_hits(out, n)

    def search_reads_approx(self, dfile, drows, pattern, max_mismatches, strands=_cabi.SEARCH_PLUS):
        """Search with mismatches in every FASTQ read of drows (haystacks as for search_reads): every start within
        max_mismatches substitutions.  -> SEARCH_HIT array of (query = read index, start, minus, mismatches) in
        (query, start, minus) order."""
        pat = bytes(pattern)
        out = C.c_void_p()
        n = C.c_int64(0)
        check(lib().fxg_search_reads_approx_host(self.ctx, dfile.handle, drows.devptr, drows.n_rows, pat, len(pat),
                                                 int(max_mismatches), int(strands), C.byref(out), C.byref(n)))
        return self._take_hits(out, n, with_mismatches=True)

    @staticmethod
    def _take_hits(out, n, with_mismatches=False):
        hits = np.zeros(n.value, dtype=_cabi.SEARCH_HIT)
        if n.value:
            C.memmove(hits.ctypes.data, out.value, n.value * _cabi.SEARCH_HIT.itemsize)
        lib().fxg_free_host(out)
        return hits if with_mismatches else hits[["query", "start", "minus"]]

    def read_one(self, dfile, drows, read_id, rlen, which=0, flags=0):
        """sequence (which = 0) or quality (1) bytes of one read: one kernel launch, one synchronisation"""
        if rlen <= 0:
            return b""
        if _fast is not None:
            return _fast.read_one(self.ctx.value, dfile.handle.value, drows.devptr, drows.n_rows, read_id, which, flags, rlen)
        buf = C.create_string_buffer(rlen)
        check(lib().fxg_read_one_host(self.ctx, dfile.handle, drows.devptr, drows.n_rows, read_id, which, flags, rlen, buf, rlen))
        return buf.raw

    def reads(self, dfile, drows, ids, flags=0, want_seq=True, want_qual=True, rlens=None):
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        nq = ids.size
        if rlens is None:
            raise ValueError("rlens (host copy of the rows' rlen for these ids) is required to size the output")
        total = int(np.asarray(rlens, dtype=np.int64).sum())
        seq = np.empty(max(total, 1), dtype=np.uint8) if want_seq else None
        qual = np.empty(max(total, 1), dtype=np.uint8) if want_qual else None
        off = np.zeros(nq + 1, dtype=np.int64)
        check(lib().fxg_reads_host(self.ctx, dfile.handle, drows.devptr, drows.n_rows, ptr(ids), nq, flags,
                                   ptr(off), ptr(seq), ptr(qual), max(total, 1)))
        return (seq[:total] if want_seq else None), (qual[:total] if want_qual else None), off
