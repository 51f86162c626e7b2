"""pyfastx-compatible object API (Fasta / Fastq / Sequence / Read) on top of the GPU engine.

Mirrors the reference's Python surface for the hot path -- same class names, constructor
arguments, indexing/slicing semantics (0-based half-open slices, 1-based inclusive `fetch`),
strand getters and error types (reference src/fasta.c, src/sequence.c, src/fastq.c, src/read.c)
-- and adds batched entry points (`fetch_many`, `reads_many`) that feed the GPU gather kernel
with thousands to millions of queries per call.

Every byte that is returned comes from the CUDA kernels in libfxg.so (a single query is a batch
of one); there is no CPU extraction path.  The file stays resident in HBM for the lifetime of
the object.
"""
import gzip as _gzip
import os

import numpy as np

from . import _cabi, fxi
from .engine import get_engine
try:
    from ._fast import extract_one as _fast_one       # compiled bridge into the C-ABI (per-object getters)
except Exception:                                      # not built: the ctypes path of engine.extract_one
    _fast_one = None

__all__ = ["Fasta", "Fastq", "Fastx", "Sequence", "Read", "FastaKeys", "FastqKeys", "version", "gzip_check",
           "reverse_complement"]

VERSION = "2.3.1+b200.1"     # tracks the reference version whose behaviour is reproduced

_RC = _cabi.X_REVERSE | _cabi.X_COMPLEMENT


def version(debug=False):
    if debug:
        return "pyfastx_b200: %s; libfxg ABI: %d; sqlite: %s" % (VERSION, _cabi.lib().fxg_abi_version(),
                                                                 fxi.sqlite3.sqlite_version)
    return VERSION


def gzip_check(file_name):
    """reference src/util.c:307-325: gzip magic number check"""
    with open(file_name, "rb") as f:
        return f.read(2) == b"\x1f\x8b"


def reverse_complement(seq):
    """reference src/module.c:37-59 -> reverse_complement_seq (src/util.c:239-249), on the GPU gather
    kernel: the string is staged as one raw record and fetched with REVERSE|COMPLEMENT|RAW."""
    data = seq.encode("latin-1") if isinstance(seq, str) else bytes(seq)
    if not data:
        return ""
    eng = get_engine()
    f = eng.stage_bytes(data)
    row = np.zeros(1, dtype=_cabi.FASTA_ROW)
    row["blen"] = row["slen"] = len(data)
    row["llen"] = len(data) + 1
    row["elen"] = row["norm"] = 1
    drows = eng.upload_rows(row)
    out, _, _ = eng.extract(f, drows, [0], [0], [len(data)], [_RC | _cabi.X_RAW])
    f.free()
    drows.free()
    return out.tobytes().decode("latin-1")


def _search_position(start, m, minus):
    """What Sequence.search returns for an occurrence at 0-based forward `start` of a pattern of length m: the 1-based
    start on both strands.  (The reference returns the 1-based forward end, start + m, for '-': src/sequence.c:548-549.)"""
    return start + 1


def _locate_args(pattern, strand):
    """(pattern bytes, strands mask) of a locate call; ValueError for a bad strand or pattern length"""
    strands = {"+": _cabi.SEARCH_PLUS, "-": _cabi.SEARCH_MINUS, "both": _cabi.SEARCH_PLUS | _cabi.SEARCH_MINUS}.get(strand)
    if strands is None:
        raise ValueError('strand must be "+", "-" or "both"')
    data = pattern.encode("latin-1") if isinstance(pattern, str) else bytes(pattern)
    if not data or len(data) > _cabi.SEARCH_MAX_PATTERN:
        raise ValueError("pattern length must be 1 .. %d" % _cabi.SEARCH_MAX_PATTERN)
    return data, strands


def _locate_result(hits):
    return (hits["query"].astype(np.int64), hits["start"].astype(np.int64), hits["minus"].astype(bool))


def _locate_approx_args(pattern, mismatches, strand):
    """(pattern bytes, mismatches, strands mask) of a locate_approx call; TypeError for a mismatches that is not an
    integer (a bool is not), ValueError for one outside 0 .. len(pattern) - 1"""
    data, strands = _locate_args(pattern, strand)
    if isinstance(mismatches, (bool, np.bool_)) or not isinstance(mismatches, (int, np.integer)):
        raise TypeError("mismatches must be an integer")
    if not 0 <= mismatches < len(data):
        raise ValueError("mismatches must be 0 .. len(pattern) - 1")
    return data, int(mismatches), strands


def _locate_approx_result(hits):
    return _locate_result(hits) + (hits["mismatches"].astype(np.int32),)


def _gzip_header_len(comp):
    """bytes of the gzip member header (RFC 1952) in front of the deflate data"""
    flg = int(comp[3])
    p = 10
    if flg & 4:
        p += 2 + (int(comp[p]) | (int(comp[p + 1]) << 8))
    for bit in (8, 16):
        if flg & bit:
            while comp[p] != 0:
                p += 1
            p += 1
    if flg & 2:
        p += 2
    return p


class _Staged:
    """file bytes resident in HBM.  Plain files are staged with pinned-chunk copies; BGZF files are
    inflated on the GPU (one thread per member); other gzip streams are inflated by zlib on the host
    while staging (a single deflate stream has no independent entry points)."""

    def __init__(self, path, index_hint=None):
        self.engine = get_engine()
        self.is_gzip = gzip_check(path)
        self.bgzf_members = 0
        self.gzip_path = None        # how a plain .gz got into HBM: "gpu-checkpoints" | "host-zlib"
        self.gzindex = None          # zran-format checkpoints for the .fxi (reference src/util.c:442-540)
        if self.is_gzip:
            with open(path, "rb") as fh:
                comp = np.frombuffer(fh.read(), dtype=np.uint8)
            try:
                cmp_off, ucmp_off = self.engine.bgzf_members(comp)
                self.dfile = self.engine.stage_bgzf(comp)
                self.bgzf_members = self.dfile.n_members
                self.gzindex = fxi.bgzf_gzindex(comp, cmp_off, ucmp_off)
            except _cabi.FxgError as ex:
                if ex.code != _cabi.FXG_EFORMAT:
                    raise
                # a single serial deflate stream.  With the checkpoints of an earlier open (the gzindex rows of the
                # .fxi) every segment is inflated by its own GPU thread, checked against the trailer's CRC-32 ...
                pts = fxi.read_gzindex(index_hint) if index_hint and index_hint != ":memory:" and os.path.exists(index_hint) else None
                if pts is not None and pts["compressed_size"] == comp.size and pts["windows"] == pts["npoints"] - 1:
                    try:
                        self.dfile = self.engine.stage_gzip_points(comp, pts)
                        self.gzindex, self.gzip_path = pts, "gpu-checkpoints"
                    except _cabi.FxgError as ex2:
                        if ex2.code != _cabi.FXG_EFORMAT:
                            raise
                if self.gzip_path is None:
                    # ... without them: the one sequential zlib pass on the host (the reference inflates the file twice:
                    # gzread under the scan, then zran_build_index), collecting the zran checkpoints in the same pass
                    view, self.gzindex, self._gz_handle = self.engine.gzip_inflate(comp)
                    self.dfile = self.engine.stage_bytes(view)
                    self.gzip_path = "host-zlib"
        else:
            import time as _t
            t0 = _t.perf_counter()
            self.dfile = self.engine.stage_path(path)
            if os.environ.get("FXG_TIMING"):
                import sys as _s
                print("[fxg timing] stage_path %.3f s (%.2f GB)" % (_t.perf_counter() - t0, self.dfile.size / 1e9), file=_s.stderr)

    def first_non_space(self):
        head = self.dfile.download(0, min(self.dfile.size, 1 << 16))
        for c in head.tolist():
            if c not in (9, 10, 11, 12, 13, 32):
                return c
        return None

    def ranges_packed(self, offsets, lengths):
        """(packed uint8, offsets[n+1]) of the given file ranges (batched GPU gather) -- no Python objects"""
        if len(offsets) == 0:
            return np.zeros(0, dtype=np.uint8), np.zeros(1, dtype=np.int64)
        return self.engine.gather_ranges(self.dfile, offsets, lengths)

    def ranges(self, offsets, lengths):
        """list of bytes objects for the given file ranges (batched GPU gather)"""
        buf, off = self.ranges_packed(offsets, lengths)
        raw = buf.tobytes()
        return [raw[off[i]:off[i + 1]] for i in range(len(offsets))]

    def close(self):
        try:
            self.dfile.free()
        except Exception:
            pass

    def __del__(self):
        try:
            h = getattr(self, "_gz_handle", None)
            if h:
                self.engine.gzip_free(h)
                self._gz_handle = None
        except Exception:
            pass


class _Keys:
    """names of an index in file order (reference FastaKeys / FastqKeys, src/fakeys.c, src/fqkeys.c: len, iteration,
    indexing, `in`); backed by the packed name buffer + the native hash table instead of SQL."""

    def __init__(self, names, what):
        self._names, self._what = names, what

    def __len__(self):
        return len(self._names)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self._names.get(k) for k in range(*i.indices(len(self)))]
        n = len(self)
        if i < 0:
            i += n
        if i < 0 or i >= n:
            raise IndexError("index out of range")
        return self._names.get(i)

    def __iter__(self):
        return (self._names.get(i) for i in range(len(self)))

    def __contains__(self, name):
        return isinstance(name, str) and self._names.find(name) >= 0

    def __eq__(self, other):
        return list(self) == list(other)

    def __repr__(self):
        return "<%s> contains %d keys" % (self._what, len(self))


class FastaKeys(_Keys):
    pass


class FastqKeys(_Keys):
    pass


class Fastx:
    """Fastx(file_name, format="auto", uppercase=False, comment=False): iterate (name, seq[, comment]) of a FASTA
    or (name, seq, qual[, comment]) of a FASTQ file without keeping an index file (reference src/fastx.c:42-43).
    Records come from the GPU scan + batched gather, a few thousand per round trip."""

    def __init__(self, file_name, format="auto", uppercase=False, comment=False):
        file_name = os.fspath(file_name)
        if not os.path.exists(file_name):
            raise FileExistsError("the input file %s does not exists" % file_name)
        self.file_name, self.uppercase, self.comment = file_name, bool(uppercase), bool(comment)
        self._st = _Staged(file_name)
        first = self._st.first_non_space()
        if format == "auto":
            format = "fasta" if first == ord(">") else ("fastq" if first == ord("@") else None)
        if format not in ("fasta", "fastq"):
            raise RuntimeError("%s is not fasta or fastq sequence file" % file_name)
        self.format = format

    def __iter__(self):
        st, eng = self._st, self._st.engine
        step = 4096
        if self.format == "fasta":
            rows, _ = eng.fasta_scan(st.dfile)
            drows = eng.upload_rows(rows)
            hoff = rows["boff"] - rows["elen"].astype(np.int64) - rows["dlen"]
            flags = _cabi.X_UPPER if self.uppercase else 0
            for a in range(0, len(rows), step):
                b = min(len(rows), a + step)
                rid = np.arange(a, b, dtype=np.int64)
                out, off, _ = eng.extract(st.dfile, drows, rid, np.zeros(b - a, np.int64), rows["slen"][a:b],
                                          np.full(b - a, flags, np.int32))
                hdr = st.ranges(hoff[a:b], rows["dlen"][a:b].astype(np.int64))
                buf = out.tobytes()
                for k in range(b - a):
                    h = hdr[k].decode("latin-1")
                    name = h[:int(rows["nlen"][a + k])]
                    seq = buf[off[k]:off[k + 1]].decode("latin-1")
                    yield (name, seq, h[len(name) + 1:]) if self.comment else (name, seq)
        else:
            rows, _ = eng.fastq_scan(st.dfile)
            drows = eng.upload_rows(rows)
            for a in range(0, len(rows), step):
                b = min(len(rows), a + step)
                ids = np.arange(a, b, dtype=np.int64)
                seq, qual, off = eng.reads(st.dfile, drows, ids, rlens=rows["rlen"][a:b])
                hdr = st.ranges(rows["soff"][a:b] - rows["dlen"][a:b], rows["dlen"][a:b].astype(np.int64) - 1)
                sb, qb = seq.tobytes(), qual.tobytes()
                for k in range(b - a):
                    h = hdr[k].rstrip(b"\r").decode("latin-1")
                    name = h[:int(rows["nlen"][a + k])]
                    s = sb[off[k]:off[k + 1]].decode("latin-1")
                    if self.uppercase:
                        s = s.upper()
                    rec = (name, s, qb[off[k]:off[k + 1]].decode("latin-1"))
                    yield rec + (h[len(name) + 1:],) if self.comment else rec


# =================================================================================================
# FASTA
# =================================================================================================
class Fasta:
    """Fasta(file_name, index_file=None, uppercase=False, build_index=True, full_index=False,
             full_name=False, memory_index=False, key_func=None)      (reference src/fasta.c:39-129)"""

    def __init__(self, file_name, index_file=None, uppercase=False, build_index=True, full_index=False,
                 full_name=False, memory_index=False, key_func=None):
        if key_func is not None and not callable(key_func):
            raise TypeError("key_func must be a callable function")
        file_name = os.fspath(file_name)
        if not os.path.exists(file_name):
            raise FileExistsError("the input fasta file %s does not exists" % file_name)
        self.file_name = file_name
        self.uppercase = bool(uppercase)
        self.full_name = bool(full_name)
        self.key_func = key_func
        self.index_file = ":memory:" if memory_index else (os.fspath(index_file) if index_file else file_name + ".fxi")
        self._st = _Staged(file_name, self.index_file)
        self.is_gzip = self._st.is_gzip
        if self._st.first_non_space() != ord(">"):
            raise RuntimeError("%s is not plain or gzip compressed fasta formatted file" % file_name)
        self._rows = None
        self._names = None
        self._drows = None
        self._con = None
        self._comp_cache = None
        self._slen_cache = None
        self._one_args = None
        if build_index:
            self.build_index()
            if full_index:
                self._calc_composition()

    # ---- index ---------------------------------------------------------------------------------
    def build_index(self):
        """load the .fxi if it exists, else scan on the GPU and write it (src/index.c:418-429)"""
        if self._rows is not None:
            return
        if self.index_file != ":memory:" and os.path.exists(self.index_file):
            self._con, self._rows, self._names, stat = fxi.load_fasta_index(self.index_file)
            self._total = int(stat[1]) if stat else int(self._rows["slen"].sum())
            self.index_matches_file = self._verify_loaded_index()
        else:
            self._scan_and_write(self.index_file)
        self._drows = self._st.engine.upload_rows(self._rows)

    def _scan_names(self, rows):
        """names of the scanned records as PackedNames (GPU gather of the header spans)"""
        name_off = rows["boff"] - rows["elen"].astype(np.int64) - rows["dlen"]
        if self.key_func is None:
            blob, off = self._st.ranges_packed(name_off, rows["nlen"].astype(np.int64))
            return fxi.PackedNames(blob, off)
        # key_func receives the header text after '>' exactly as the reference passes it
        # (NUL-terminated line, i.e. including a trailing '\r'), src/index.c:304-318
        hdrs = self._st.ranges(name_off, rows["dlen"].astype(np.int64) + rows["elen"].astype(np.int64) - 1)
        return fxi.PackedNames.from_list([str(self.key_func(h.decode("latin-1"))).encode("utf-8") for h in hdrs])

    def _scan_and_write(self, index_file):
        import time as _t
        eng = self._st.engine
        t0 = _t.perf_counter()
        rows, st = eng.fasta_scan(self._st.dfile, full_name=self.full_name)
        t1 = _t.perf_counter()
        self._names = self._scan_names(rows)
        t2 = _t.perf_counter()
        self._rows, self._total = rows, int(st["total_len"])
        self._con = fxi.write_fasta_index_packed(index_file, rows, self._names.blob, self._names.off, self._total,
                                                 gz=self._st.gzindex)
        if os.environ.get("FXG_TIMING"):
            import sys as _s
            print("[fxg timing] scan %.3f s, names %.3f s, fxi %.3f s" % (t1 - t0, t2 - t1, _t.perf_counter() - t2), file=_s.stderr)

    def _verify_loaded_index(self):
        """A loaded .fxi carries no line-uniformity bits; one GPU scan (milliseconds) recovers them and doubles
        as a staleness check.  Rows that disagree with the file never reach the kernels: the scan's own rows
        (and names) replace them in memory, and the stale file is left alone."""
        rows, st = self._st.engine.fasta_scan(self._st.dfile, full_name=self.full_name)
        same = len(rows) == len(self._rows) and all(
            np.array_equal(rows[f], self._rows[f]) for f in ("boff", "blen", "slen", "llen", "elen", "norm", "dlen"))
        if same:
            self._rows["pad"] = rows["pad"]
        else:
            self._names = self._scan_names(rows)
            self._rows, self._total = rows, int(st["total_len"])
        return same

    def _need_index(self):
        if self._rows is None:
            self.build_index()

    # ---- container protocol -----------------------------------------------------------------------
    def __len__(self):
        self._need_index()
        return len(self._rows)

    @property
    def size(self):
        self._need_index()
        return self._total

    def __contains__(self, name):
        self._need_index()
        return isinstance(name, str) and self._names.find(name) >= 0

    def keys(self):
        self._need_index()
        return FastaKeys(self._names, "FastaKeys")

    def _row_id(self, key):
        self._need_index()
        if isinstance(key, (int, np.integer)):
            i = int(key)
            if i < 0:
                i += len(self._rows)
            if i < 0 or i >= len(self._rows):
                raise IndexError("index out of range")
            return i
        if isinstance(key, str):
            i = self._names.find(key)
            if i < 0:
                raise KeyError("%s does not exist in fasta file" % key)
            return i
        raise KeyError("the key must be index number or sequence name")

    def __getitem__(self, key):
        i = self._names.find(key) if type(key) is str else -2       # the common call: a name
        if i < 0:
            i = self._row_id(key)
        sl = self._slen_cache
        if sl is None or len(sl) != len(self._rows):
            sl = self._slen_cache = np.ascontiguousarray(self._rows["slen"])
        return Sequence(self, i, 0, int(sl[i]), True, report_end=False)

    def __iter__(self):
        self._need_index()
        for i in range(len(self._rows)):
            yield Sequence(self, i, 0, int(self._rows["slen"][i]), True)

    def __repr__(self):
        return "<Fasta> %s contains %d seqs" % (self.file_name, len(self))

    # ---- batched extraction (additive API feeding K3) -----------------------------------------------
    def _flags(self, extra=0):
        return (_cabi.X_UPPER if self.uppercase else 0) | extra

    def extract(self, row_id, start, end, strand_minus=None, want_acgt=False, whole_record=False):
        """Batched 0-based half-open queries -> (packed uint8 array, offsets[nq+1], acgt[nq,4] | None).
        whole_record=True gives Fasta.fetch semantics (index into the whole stripped record)."""
        self._need_index()
        row_id = np.asarray(row_id, dtype=np.int64)
        s = np.asarray(start, dtype=np.int64)
        e = np.asarray(end, dtype=np.int64)
        slen = self._rows["slen"][row_id]
        s = np.clip(s, 0, slen)
        e = np.clip(e, s, slen)
        flags = np.full(row_id.size, self._flags(_cabi.X_WHOLE if whole_record else 0), dtype=np.int32)
        if strand_minus is not None:
            flags |= np.where(np.asarray(strand_minus, dtype=bool), _RC, 0).astype(np.int32)
        return self._st.engine.extract(self._st.dfile, self._drows, row_id, s, e, flags, want_acgt=want_acgt)

    def fetch_many(self, names, starts, ends, strands=None):
        """Batched form of fetch(): 1-based inclusive (start, end) per query, strand '+'/'-'.
        Returns a list of str."""
        self._need_index()
        names = list(names) if not isinstance(names, (list, fxi.PackedNames)) else names
        if isinstance(names, fxi.PackedNames) or all(isinstance(n, str) for n in names):
            rid = self._names.lookup(names)          # native batched name -> row (one call, many threads)
            bad = np.nonzero(rid < 0)[0]
            if bad.size:
                k = int(bad[0])
                raise NameError("Sequence %s does not exists" % (names.get(k) if isinstance(names, fxi.PackedNames) else names[k]))
        else:
            rid = np.fromiter((self._row_id(n) for n in names), dtype=np.int64)
        s = np.asarray(starts, dtype=np.int64)
        e = np.asarray(ends, dtype=np.int64)
        if (s > e).any():
            raise ValueError("start position should less than end position")
        minus = None if strands is None else np.array([c == "-" for c in strands], dtype=bool)
        out, off, _ = self.extract(rid, s - 1, e, minus, whole_record=True)
        buf = out.tobytes()
        return [buf[off[i]:off[i + 1]].decode("latin-1") for i in range(rid.size)]

    def _one(self, i, s, e, extra=0):
        if _fast_one is not None:
            a = self._one_args
            if a is None or a[3] is not self._drows:
                eng = self._st.engine
                a = self._one_args = (eng.ctx.value, self._st.dfile.handle.value, self._drows.devptr, self._drows, self._drows.n_rows)
            if e <= s:
                return ""
            return _fast_one(a[0], a[1], a[2], a[4], i, s, e, (_cabi.X_UPPER if self.uppercase else 0) | extra).decode("latin-1")
        return self._st.engine.extract_one(self._st.dfile, self._drows, i, s, e, self._flags(extra)).decode("latin-1")

    def locate(self, pattern, strand="+"):
        """Every occurrence of `pattern` (str or bytes, compared byte for byte, case-sensitive) in every record, found by
        the search kernel on the resident file: strand "+" the pattern, "-" its reverse complement, "both" either;
        overlapping occurrences all count.  With uppercase=True the records are upper-cased first, as their .seq is.
        -> (row_id int64, start int64, minus bool) arrays sorted by (row_id, start, minus); start is the 0-based start in
        the record's forward coordinates."""
        data, strands = _locate_args(pattern, strand)
        self._need_index()
        return _locate_result(self._st.engine.search(self._st.dfile, self._drows, None, None, None, self._flags(), data,
                                                     strands))

    def locate_approx(self, pattern, mismatches, strand="+"):
        """Every start in every record where `pattern` matches with at most `mismatches` substituted bytes (Hamming
        distance; byte for byte and case-sensitive, so N against A is a mismatch), found by the search kernel on the
        resident file.  Strand and uppercase=True as for locate; a match never runs past its record's end.
        0 <= mismatches < len(pattern); mismatches = 0 gives locate's hits.
        -> (row_id int64, start int64, minus bool, mismatches int32) arrays sorted by (row_id, start, minus); the last
        holds each hit's count of mismatches against the strand it matched."""
        data, k, strands = _locate_approx_args(pattern, mismatches, strand)
        self._need_index()
        return _locate_approx_result(self._st.engine.search_approx(self._st.dfile, self._drows, None, None, None,
                                                                   self._flags(), data, k, strands))

    # ---- reference methods -------------------------------------------------------------------------
    def fetch(self, chrom, intervals, strand="+"):
        """1-based inclusive interval(s) of `chrom`; '-' = reverse complement of the concatenation
        (reference src/fasta.c:384-515)."""
        if not isinstance(intervals, (list, tuple)):
            raise ValueError("intervals must be list or tuple")
        self._need_index()
        i = self._names.find(chrom) if isinstance(chrom, str) else -1
        if i < 0:
            raise NameError("Sequence %s does not exists" % chrom)
        if intervals and isinstance(intervals[0], (int, np.integer)):
            if len(intervals) != 2:
                raise ValueError("list or tuple should include only start and end")
            ivs = [(int(intervals[0]), int(intervals[1]))]
        else:
            ivs = [(int(a), int(b)) for a, b in intervals]
        for a, b in ivs:
            if a > b:
                raise ValueError("start position should less than end position")
        minus = strand == "-"
        if minus:
            ivs = ivs[::-1]            # RC(concat(a, b)) == RC(b) + RC(a)
        rid = np.full(len(ivs), i, dtype=np.int64)
        s = np.array([a - 1 for a, _ in ivs], dtype=np.int64)
        e = np.array([b for _, b in ivs], dtype=np.int64)
        out, _, _ = self.extract(rid, s, e, np.full(len(ivs), minus), whole_record=True)
        return out.tobytes().decode("latin-1")

    def flank(self, chrom, start, end, flank_length=50, use_cache=False):
        """(left, right) flanks of the 1-based inclusive interval (reference src/fasta.c:322-382)."""
        if flank_length < 0:
            raise ValueError("Flank length must be non-negative")
        self._need_index()
        i = self._names.find(chrom) if isinstance(chrom, str) else -1
        if i < 0:
            raise NameError("sequence %s does not exists" % chrom)
        slen = int(self._rows["slen"][i])
        ls, le = max(0, start - flank_length - 1), max(0, start - 1)
        rs, re = min(end, slen), min(end + flank_length, slen)
        out, off, _ = self.extract([i, i], [ls, rs], [le, re])
        buf = out.tobytes().decode("latin-1")
        return buf[off[0]:off[1]], buf[off[1]:off[2]]

    # ---- statistics ------------------------------------------------------------------------------------
    def _lengths(self):
        self._need_index()
        return self._rows["slen"]

    @property
    def longest(self):
        i = int(np.argmax(self._lengths()))
        return self[i]

    @property
    def shortest(self):
        i = int(np.argmin(self._lengths()))
        return self[i]

    @property
    def mean(self):
        return float(self.size) / len(self)

    @property
    def median(self):
        return float(np.median(self._lengths()))

    def count(self, n):
        return int((self._lengths() >= n).sum())

    def nl(self, p=50):
        """(N, L) statistics, e.g. nl(50) = (N50, L50) (reference src/fasta.c:599-683)."""
        if p < 0 or p > 100:
            raise ValueError("the value must between 0 and 100")
        lens = np.sort(self._lengths())[::-1]
        half = p / 100.0 * self.size
        csum = np.cumsum(lens)
        k = int(np.searchsorted(csum, half, side="left"))
        k = min(k, len(lens) - 1)
        return int(lens[k]), k + 1

    def _calc_composition(self):
        """pyfastx_fasta_calc_composition (src/fasta.c:851-961): per-record byte composition -> `comp` rows, computed
        once on the GPU (fxg_fasta_composition) and persisted in the .fxi like the reference does on first use."""
        if self._comp_cache is not None:
            return self._comp_cache
        self._need_index()
        comp = None
        if self._con is not None:
            try:
                comp = fxi.load_comp(self._con)
            except Exception:
                comp = None
        if comp is None or len(comp) == 0:
            rows, total = self._st.engine.fasta_composition(self._st.dfile, self._drows)
            tot_rows = np.zeros(128, dtype=_cabi.COMP_ROW)           # the reference's 128 rows with seqid 0
            tot_rows["abc"] = np.arange(128)
            tot_rows["num"] = total
            comp = np.concatenate([rows, tot_rows])
            if self.index_file != ":memory:":
                if self._con is not None:
                    self._con.close()
                self._con = fxi.write_fasta_index_packed(self.index_file, self._rows, self._names.blob, self._names.off,
                                                         self._total, gz=self._st.gzindex, comp=comp)
        self._comp_rows = comp
        tot = np.zeros(128, dtype=np.int64)
        z = comp[comp["seqid"] == 0]
        tot[z["abc"]] = z["num"]
        self._comp_cache = tot
        return tot

    @property
    def composition(self):
        h = self._calc_composition()
        return {chr(i): int(h[i]) for i in range(32, 127) if h[i] > 0}       # src/fasta.c:1092

    @property
    def gc_content(self):
        h = self._calc_composition()
        a, c, g, t = (int(h[ord(x)] + h[ord(x.lower())]) for x in "ACGT")
        if a + c + g + t <= 0:
            raise RuntimeError("could not calculate gc content")
        return float(np.float32(g + c) / np.float32(a + c + g + t) * np.float32(100))

    @property
    def gc_skew(self):
        h = self._calc_composition()
        c, g = (int(h[ord(x)] + h[ord(x.lower())]) for x in "CG")
        if c + g <= 0:
            raise RuntimeError("could not calculate gc skew")
        return float(np.float32(g - c) / np.float32(g + c))

    @property
    def type(self):
        """DNA / RNA / protein / unknown from the alphabet in use (reference src/fasta.c:1104-1154)"""
        h = self._calc_composition()
        alpha = {chr(i) for i in range(33, 127) if h[i] > 0}
        if alpha <= set("ACGTNacgtn") or alpha <= set("abcdghkmnrstvwyABCDGHKMNRSTVWY*-"):
            return "DNA"
        if alpha <= set("ACGUNacgun") or alpha <= set("abcdghkmnrsuvwyABCDGHKMNRSUVWY*-"):
            return "RNA"
        if alpha <= set("acdefghiklmnpqrstvwyACDEFGHIKLMNPQRSTVWY*-"):
            return "protein"
        return "unknown"


class Sequence:
    """A record or a slice of one (reference src/sequence.c).  start/end are 1-based inclusive."""

    def __init__(self, fasta, row_id, s, e, complete, report_end=True):
        self._fa, self.id = fasta, row_id + 1
        self._i, self._s, self._e = row_id, s, e
        self._complete = complete
        # reference quirk Q10 (SURVEY 8a), reproduced: a whole record obtained by index or name reports end = 0
        # (src/index.c:482-483); only the iterator sets end = seq_len (src/index.c:522); slices report s + 1 .. e
        self.start, self.end = s + 1, (e if report_end else 0)

    @property
    def name(self):
        return self._fa._names.get(self._i)

    def __len__(self):
        return self._e - self._s

    def _get(self, extra=0):
        if self._e <= self._s:
            return ""
        return self._fa._one(self._i, self._s, self._e, extra)

    @property
    def seq(self):
        return self._get()

    @property
    def reverse(self):
        return self._get(_cabi.X_REVERSE)

    @property
    def complement(self):
        return self._get(_cabi.X_COMPLEMENT)

    @property
    def antisense(self):
        return self._get(_RC)

    def __str__(self):
        return self.seq

    def __repr__(self):
        if self._complete:
            return "<Sequence> %s with length of %d" % (self.name, len(self))
        return "<Sequence> %s from %d to %d" % (self.name, self.start, self.end)

    def __getitem__(self, item):
        n = len(self)
        if isinstance(item, slice):
            a, b, step = item.indices(n)
            if step != 1:
                raise ValueError("slice step cannot > 1" if step else "slice step cannot be zero")
            b = max(a, b)
            return Sequence(self._fa, self._i, self._s + a, self._s + b, self._complete and (b - a) == n)
        i = int(item)
        if i < 0:
            i += n
        if i < 0 or i >= n:
            raise IndexError("index out of range")
        return self._fa._one(self._i, self._s + i, self._s + i + 1)

    def __contains__(self, sub):
        if isinstance(sub, str) and 0 < len(sub) <= _cabi.SEARCH_MAX_PATTERN:
            try:
                data = sub.encode("latin-1")
            except UnicodeEncodeError:
                return False
            return self._first_hit(data, False) is not None
        return sub in self.seq

    def __iter__(self):
        """sequence lines of a complete record (reference src/sequence.c:162-263)"""
        if not self._complete:
            raise RuntimeError("sliced subsequence cannot be read line by line")
        r = self._fa._rows[self._i]
        raw = bytes(self._fa._st.dfile.download(int(r["boff"]), min(int(r["blen"]), self._fa._st.dfile.size - int(r["boff"]))))
        for line in raw.split(b"\n"):
            line = line.rstrip(b"\r")
            if line:
                yield line.decode("latin-1")

    @property
    def description(self):
        r = self._fa._rows[self._i]
        a = int(r["boff"]) - int(r["elen"]) - int(r["dlen"])
        return bytes(self._fa._st.dfile.download(a, int(r["dlen"]))).decode("latin-1")

    @property
    def raw(self):
        r = self._fa._rows[self._i]
        if self._complete:
            a = int(r["boff"]) - int(r["elen"]) - int(r["dlen"]) - 1
            n = min(int(r["boff"]) + int(r["blen"]), self._fa._st.dfile.size) - a
        else:
            bpl = int(r["llen"]) - int(r["elen"])
            a = int(r["boff"]) + self._s + int(r["elen"]) * (self._s // bpl)
            n = (self._e - self._s) + (self._e // bpl - self._s // bpl) * int(r["elen"])
        return bytes(self._fa._st.dfile.download(a, n)).decode("latin-1")

    def _acgt(self):
        _, _, acgt = self._fa.extract([self._i], [self._s], [self._e], want_acgt=True)
        return [int(x) for x in acgt[0]]

    @property
    def gc_content(self):
        a, c, g, t = self._acgt()
        return float(np.float32(g + c) / np.float32(a + c + g + t) * np.float32(100))

    @property
    def gc_skew(self):
        _, c, g, _ = self._acgt()
        return float(np.float32(g - c) / np.float32(g + c))

    @property
    def composition(self):
        fa = self._fa
        h = np.zeros((1, 256), dtype=np.int64)
        one = lambda v: np.array([v], dtype=np.int64)
        rid, s, e = one(self._i), one(self._s), one(self._e)
        fl = np.array([fa._flags()], dtype=np.int32)
        _cabi.check(_cabi.lib().fxg_composition_host(fa._st.engine.ctx, fa._st.dfile.handle, fa._drows.devptr,
                                                    len(fa._rows), rid.ctypes.data, s.ctypes.data, e.ctypes.data,
                                                    fl.ctypes.data, 1, h.ctypes.data))
        return {chr(i): int(h[0, i]) for i in range(32, 127) if h[0, i] > 0}

    def _first_hit(self, data, minus):
        """0-based start of the first occurrence of `data` (bytes, 1 .. SEARCH_MAX_PATTERN long) in this sequence, or of
        its reverse complement if `minus`, found by the search kernel where the record lies in HBM; None if there is none"""
        fa = self._fa
        q = np.array([self._i, self._s, self._e], dtype=np.int64)
        hits = fa._st.engine.search(fa._st.dfile, fa._drows, q[0:1], q[1:2], q[2:3], fa._flags(), data,
                                    _cabi.SEARCH_MINUS if minus else _cabi.SEARCH_PLUS, first=True)
        return int(hits["start"][0]) if hits.size else None

    def search(self, subseq, strand="+"):
        """1-based position of the first match or None (reference src/sequence.c:519-560).  A str pattern of up to
        SEARCH_MAX_PATTERN characters is searched on the GPU; any other pattern takes the host scan of the sequence."""
        minus = strand != "+"
        if isinstance(subseq, str):
            if not subseq:
                return 1                                       # str.find("") == 0
            if len(subseq) <= _cabi.SEARCH_MAX_PATTERN:
                try:
                    data = subseq.encode("latin-1")
                except UnicodeEncodeError:                     # the sequence holds latin-1 characters only
                    data = None
                if data is not None:
                    k = self._first_hit(data, minus)
                    return None if k is None else _search_position(k, len(data), minus)
                if not minus:
                    return None
        q = reverse_complement(subseq) if minus else subseq
        k = self.seq.find(q)
        return _search_position(k, len(q), minus) if k >= 0 else None


# =================================================================================================
# FASTQ
# =================================================================================================
class Fastq:
    """Fastq(file_name, index_file=None, phred=0, build_index=True, full_index=False, full_name=False)
    (reference src/fastq.c:257-376)"""

    def __init__(self, file_name, index_file=None, phred=0, build_index=True, full_index=False, full_name=False):
        file_name = os.fspath(file_name)
        if not os.path.exists(file_name):
            raise FileExistsError("input fastq file %s does not exists" % file_name)
        self.file_name = file_name
        self.index_file = os.fspath(index_file) if index_file else file_name + ".fxi"
        self._st = _Staged(file_name, self.index_file)
        self.is_gzip = self._st.is_gzip
        if self._st.first_non_space() != ord("@"):
            raise RuntimeError("%s is not plain or gzip compressed fastq formatted file" % file_name)
        self._phred = phred
        self._rows = None
        self._meta = None
        self._full_index = bool(full_index)
        if build_index:
            self.build_index()
            if full_index:
                self._calc_composition()

    def build_index(self):
        if self._rows is not None:
            return True
        if os.path.exists(self.index_file):
            self._con, self._rows, self._names, stat = fxi.load_fastq_index(self.index_file)
            self._counts, self.size, self.avglen = int(stat[0]), int(stat[1]), stat[2]
            self._n_lines = None                     # a loaded index does not say whether a partial record trails
            self._validate_loaded_rows()
        else:
            eng = self._st.engine
            rows, st, self._tail_row = eng.fastq_scan(self._st.dfile, with_tail=True)
            self._n_lines = int(st["n_lines"])
            blob, off = self._st.ranges_packed(rows["soff"] - rows["dlen"], rows["nlen"].astype(np.int64))
            self._names = fxi.PackedNames(blob, off)
            self._rows = rows
            self._counts = st["n_lines"] // 4
            self.size = int(st["total_len"])
            self.avglen = self.size * 1.0 / self._counts if self._counts else float("nan")
            self._con = fxi.write_fastq_index_packed(self.index_file, rows, blob, off, st["n_lines"], self.size,
                                                     gz=self._st.gzindex)
        self._drows = self._st.engine.upload_rows(self._rows)
        return True

    def _validate_loaded_rows(self):
        """rows of a loaded .fxi must address bytes inside the staged file before they reach the kernels"""
        r, n = self._rows, self._st.dfile.size
        ok = ((r["soff"] >= 0) & (r["qoff"] >= 0) & (r["rlen"] >= 0) & (r["soff"] + r["rlen"] <= n) &
              (r["qoff"] + r["rlen"] <= n) & (r["dlen"] >= 0) & (r["soff"] - r["dlen"] >= 0)).all()
        if not ok:
            raise RuntimeError("the index file %s does not match %s" % (self.index_file, self.file_name))

    def __len__(self):
        self.build_index()
        return self._counts

    def __contains__(self, name):
        self.build_index()
        return isinstance(name, str) and self._names.find(name) >= 0

    def keys(self):
        self.build_index()
        return FastqKeys(self._names, "FastqKeys")

    def _row_id(self, key):
        self.build_index()
        if isinstance(key, (int, np.integer)):
            i = int(key)
            if i < 0:
                i += len(self._rows)
            if i < 0 or i >= len(self._rows):
                raise IndexError("index out of range")
            return i
        if isinstance(key, str):
            i = self._names.find(key)
            if i < 0:
                raise KeyError("%s does not exist in fastq file" % key)
            return i
        raise KeyError("the key must be index number or read name")

    def __getitem__(self, key):
        return Read(self, self._row_id(key))

    def __iter__(self):
        self.build_index()
        for i in range(len(self._rows)):
            yield Read(self, i)

    def __repr__(self):
        return "<Fastq> %s contains %d reads" % (self.file_name, len(self))

    def reads_many(self, ids, want_qual=True, strand_minus=False):
        """Batched read fetch -> (seq packed uint8, qual packed uint8 | None, offsets[n+1])"""
        self.build_index()
        ids = np.asarray(ids, dtype=np.int64)
        flags = _RC if strand_minus else 0
        return self._st.engine.reads(self._st.dfile, self._drows, ids, flags=flags, want_qual=want_qual,
                                     rlens=self._rows["rlen"][ids])

    def locate(self, pattern, strand="+"):
        """Every occurrence of `pattern` (str or bytes, compared byte for byte, case-sensitive) in every read's sequence
        (exactly Read.seq: nothing stripped or upper-cased), found by the search kernel on the resident file: strand "+"
        the pattern, "-" its reverse complement, "both" either; overlapping occurrences all count, and no occurrence runs
        past the end of its read.  -> (read_id int64, start int64, minus bool) arrays sorted by (read_id, start, minus);
        fq[int(read_id[k])] is the read of hit k, start its 0-based forward start."""
        data, strands = _locate_args(pattern, strand)
        self.build_index()
        return _locate_result(self._st.engine.search_reads(self._st.dfile, self._drows, data, strands))

    def locate_approx(self, pattern, mismatches, strand="+"):
        """Every start in every read's sequence (exactly Read.seq) where `pattern` matches with at most `mismatches`
        substituted bytes (Hamming distance; byte for byte and case-sensitive, so N against A is a mismatch), found by
        the search kernel on the resident file.  Strand as for locate; a match never runs past its read's end.
        0 <= mismatches < len(pattern); mismatches = 0 gives locate's hits.
        -> (read_id int64, start int64, minus bool, mismatches int32) arrays sorted by (read_id, start, minus); the last
        holds each hit's count of mismatches against the strand it matched."""
        data, k, strands = _locate_approx_args(pattern, mismatches, strand)
        self.build_index()
        return _locate_approx_result(self._st.engine.search_reads_approx(self._st.dfile, self._drows, data, k, strands))

    def _calc_composition(self):
        """pyfastx_fastq_calc_composition (src/fastq.c:663-795): base totals, min / max length and quality, phred
        guess -- one GPU pass over the sequence and quality lines; persisted in the `base` / `meta` tables."""
        if self._meta is not None:
            return self._meta
        self.build_index()
        meta = None
        if self._con is not None:
            try:
                m = self._con.execute("SELECT maxlen,minlen,minqs,maxqs,phred FROM meta LIMIT 1").fetchone()
                b = self._con.execute("SELECT a,c,g,t,n FROM base LIMIT 1").fetchone()
                if m and b:
                    meta = dict(zip(("maxlen", "minlen", "minqs", "maxqs", "phred", "a", "c", "g", "t", "n"), [int(x) for x in m + b]))
            except Exception:
                meta = None
        if meta is None:
            eng = self._st.engine
            # a trailing partial record's sequence line is counted by the reference too (it walks lines, not reads)
            trailing = (self._n_lines % 4) >= 2 if self._n_lines is not None else False
            drows = self._drows
            if trailing:
                full = np.zeros(len(self._rows) + 1, dtype=_cabi.FASTQ_ROW)
                full[:-1] = self._rows
                full[-1] = self._tail_row
                drows = eng.upload_rows(full)
            meta = eng.fastq_stats(self._st.dfile, drows, len(self._rows), trailing_seq=trailing)
            if self._con is not None and self._n_lines is not None:
                self._con.close()
                self._con = fxi.write_fastq_index_packed(self.index_file, self._rows, self._names.blob, self._names.off,
                                                         self._n_lines, self.size, gz=self._st.gzindex, meta=meta)
        self._meta = meta
        return meta

    @property
    def phred(self):
        if self._phred:
            return self._phred
        return self._calc_composition()["phred"]

    @property
    def encoding_type(self):
        """possible quality encodings from the min / max quality (reference src/fastq.c:797-878)"""
        m = self._calc_composition()
        lo, hi = m["minqs"], m["maxqs"]
        if lo < 33 or hi > 126:
            return ["Unknown"]
        out = []
        if hi <= 73:
            out.append("Sanger Phred+33")
        if hi <= 74:
            out.append("Illumina 1.8+ Phred+33")
        if lo >= 59 and hi <= 104:
            out.append("Solexa Solexa+64")
        if lo >= 64 and hi <= 104:
            out.append("Illumina 1.3+ Phred+64")
        if lo >= 66 and hi <= 104:
            out.append("Illumina 1.5+ Phred+64")
        out.append("PacBio HiFi Phred+33")
        return out

    @property
    def gc_content(self):
        m = self._calc_composition()
        return float(np.float32(m["g"] + m["c"]) / np.float32(m["a"] + m["c"] + m["g"] + m["t"]) * np.float32(100))

    @property
    def composition(self):
        m = self._calc_composition()
        return {k.upper(): m[k] for k in ("a", "c", "g", "t", "n")}

    @property
    def maxlen(self):
        """meta.maxlen if the statistics were computed, else MAX(rlen) of the index (src/fastq.c:947-978)"""
        self.build_index()
        if self._meta is not None:
            return self._meta["maxlen"]
        return int(self._rows["rlen"].max()) if len(self._rows) else 0

    @property
    def minlen(self):
        self.build_index()
        if self._meta is not None:
            return self._meta["minlen"]
        return int(self._rows["rlen"].min()) if len(self._rows) else 0

    @property
    def maxqual(self):
        return self._calc_composition()["maxqs"]

    @property
    def minqual(self):
        return self._calc_composition()["minqs"]


class Read:
    """one FASTQ record (reference src/read.c)"""

    def __init__(self, fq, i):
        self._fq, self._i = fq, i
        self.id = i + 1
        self.name = fq._names.get(i)

    def __len__(self):
        return int(self._fq._rows["rlen"][self._i])

    def _fetch(self, flags=0, qual=False):
        fq = self._fq
        return fq._st.engine.read_one(fq._st.dfile, fq._drows, self._i, len(self), 1 if qual else 0, flags).decode("latin-1")

    @property
    def seq(self):
        return self._fetch()

    @property
    def qual(self):
        return self._fetch(qual=True)

    @property
    def quali(self):
        fq = self._fq                    # src/read.c:251-278: the phred offset if one is known, else 33
        p = fq._phred or (fq._meta["phred"] if fq._meta else 0) or 33
        return [c - p for c in self._fetch(qual=True).encode("latin-1")]

    @property
    def reverse(self):
        return self._fetch(_cabi.X_REVERSE)

    @property
    def complement(self):
        return self._fetch(_cabi.X_COMPLEMENT)

    @property
    def antisense(self):
        return self._fetch(_RC)

    @property
    def description(self):
        r = self._fq._rows[self._i]
        raw = bytes(self._fq._st.dfile.download(int(r["soff"]) - int(r["dlen"]) - 1, int(r["dlen"])))
        return raw.rstrip(b"\r").decode("latin-1")

    @property
    def raw(self):
        r = self._fq._rows[self._i]
        a = int(r["soff"]) - int(r["dlen"]) - 1
        end = min(int(r["qoff"]) + int(r["rlen"]) + 2, self._fq._st.dfile.size)
        raw = bytes(self._fq._st.dfile.download(a, end - a))
        k = raw.find(b"\n", int(r["qoff"]) - a)
        return raw[:k + 1 if k >= 0 else len(raw)].decode("latin-1")

    def __str__(self):
        return self.seq

    def __repr__(self):
        return "<Read> %s with length of %d" % (self.name, len(self))
