"""Layouts and helpers for the sharded index build tests (test_shard_scale_cpu.py, test_shard_scale_gpu.py).

A sharded build cuts one file into byte ranges that start at a line (FASTQ) or a header line (FASTA).  Every rank
stages its range through the 16 MiB pinned-piece ring (fxg_file_from_path_range) and runs fxg_scan_begin: mark,
prefix, and edge_kernel, which finds the shard's first three lines.  The ranks all-gather their 128-byte
fxg_shard_info, then run fxg_scan_finish.  For FASTQ, fastq_stitch_kernel completes a shard's last read from the
edge lines of later shards.

Each layout below says which cut it aims at (`aims`), and test_shard_scale_cpu.py checks on the bytes that the cut
is there.  Expected values never come from the GPU: they come from the whole-file oracle or plain Python.
"""
import functools
import os

import numpy as np

REGION = 2048                       # bytes per mark warp, and the granule of edge_kernel's region loop
EDGE_GROUP = 32                     # regions per step of edge_kernel's region loop
PS_BLOCK_BYTES = 4096 * REGION      # one prefix block (PS_BLOCK regions): 8 MiB
RING_PIECE = 16 << 20               # piece of stage_path_range's pinned ring
RING_SLOTS = 32
PREAD_WINDOW = 1 << 20              # window of fxg_split_point_path
SPLIT_STEP = 256 * 16               # bytes per step of split_point_kernel
MiB = 1 << 20

_ACGT = np.frombuffer(b"ACGT", np.uint8)


# ---- plain Python on the bytes ----------------------------------------------------------------------------
def lines(data):
    """[(start, length without the '\\n')] of every line, an unterminated last line included"""
    out, pos, n = [], 0, len(data)
    while pos < n:
        k = data.find(b"\n", pos)
        if k < 0:
            out.append((pos, n - pos))
            break
        out.append((pos, k - pos))
        pos = k + 1
    return out


def n_lines(data):
    """lines of a buffer as the scan counts them: every '\\n', plus one if the last line has none"""
    return data.count(b"\n") + (1 if data and not data.endswith(b"\n") else 0)


def line_index(data, off):
    """global index of the line that starts at `off`"""
    assert off == 0 or data[off - 1:off] == b"\n", off
    return data.count(b"\n", 0, off)


def edge_lines(shard, base):
    """(edge_n, edge_off[3], edge_len[3]) of a shard: its first three lines, a trailing '\\r' not counted"""
    ls = lines(shard)[:3]
    off, ln = [0, 0, 0], [0, 0, 0]
    for j, (s, L) in enumerate(ls):
        off[j] = base + s
        ln[j] = L - (1 if L > 0 and shard[s + L - 1:s + L] == b"\r" else 0)
    return len(ls), off, ln


def shard_info(shard, base, mode):
    """the fxg_shard_info fields edge_kernel writes, from the shard's bytes"""
    en, eo, el = edge_lines(shard, base)
    return {"n_rows": sum(1 for s, _ in lines(shard) if shard[s:s + 1] == b">") if mode == 0 else 0,
            "n_lines": n_lines(shard), "bytes": len(shard), "base_offset": base,
            "end_position": len(shard) + (1 if shard and not shard.endswith(b"\n") else 0),
            "edge_n": en, "edge_off": eo, "edge_len": el}


def fasta_lead(shard):
    """(lines, bytes) before the shard's first header line; the whole shard if it has none"""
    for i, (s, _) in enumerate(lines(shard)):
        if shard[s:s + 1] == b">":
            return i, s
    return n_lines(shard), len(shard)


def header_starts(data):
    """offsets of every FASTA header line"""
    return [s for s, _ in lines(data) if data[s:s + 1] == b">"]


def line_starts(data):
    return [s for s, _ in lines(data)]


# ---- layouts ----------------------------------------------------------------------------------------------
class Layout:
    """one file, the format, the cuts it is built around and what each cut aims at.

    cuts: inner cut offsets in order (repeats give empty shards); shard r is [pts[r], pts[r + 1]) with
    pts = [0] + cuts + [len(data)].  aims: tuples checked by check_aim."""

    def __init__(self, name, fmt, data, cuts, aims, full_name=False):
        self.name, self.fmt, self.data, self.cuts, self.aims, self.full_name = name, fmt, data, list(cuts), aims, full_name

    @property
    def mode(self):
        return 0 if self.fmt == "fasta" else 1

    @property
    def pts(self):
        return [0] + self.cuts + [len(self.data)]

    def shard(self, r):
        p = self.pts
        return self.data[p[r]:p[r + 1]]

    def write(self, directory):
        path = os.path.join(directory, self.name + (".fa" if self.fmt == "fasta" else ".fq"))
        if not os.path.exists(path):
            with open(path, "wb") as f:
                f.write(self.data)
        return path


def check_aim(lay, aim):
    """True if the layout's bytes hold what `aim` states:
      ("phase", r, p)        shard r starts on a line whose global index is p mod 4
      ("header", r)          shard r starts with a header line
      ("nl", r, j, x)        the j-th newline of shard r is at byte x of the shard
      ("edge_regions", r, m) the last of shard r's first three newlines lies in region m or later
      ("lines", r, k)        shard r holds k lines
      ("empty", r)           shard r is empty
      ("no_eol_end", tail)   the file ends without '\\n'; its last bytes are `tail`
      ("crlf",)              every line of the file ends in '\\r\\n' (an unterminated last line aside)
      ("lead", k)            the file's first header line starts at byte k > 0
      ("blocks", r, k)       shard r spans at least k prefix blocks (its regions, virtual newline included)
      ("len", r, k)          shard r is k bytes long
      ("record_over_block",) a record (FASTA) or read line (FASTQ) is longer than a prefix block
      ("general", r)         shard r has a region holding more than 128 newlines"""
    kind, d, pts = aim[0], lay.data, lay.pts
    if kind == "phase":
        return pts[aim[1]] < len(d) and line_index(d, pts[aim[1]]) % 4 == aim[2]
    if kind == "header":
        return lay.shard(aim[1])[:1] == b">"
    if kind == "nl":
        nl = [i for i, c in enumerate(lay.shard(aim[1])[:aim[3] + 1]) if c == 10]
        return len(nl) > aim[2] and nl[aim[2]] == aim[3]
    if kind == "edge_regions":
        s = lay.shard(aim[1])
        ls = lines(s)
        s3, l3 = ls[min(2, len(ls) - 1)]
        return (s3 + l3) // REGION >= aim[2]
    if kind == "lines":
        return n_lines(lay.shard(aim[1])) == aim[2]
    if kind == "empty":
        return len(lay.shard(aim[1])) == 0
    if kind == "no_eol_end":
        return not d.endswith(b"\n") and d.endswith(aim[1])
    if kind == "crlf":
        ls = lines(d)
        return all(d[s + L - 1:s + L] == b"\r" for s, L in ls[:-1]) and d.count(b"\n") == d.count(b"\r\n")
    if kind == "lead":
        hs = header_starts(d)
        return bool(hs) and hs[0] == aim[1] > 0
    if kind == "blocks":
        nreg = (len(lay.shard(aim[1])) + 1 + REGION - 1) // REGION
        return (nreg + 4095) // 4096 >= aim[2]
    if kind == "len":
        return len(lay.shard(aim[1])) == aim[2]
    if kind == "record_over_block":
        if lay.mode == 0:
            hs = header_starts(d) + [len(d)]
            return max(b - a for a, b in zip(hs, hs[1:])) > PS_BLOCK_BYTES
        return max(L for _, L in lines(d)) > PS_BLOCK_BYTES
    if kind == "general":
        a = np.frombuffer(lay.shard(aim[1]), np.uint8)
        nreg = (a.size + REGION - 1) // REGION
        cnt = np.bincount(np.flatnonzero(a == 10) // REGION, minlength=nreg)
        return bool((cnt > 128).any())
    raise ValueError(kind)


def _seq(rng, n):
    return _ACGT[rng.integers(0, 4, size=n)].tobytes()


def _qual(rng, n):
    return rng.integers(33, 75, size=n).astype(np.uint8).tobytes()        # may hold '@', '+' and '>'


def _read(name, seq, qual, eol):
    return b"@" + name + eol + seq + eol + b"+" + eol + qual + eol


# read lengths of the long-read layouts: the line that ends at byte 2047 / 2048 of a region, the one whose newline is
# in region 31 (the last of edge_kernel's first group of 32), 70 kB (past the first group), 131 kB (past 64 regions)
# and 2048 k +- 1
LONG_READS = (2046, 2047, 2048, 64000, 70000, 131000, 2048 * 20 - 1, 2048 * 20, 2048 * 20 + 1)


def fastq_long(eol, phase, seed=1):
    """short reads with the LONG_READS among them; every long read is cut at its line `phase` (0 name, 1 sequence,
    2 '+', 3 quality), so the shard that starts there begins with that line"""
    rng = np.random.default_rng(seed + 10 * phase + (5 if eol == b"\r\n" else 0))
    parts, cuts, aims, pos = [], [], [], 0
    for i, L in enumerate((150, 90) + sum(((L, 120 + i) for i, L in enumerate(LONG_READS)), ()) + (80,)):
        name = b"r%d len=%d" % (i, L)
        rec = _read(name, _seq(rng, L), _qual(rng, L), eol)
        if L in LONG_READS:
            seq_at = 1 + len(name) + len(eol)
            plus_at = seq_at + L + len(eol)
            cuts.append(pos + (0, seq_at, plus_at, plus_at + 1 + len(eol))[phase])
            r = len(cuts)
            aims.append(("phase", r, phase))
            if phase == 1:
                # the sequence line is the shard's first line: its newline is byte L (+1 for the '\r') of the shard,
                # and the quality line's newline lies about 2 L bytes in
                aims.append(("nl", r, 0, L + len(eol) - 1))
                aims.append(("edge_regions", r, (2 * L) // REGION))
            if phase == 3:
                aims.append(("nl", r, 0, L + len(eol) - 1))
        parts.append(rec)
        pos += len(rec)
    data = b"".join(parts)
    if eol == b"\r\n":
        aims.append(("crlf",))
    return Layout("fq_long_%s_p%d" % ("crlf" if eol == b"\r\n" else "lf", phase), "fastq", data, cuts, aims)


def fastq_tiny_shards(eol, two_line):
    """the last read (70 kB) spans three or four shards of one or two lines; the file ends inside its quality line
    without '\\n' (CRLF: the last byte is the '\\r')"""
    rng = np.random.default_rng(7 + (1 if two_line else 0) + (2 if eol == b"\r\n" else 0))
    head = b"".join(_read(b"a%d" % i, _seq(rng, 100 + i), _qual(rng, 100 + i), eol) for i in range(6))
    L = 70000
    name, seq, qual = b"last x", _seq(rng, L), _qual(rng, L)
    ends = [len(head)]
    for ln in (b"@" + name, seq, b"+"):
        ends.append(ends[-1] + len(ln) + len(eol))
    tail = qual + (b"\r" if eol == b"\r\n" else b"")
    data = head + b"@" + name + eol + seq + eol + b"+" + eol + tail
    if two_line:
        cuts = [ends[0], ends[1], ends[3]]                 # [name], [seq, +], [qual]
        aims = [("lines", 1, 1), ("lines", 2, 2), ("lines", 3, 1), ("phase", 1, 0), ("phase", 2, 1), ("phase", 3, 3)]
    else:
        cuts = [ends[0], ends[1], ends[2], ends[3]]        # one line each
        aims = [("lines", r, 1) for r in (1, 2, 3, 4)] + [("phase", r, r - 1) for r in (1, 2, 3, 4)]
    aims.append(("no_eol_end", tail[-8:]))
    if eol == b"\r\n":
        aims.append(("crlf",))
    return Layout("fq_tiny_%s_%s" % ("two" if two_line else "one", "crlf" if eol == b"\r\n" else "lf"), "fastq",
                  data, cuts, aims)


def fastq_partial_tail_cr():
    """CRLF reads ending in a partial record whose sequence line is unterminated and ends in '\\r'; that line is a
    shard of its own"""
    rng = np.random.default_rng(31)
    eol = b"\r\n"
    head = b"".join(_read(b"p%d d" % i, _seq(rng, 3000 + i), _qual(rng, 3000 + i), eol) for i in range(5))
    data = head + b"@tail x" + eol + _seq(rng, 2500) + b"\r"
    cuts = [len(head), len(head) + len(b"@tail x") + 2]
    return Layout("fq_partial_tail_cr", "fastq", data, cuts,
                  [("phase", 1, 0), ("phase", 2, 1), ("lines", 2, 1), ("no_eol_end", b"\r"), ("crlf",)])


def fastq_few_reads():
    """three reads and sixteen shards: most shards are empty"""
    data = b"@a\nAC\n+\nII\n@b x\nACGT\n+\nIIII\n@c\nA\n+\nI\n"
    ls = line_starts(data)
    cuts = [ls[1], ls[1], ls[5], ls[5], len(data), len(data)]
    return Layout("fq_few_reads", "fastq", data, cuts,
                  [("empty", 1), ("empty", 3), ("empty", 5), ("empty", 6), ("lines", 2, 4), ("phase", 2, 1),
                   ("phase", 4, 1)])


def fastq_read_over_block():
    """a 9 MiB read between short ones: the shards that start at its sequence and quality lines run through more
    than one prefix block before their first newline"""
    rng = np.random.default_rng(41)
    L = 9 * MiB
    head = b"".join(_read(b"s%d" % i, _seq(rng, 150), _qual(rng, 150), b"\n") for i in range(20))
    big = _read(b"big", _seq(rng, L), _qual(rng, L), b"\n")
    tail = b"".join(_read(b"t%d" % i, _seq(rng, 150), _qual(rng, 150), b"\n") for i in range(20))
    s = len(head) + len(b"@big\n")
    data = head + big + tail
    cuts = [s, s + L + 1 + 2]
    return Layout("fq_read_over_block", "fastq", data, cuts,
                  [("phase", 1, 1), ("phase", 2, 3), ("record_over_block",), ("blocks", 1, 2), ("nl", 1, 0, L)])


def _fastq_fill(rng, nbytes, eol, tag):
    """FASTQ reads of exactly nbytes: 150 bp reads made in one numpy pass, then one read padded to fit"""
    e = np.frombuffer(eol, np.uint8)
    L = 150
    rec = 1 + 10 + len(eol) + L + len(eol) + 1 + len(eol) + L + len(eol)
    n = max(0, (nbytes - 64) // rec)
    rows = np.empty((n, rec), np.uint8)
    rows[:, 0] = ord("@")
    idx = np.arange(n, dtype=np.int64)
    rows[:, 1] = ord(tag)
    for k in range(9):
        rows[:, 10 - k] = 48 + (idx // 10 ** k) % 10
    c = 11
    rows[:, c:c + len(eol)] = e; c += len(eol)
    rows[:, c:c + L] = _ACGT[rng.integers(0, 4, size=(n, L))]; c += L
    rows[:, c:c + len(eol)] = e; c += len(eol)
    rows[:, c] = ord("+"); c += 1
    rows[:, c:c + len(eol)] = e; c += len(eol)
    rows[:, c:c + L] = rng.integers(35, 75, size=(n, L)); c += L
    rows[:, c:c + len(eol)] = e
    rest = nbytes - n * rec
    fill_len = 1
    pad = rest - (1 + len(eol) + fill_len + len(eol) + 1 + len(eol) + fill_len + len(eol))
    assert pad >= 1
    filler = _read(b"f" * pad, b"A", b"I", eol)
    return rows.tobytes() + filler


def _fasta_fill(rng, nbytes, eol, tag, width=80, per_record=100):
    """FASTA records of exactly nbytes: records of `per_record` full lines in one numpy pass, then one record padded
    to fit"""
    e = np.frombuffer(eol, np.uint8)
    hdr = 1 + 10 + 2 + len(eol)                          # '>' tag + 9 digits + ' d' + eol
    line = width + len(eol)
    rec = hdr + per_record * line
    n = max(0, (nbytes - 256) // rec)
    rows = np.empty((n, rec), np.uint8)
    rows[:, 0] = ord(">")
    rows[:, 1] = ord(tag)
    idx = np.arange(n, dtype=np.int64)
    for k in range(9):
        rows[:, 10 - k] = 48 + (idx // 10 ** k) % 10
    rows[:, 11] = ord(" ")
    rows[:, 12] = ord("d")
    rows[:, 13:13 + len(eol)] = e
    body = rows[:, hdr:].reshape(n, per_record, line)
    body[:, :, :width] = _ACGT[rng.integers(0, 4, size=(n, per_record, width))]
    body[:, :, width:] = e
    rest = nbytes - n * rec
    pad = rest - (1 + len(eol) + 10 + len(eol))
    assert pad >= 1
    filler = b">" + b"g" * pad + eol + b"ACGTACGTAC" + eol
    return rows.tobytes() + filler


# shard lengths of the block-scale layouts: k * 8 MiB +- {0, 1, 2047, 2048}
BLOCK_SHARDS = (2 * PS_BLOCK_BYTES + 1, PS_BLOCK_BYTES - 2048, 2 * PS_BLOCK_BYTES, PS_BLOCK_BYTES + 2047,
                PS_BLOCK_BYTES - 1, 2 * PS_BLOCK_BYTES - 1)


def blocks_layout(fmt):
    """a 60-80 MB file whose cuts sit at k * 8 MiB +- {0, 1, 2047, 2048}: shards of several prefix blocks, and
    shards whose last block holds one region (or none beyond the virtual newline)"""
    rng = np.random.default_rng(61 if fmt == "fastq" else 62)
    eol = b"\n" if fmt == "fastq" else b"\r\n"
    fill = _fastq_fill if fmt == "fastq" else _fasta_fill
    parts = [fill(rng, L, eol, chr(ord("a") + i)) for i, L in enumerate(BLOCK_SHARDS)]
    parts.append(fill(rng, 3 * MiB + 777, eol, "z"))
    cuts = list(np.cumsum([len(p) for p in parts[:-1]]))
    cuts = [int(c) for c in cuts]
    data = b"".join(parts)
    aims = [("len", r, L) for r, L in enumerate(BLOCK_SHARDS)] + [("blocks", 0, 3), ("blocks", 2, 3), ("blocks", 5, 2)]
    aims += [("phase", r, 0) if fmt == "fastq" else ("header", r) for r in range(1, len(cuts) + 1)]
    if fmt == "fasta":
        aims.append(("crlf",))
    return Layout("%s_blocks" % fmt, fmt, data, cuts, aims)


def fasta_records(rng, n, eol, width, name=b"s", desc=True, min_len=0, max_len=3000):
    out = []
    for i in range(n):
        L = int(rng.integers(min_len, max_len + 1))
        seq = _seq(rng, L)
        hdr = b">" + name + b"%d" % i + (b" desc %d\tx" % i if desc and i % 2 else b"")
        out.append(hdr + eol + b"".join(seq[k:k + width] + eol for k in range(0, L, width)))
    return out


def _fasta_cut_layout(name, recs, cut_records, aims=(), lead=b"", full_name=False):
    data = lead + b"".join(recs)
    starts = np.cumsum([len(lead)] + [len(r) for r in recs])[:-1]
    cuts = [int(starts[i]) for i in cut_records]
    aims = list(aims) + [("header", r) for r in range(1, len(cuts) + 1) if cuts[r - 1] < len(data)]
    return Layout(name, "fasta", data, cuts, aims, full_name=full_name)


def fasta_crlf():
    rng = np.random.default_rng(71)
    recs = fasta_records(rng, 40, b"\r\n", 60)
    return _fasta_cut_layout("fa_crlf", recs, [3, 4, 17, 30, 39], [("crlf",)])


def fasta_general():
    """short lines (7 and 14 bytes) put more than 128 newlines in a region: the rows pass's general path"""
    rng = np.random.default_rng(72)
    recs = fasta_records(rng, 12, b"\n", 7, min_len=2000, max_len=9000) + \
        fasta_records(rng, 12, b"\n", 14, name=b"w", min_len=2000, max_len=9000)
    return _fasta_cut_layout("fa_general", recs, [2, 9, 13, 20], [("general", 1), ("general", 3)])


def fasta_with_lead(first_cut_at_header):
    """the file starts with lines before any header: rank 0's lead part (alone in shard 0, or with records)"""
    rng = np.random.default_rng(73)
    lead = b"junk line\nmore junk\r\n\n;comment\n"
    recs = fasta_records(rng, 20, b"\n", 70)
    cut = [0, 6, 11] if first_cut_at_header else [5, 12]
    aims = [("lead", len(lead))] + ([("len", 0, len(lead))] if first_cut_at_header else [])
    return _fasta_cut_layout("fa_lead_%s" % ("alone" if first_cut_at_header else "with_records"), recs, cut, aims,
                             lead=lead)


def fasta_full_name():
    rng = np.random.default_rng(74)
    recs = fasta_records(rng, 30, b"\n", 80)
    return _fasta_cut_layout("fa_full_name", recs, [1, 10, 29], full_name=True)


def fasta_few_records():
    """three records and sixteen shards: most shards are empty"""
    data = b">a\nACGT\n>b x\nGG\nTT\n>c\nA\n"
    hs = header_starts(data)
    cuts = [hs[1], hs[1], hs[2], hs[2], len(data), len(data)]
    return Layout("fa_few_records", "fasta", data, cuts,
                  [("empty", 1), ("empty", 3), ("empty", 5), ("empty", 6), ("header", 2), ("header", 4)])


def fasta_record_over_block():
    """a 9 MiB record between small ones, cut at its header and at the next: its shard spans two prefix blocks"""
    rng = np.random.default_rng(75)
    small = fasta_records(rng, 8, b"\n", 60)
    big = fasta_records(rng, 1, b"\n", 80, name=b"big", min_len=9 * MiB, max_len=9 * MiB)
    recs = small[:4] + big + small[4:]
    return _fasta_cut_layout("fa_record_over_block", recs, [4, 5], [("record_over_block",), ("blocks", 1, 2)])


SMALL_LAYOUTS = ([functools.partial(fastq_long, eol, p) for eol in (b"\n", b"\r\n") for p in range(4)] +
                 [functools.partial(fastq_tiny_shards, eol, two) for eol in (b"\n", b"\r\n") for two in (False, True)] +
                 [fastq_partial_tail_cr, fastq_few_reads, fasta_crlf, fasta_general,
                  functools.partial(fasta_with_lead, True), functools.partial(fasta_with_lead, False), fasta_full_name,
                  fasta_few_records])
BIG_LAYOUTS = [fastq_read_over_block, fasta_record_over_block, functools.partial(blocks_layout, "fastq"),
               functools.partial(blocks_layout, "fasta")]


def _builder_name(b):
    if isinstance(b, functools.partial):
        return b.func.__name__ + "_" + "_".join(x.decode().replace("\n", "lf").replace("\r", "cr")
                                               if isinstance(x, bytes) else str(x) for x in b.args)
    return b.__name__


@functools.lru_cache(maxsize=None)
def _layout(i):
    lay = (SMALL_LAYOUTS + BIG_LAYOUTS)[i]()
    lay.id = layout_ids()[i]
    return lay


def layout_ids():
    return [_builder_name(b) for b in SMALL_LAYOUTS + BIG_LAYOUTS]


def layout(name):
    return _layout(layout_ids().index(name))


# ---- the split-point windows ----------------------------------------------------------------------------
def split_window_file():
    """FASTA with ~3.2 MiB of 60-column sequence between two headers, then a 3 MiB line without a newline, a header
    and a few records -> (data, x) where data[x:x + 2] == b'\\n>' is the first header start after the first
    record.  fxg_split_point_path reads 1 MiB windows from from - 1; from = x + 2 - k MiB puts that '\\n' on the
    last byte of window k - 1 and the '>' on the first byte of window k."""
    rng = np.random.default_rng(81)
    first = b">one\n" + b"".join(_seq(rng, 60) + b"\n" for _ in range(55000))
    second = b">two x\n" + _seq(rng, 3 * MiB) + b"\n"
    rest = b"".join(fasta_records(rng, 5, b"\n", 60, name=b"r"))
    data = first + second + rest
    return data, len(first) - 1


def split_froms(x, n):
    """`from` values around the pread windows for an anchor '\\n' at x: the '\\n' as the last byte of window
    k - 1 (k = 1..3), one byte either side, plus the ends of the file"""
    out = {0, 1, n - 1, n, n + 5}
    for k in (1, 2, 3):
        for d in (-2, -1, 0, 1, 2):
            f = x + 2 - k * PREAD_WINDOW + d
            if f >= 0:
                out.add(f)
    return sorted(out)


# ---- the loop-back emulation of N ranks on one GPU --------------------------------------------------------
def emulate(engs, pts, mode, path=None, data=None, stager=None, C=0, full_name=False):
    """The sharded build of N = len(pts) - 1 ranks, run on one GPU: rank r's own Engine engs[r] runs
    fxg_scan_begin on its range [pts[r], pts[r + 1]), the all-gather of the 128-byte fxg_shard_info is done by
    hand (download, concatenate, upload), then every rank runs fxg_scan_finish and gathers its names the way
    shard.build_index_sharded does.  Buffers come from stage_path_range(path, a, b) (by `stager`, an Engine whose
    one pinned ring serves every rank) or, with data, from stage_bytes.  C is added to every rank's base_offset.
    -> list per rank of dict(rows, stats, infos, names, name_off, info_own)"""
    from pyfastx_b200 import _cabi
    world = len(pts) - 1
    assert len(engs) >= world
    files = []
    for r in range(world):
        a, b = pts[r], pts[r + 1]
        files.append(stager.stage_path_range(path, a, b) if data is None else engs[r].stage_bytes(data[a:b]))
    slots = [engs[r].dev_alloc(_cabi.SHARD_INFO.itemsize) for r in range(world)]
    infos = np.zeros(world, dtype=_cabi.SHARD_INFO)
    out = []
    try:
        for r in range(world):
            engs[r].scan_begin(files[r], mode, base_offset=pts[r] + C, full_name=full_name, d_info=slots[r].devptr)
        for r in range(world):
            engs[r].sync()
            one = np.zeros(1, dtype=_cabi.SHARD_INFO)
            _cabi.check(_cabi.lib().fxg_rows_download(engs[r].ctx, slots[r].devptr, 1, _cabi.SHARD_INFO.itemsize,
                                                      one.ctypes.data))
            infos[r] = one[0]
        dt = _cabi.FASTA_ROW if mode == 0 else _cabi.FASTQ_ROW
        for r in range(world):
            d_all = engs[r].upload_rows(infos)
            try:
                rows, st, got = engs[r].scan_finish(d_all.devptr, world, r, dt)
            finally:
                d_all.free()
            a = pts[r] + C
            if mode == 0:
                noff = rows["boff"] - rows["elen"].astype(np.int64) - rows["dlen"] - a
            else:
                noff = rows["soff"] - rows["dlen"] - a
            if len(rows):
                names, name_off = engs[r].gather_ranges(files[r], noff, rows["nlen"].astype(np.int64))
            else:
                names, name_off = np.zeros(0, np.uint8), np.zeros(1, np.int64)
            out.append({"rows": rows, "stats": st, "infos": got, "names": names, "name_off": name_off})
    finally:
        for r in range(world):
            files[r].free()
            slots[r].free()
    return out, infos


def split_names(names, name_off):
    return [names[name_off[i]:name_off[i + 1]].tobytes() for i in range(len(name_off) - 1)]


def merged_index(res):
    """rank 0's merge as build_index_sharded does it: rows concatenated, names packed with rebased offsets"""
    rows = np.concatenate([p["rows"] for p in res])
    blob = np.concatenate([np.asarray(p["names"], np.uint8) for p in res])
    offs, acc = [], 0
    for p in res:
        offs.append(np.asarray(p["name_off"][:-1], np.int64) + acc)
        acc += int(p["name_off"][-1])
    return rows, blob, np.concatenate(offs + [np.array([acc], np.int64)])
