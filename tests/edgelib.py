"""Byte-level FASTA / FASTQ edge patterns placed exactly on the cut points of the GPU scan and of the kernels after it.

The scan splits a file into 2 KiB regions (one warp each in mark), prefixes the region counts in blocks of 4096 regions
(8 MiB), and the FASTQ records kernel gives each warp 8 regions (16 KiB).  A look-back or look-ahead that is wrong only
when a '\\r', a blank line or a header start falls on one of those edges is invisible to inputs where the edge lands on
an ordinary byte.  This module builds inputs where it does not:

- CATALOGUE: short byte patterns (CRLF split either side, blank lines, '>' as the first byte of a region, the name cut
  at header bytes 63 / 64 / 65, NUL and bytes >= 0x80 in a line, '@' / '+' starting a quality line, ...), each with
  one named anchor byte.  An anchor equal to the pattern's length stands for the end of the file.
- place(pattern, boundary, shift, dense): filler records, one adjustable line (or FASTQ record) sized so that the anchor
  lands at boundary + shift exactly, the pattern, then more filler.  dense = 1 packs the lines around the anchor so
  that its region has 33..128 newlines (mark's general path), dense = 2 so that it has more than 128 (the counts-only
  path, the rows kernels re-read the bytes).
- place_sites(pattern, sites, dense): the same with one copy of the pattern per (boundary, shift) site, far enough
  apart that the sites do not interact; the GPU tests check a whole file at once.

Also here: the plain numpy restatements of full-index composition and of the reference's FASTQ statistics loop
(src/fastq.c:715-752), and region_view, the rule mark applies to the region holding an anchor."""
import functools
import itertools

import numpy as np

REGION = 2048                     # bytes per mark warp (fxg_scan.cu REGION)
LF_MAX = 3                        # line facts a region settled by mark can hold
SEGCAP = 128                      # newline-list entries per region; more: the counts-only path
NAME_SCAN = 64                    # header bytes mark searches for the name cut
PS_BLOCK = 4096                   # regions per prefix block
BLOCK_BYTES = PS_BLOCK * REGION   # 8 MiB
WINDOW = 8 * REGION               # FASTQ records kernel: bytes per warp
SHIFTS = tuple(range(-3, 4))
PACK = REGION + 512               # dense packing reaches this far on both sides of an anchor

S = b"ACGTTGCAACGGATCCTAGCATGCAAGTCCGATTACGAGCTTGACCATGGTACAGTCAGA"   # 60 bytes
assert len(S) == 60
SQ = (S * 3)[:150]
QUAL = bytes(33 + (i * 7) % 41 for i in range(150))                      # '!'..'I', no '@' or '+' at position 0


class Pattern:
    def __init__(self, name, kind, pre, post, eol=b"\n", tail=False):
        self.name, self.kind, self.eol, self.tail = name, kind, eol, tail
        self.data = pre + post
        self.anchor = len(pre)                 # index of the anchor byte (len(data): the end of the file)

    def __repr__(self):
        return "Pattern(%s)" % self.name


CRLF = b"\r\n"


def _fa(name, pre, post, eol=b"\n", tail=False):
    return Pattern(name, "fasta", pre, post, eol, tail)


def _fq(name, pre, post, eol=b"\n", tail=False):
    return Pattern(name, "fastq", pre, post, eol, tail)


FASTA = [
    _fa("crlf_header_cr", b">h x", CRLF + S + CRLF, CRLF),                      # '\r' of a header's CRLF at the anchor
    _fa("crlf_header_lf", b">h x\r", b"\n" + S + CRLF, CRLF),                   # ... its '\n'
    _fa("crlf_seq_cr", S[:37], CRLF + S + CRLF, CRLF),
    _fa("crlf_seq_lf", S[:37] + b"\r", b"\n" + S + CRLF, CRLF),
    _fa("cr_cr_lf", S[:20] + b"\r", b"\r\n" + S + CRLF, CRLF),
    _fa("lone_cr", S[:30], b"\r" + S[:20] + b"\n" + S + b"\n"),
    _fa("blank_lf", b"", b"\n" + S + b"\n"),
    _fa("blank_crlf_cr", b"", CRLF + S + CRLF, CRLF),
    _fa("blank_crlf_lf", b"\r", b"\n" + S + CRLF, CRLF),
    _fa("header_start", b"", b">gt desc\n" + S + b"\n"),                        # '>' at the anchor
    _fa("header_start_crlf", b"", b">gt desc\r\n" + S + CRLF, CRLF),
    _fa("gt_in_line", S[:25], b">" + S[:30] + b"\n"),
    _fa("name_space_63", b">" + b"n" * 63, b" d e\n" + S + b"\n"),              # first ' ' / '\t' at name byte 63..65
    _fa("name_space_64", b">" + b"n" * 64, b" d e\n" + S + b"\n"),
    _fa("name_space_65", b">" + b"n" * 65, b" d e\n" + S + b"\n"),
    _fa("name_tab_63", b">" + b"n" * 63, b"\td e\n" + S + b"\n"),
    _fa("name_tab_64", b">" + b"n" * 64, b"\td e\n" + S + b"\n"),
    _fa("name_tab_65", b">" + b"n" * 65, b"\td e\r\n" + S + CRLF, CRLF),
    _fa("header_crossing", b">cross" + b"y" * 20, b"z" * 20 + b" d\n" + S + b"\n"),
    _fa("two_headers", b">a1\n", b">a2 x\n" + S + b"\n"),
    _fa("lone_gt", b"", b">\n" + S + b"\n"),
    _fa("first_line_shorter", b">fs\n", S[:17] + b"\n" + S + b"\n" + S + b"\n"),
    _fa("last_line_longer", b">ll\n" + S + b"\n" + S + b"\n", S + S[:13] + b"\n"),
    _fa("length_change", S + b"\n", S[:45] + b"\n" + S[:45] + b"\n"),
    _fa("space_tab", S[:20], b" " + S[:10] + b"\t" + S[:10] + b"\n" + S + b"\n"),
    _fa("nul", S[:20], b"\x00" + S[:10] + b"\n" + S + b"\n"),
    _fa("high_bytes", S[:20], b"\x80\xff" + S[:10] + b"\xc1\n" + S + b"\n"),
    _fa("mixed_lf_crlf", b">mx\n" + S + b"\n" + S, b"\r\n" + S + b"\n" + S + b"\r\n"),
    # the file ends with the pattern
    _fa("header_at_eof", b"", b">eof x", tail=True),
    _fa("header_at_eof_nl", b"", b">eof x\n", tail=True),
    _fa("no_newline_at_end", S[:50], b"", tail=True),                              # n = boundary + shift
    _fa("no_newline_at_end_crlf", S[:50], b"", CRLF, tail=True),
]

FASTQ = [
    _fq("qual_starts_at", b"@q1\n" + SQ + b"\n+\n", b"@" + QUAL[1:] + b"\n"),
    _fq("qual_starts_plus", b"@q2\n" + SQ + b"\n+\n", b"+" + QUAL[1:] + b"\n"),
    _fq("crlf_split_name", b"@c1 x\r", b"\n" + SQ + b"\r\n+\r\n" + QUAL + CRLF, CRLF),
    _fq("crlf_split_seq", b"@c2 x\r\n" + SQ + b"\r", b"\n+\r\n" + QUAL + CRLF, CRLF),
    _fq("crlf_split_qual", b"@c3 x\r\n" + SQ + b"\r\n+\r\n" + QUAL + b"\r", b"\n", CRLF),
    _fq("plus_name", b"@p4 d\n" + SQ + b"\n", b"+p4 d\n" + QUAL + b"\n"),
    _fq("empty_read", b"@r\n", b"\n+\n\n"),
    _fq("window_crossing", b"@w\n" + SQ * 4, SQ * 4 + b"\n+\n" + QUAL * 8 + b"\n"),
    _fq("partial_tail", b"@pt x\nACGT\n+\n", b"", tail=True),
    _fq("no_newline_at_end", b"@nt\nACGT\n+\nIIII", b"", tail=True),
]

CATALOGUE = {p.kind + ":" + p.name: p for p in FASTA + FASTQ}

# a few patterns also go to the 8 MiB prefix-block edge
BLOCK_EDGE = ("fasta:header_start", "fasta:crlf_seq_lf", "fasta:blank_lf", "fastq:crlf_split_seq")
BLOCK_EDGE_DENSE = "fasta:header_start"          # ... this one also on the counts-only path (a prefix block's gblk flag)


# ---------------------------------------------------------------------------------------------
# filler and placement
# ---------------------------------------------------------------------------------------------
REC_LINES = (17, 40, 5, 33, 2, 26, 11)          # FASTA filler: sequence lines per record, cycled


class _Builder:
    """appends filler; width(pos) gives the line width (FASTA) or read length (FASTQ) at file position pos"""

    def __init__(self, kind, eol, dense):
        self.kind, self.eol, self.dense = kind, eol, dense
        self.out = bytearray()
        self.rec = 0
        self.left = 0                      # FASTA: sequence lines left in the current filler record (0: header next)
        self.packs = []                    # (lo, hi) ranges packed with short lines

    def width(self, pos):
        packed = any(lo <= pos < hi for lo, hi in self.packs)
        if self.kind == "fasta":
            return {0: 80, 1: 20, 2: 6}[self.dense] if packed else 80
        return {0: 150, 1: 40, 2: 4}[self.dense] if packed else 150

    def next_item(self):
        """bytes of the next filler item"""
        pos = len(self.out)
        w = self.width(pos)
        if self.kind == "fasta":
            if self.left == 0:
                return b">f%d d" % self.rec + self.eol
            return (S * 4)[(self.left * 7) % 60:][:w] + self.eol
        q = bytes(QUAL[(self.rec + i) % 150] for i in range(w))
        return b"@f%d" % self.rec + self.eol + SQ[:w] + self.eol + b"+" + self.eol + q + self.eol

    def push(self, item):
        self.out += item
        if self.kind == "fasta":
            if self.left == 0:
                self.left = REC_LINES[self.rec % len(REC_LINES)]
                self.rec += 1
            else:
                self.left -= 1
        else:
            self.rec += 1

    def fill_to(self, end):
        while len(self.out) < end:
            self.push(self.next_item())

    def adjust_to(self, target):
        """filler up to exactly `target`, the last item sized to end there"""
        minimum = len(self.eol) + 1 if self.kind == "fasta" else 4 * len(self.eol) + 12
        n0 = len(self.out)
        while True:
            item = self.next_item()
            if target - len(self.out) - len(item) < minimum:
                break
            self.push(item)
        need = target - len(self.out)
        assert need >= minimum and len(self.out) > n0, "sites too close (%d, %d)" % (n0, target)
        if self.kind == "fasta":        # one more sequence line of the current filler record
            self.out += (S * 8)[:need - len(self.eol)] + self.eol
            return
        e = len(self.eol)
        name = b"@f%d" % self.rec
        r = max(1, min(self.width(len(self.out)), (need - 4 * e - 1 - len(name)) // 2))
        pad = need - (len(name) + 4 * e + 1 + 2 * r)
        assert pad >= 0
        name += b"_" * pad
        self.out += name + self.eol + SQ[:r] + self.eol + b"+" + self.eol + QUAL[:r] + self.eol
        self.rec += 1

    def put_pattern(self, pat):
        self.out += pat.data
        if self.kind == "fasta":
            self.left = 0               # the filler after a pattern starts with a new record


def place_sites(pattern, sites, dense=0):
    """file bytes with `pattern` placed so that its anchor lands at boundary + shift for every (boundary, shift) of
    `sites` (increasing).  -> (data, anchor positions)"""
    b = _Builder(pattern.kind, pattern.eol, dense)
    start = (sites[0][0] + sites[0][1] - 3 * REGION) // (4 * WINDOW) * (4 * WINDOW)
    if start > 16 * WINDOW:                         # the plain filler before a far site is shared by every such file
        out, b.rec, b.left = _prefix(pattern.kind, pattern.eol, start)
        b.out = bytearray(out)
    if dense:
        b.packs = [(bd + sh - PACK, bd + sh + PACK) for bd, sh in sites]
    anchors = []
    for bd, sh in sites:
        at = bd + sh
        b.adjust_to(at - pattern.anchor)
        b.put_pattern(pattern)
        anchors.append(at)
    if not pattern.tail:
        b.fill_to(len(b.out) + (PACK if dense else 0) + 3000)
        if b.kind == "fasta" and b.left:            # end on a complete record
            while b.left:
                b.push(b.next_item())
    return bytes(b.out), anchors


@functools.lru_cache(maxsize=4)
def _prefix(kind, eol, upto):
    b = _Builder(kind, eol, 0)
    b.fill_to(upto)
    return bytes(b.out), b.rec, b.left


def place(pattern, boundary, shift, dense=0):
    """one site: -> file bytes with the anchor at boundary + shift"""
    return place_sites(pattern, [(boundary, shift)], dense)[0]


def small_file(pattern):
    """the pattern with one record (or read) of context on each side, without any placement"""
    e = pattern.eol
    if pattern.kind == "fasta":
        head, after = b">pre x" + e + S + e + S[:33] + e, b">post" + e + S + e
    else:
        head = b"@pre x" + e + SQ[:40] + e + b"+" + e + QUAL[:40] + e
        after = b"@post" + e + SQ[:20] + e + b"+" + e + QUAL[:20] + e
    return head + pattern.data + (b"" if pattern.tail else after)


def small_sites():
    """(boundary, shift) sites of one multi-site file: every shift at a 16 KiB window edge and at a region edge
    3 regions later, 32 KiB apart"""
    out = []
    for i, d in enumerate(SHIFTS):
        w = WINDOW * (2 * i + 1)
        out += [(w, d), (w + 3 * REGION, d)]
    return out


def dense_levels(pattern):
    return (0, 1, 2) if pattern.kind == "fasta" else (0, 2)


@functools.lru_cache(maxsize=None)
def layouts():
    """every placed input: key -> (pattern key, sites, dense).  Patterns that end the file get one file per shift at
    16384 * 2 (dense 0 and 2); the others one file per dense level with every small site; BLOCK_EDGE patterns
    also one file per shift at the 8 MiB prefix-block edge (dense 0, and dense 2 for BLOCK_EDGE_DENSE)."""
    out = {}
    for key, p in CATALOGUE.items():
        for dense in dense_levels(p):
            if p.tail:
                if dense == 1:
                    continue
                for bd, d in itertools.product((2 * WINDOW,), SHIFTS):
                    out["%s/%d%+d/d%d" % (key, bd, d, dense)] = (key, ((bd, d),), dense)
            else:
                out["%s/small/d%d" % (key, dense)] = (key, tuple(small_sites()), dense)
        if key in BLOCK_EDGE:
            for dense, d in itertools.product((0, 2) if key == BLOCK_EDGE_DENSE else (0,), SHIFTS):
                out["%s/8MiB%+d/d%d" % (key, d, dense)] = (key, ((BLOCK_BYTES, d),), dense)
    return out


@functools.lru_cache(maxsize=8)
def build(layout_key):
    """-> (data, anchors, pattern) of one layout"""
    key, sites, dense = layouts()[layout_key]
    p = CATALOGUE[key]
    data, anchors = place_sites(p, list(sites), dense)
    return data, anchors, p


# ---------------------------------------------------------------------------------------------
# the rule mark applies to the region holding an anchor
# ---------------------------------------------------------------------------------------------
def region_view(data, pos):
    """(newlines, line facts k >= 2, k of the line holding byte pos) of the region holding pos, by the rule of
    test_fasta_line_record_cpu.region_stats (a virtual newline at n when the file does not end in one); k is None when
    that line ends in a later region"""
    a = np.frombuffer(data, np.uint8)
    n = a.size
    r = min(pos, n) // REGION
    lo, hi = r * REGION, (r + 1) * REGION
    seg = a[lo:hi]
    ent = (lo + np.nonzero(seg == 10)[0]).tolist()
    if n and a[-1] != 10 and lo <= n < hi:
        ent.append(n)
    hdr = lambda e: e + 1 < n and a[e + 1] == ord(">")
    facts = 0
    for k in range(2, len(ent)):
        p, p1, p2 = ent[k], ent[k - 1], ent[k - 2]
        if hdr(p1) or hdr(p2) or p - p1 != p1 - p2:
            facts += 1
    k_at = next((k for k, e in enumerate(ent) if e >= pos), None)
    return len(ent), facts, k_at


def region_path(kind, nl, facts):
    """'dense' (counts only), 'general' (newline list) or, for FASTA, 'fast' (settled by mark)"""
    if nl > SEGCAP:
        return "dense"
    return "general" if kind == "fastq" or nl > 32 or facts > LF_MAX else "fast"


# ---------------------------------------------------------------------------------------------
# numpy restatements
# ---------------------------------------------------------------------------------------------
def composition(data, rows):
    """full-index composition: per record, the bytes < 128 of [boff, boff + blen) other than '\\n' ->
    ([(seqid, byte, count)] in (seqid, byte) order, whole-file totals[128])"""
    a = np.frombuffer(data, np.uint8)
    n = len(rows)
    if n == 0:
        return [], np.zeros(128, np.int64)
    boff = rows["boff"].astype(np.int64)
    end = np.minimum(boff + rows["blen"].astype(np.int64), a.size)
    ln = np.maximum(end - boff, 0)
    rid = np.repeat(np.arange(n), ln)
    pos = np.arange(ln.sum()) - np.repeat(np.cumsum(ln) - ln, ln) + np.repeat(boff, ln)
    b = a[pos]
    keep = (b != 10) & (b < 128)
    h = np.bincount(rid[keep] * 128 + b[keep], minlength=n * 128).reshape(n, 128)
    nz = np.nonzero(h)
    return [(int(i) + 1, int(c), int(h[i, c])) for i, c in zip(*nz)], h.sum(axis=0)


def fastq_stats(data):
    """the reference's statistics loop (src/fastq.c:715-752) over the lines of the whole file: base counts of every
    second line of four, and of every fourth its length and quality range, where each '\\r' met shortens the line by
    one and is skipped -> dict like Engine.fastq_stats"""
    lines = data.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    a = c = g = t = nn = 0
    mn, mx, maxlen, minlen = 104, 33, 0, 10000000000
    for k, ln in enumerate(lines):
        if k % 4 == 1:
            a += ln.count(b"A"); c += ln.count(b"C"); g += ln.count(b"G"); t += ln.count(b"T")
            nn += len(ln) - ln.count(b"A") - ln.count(b"C") - ln.count(b"G") - ln.count(b"T") - ln.count(b"\r")
        elif k % 4 == 3:
            L, i = len(ln), 0
            if b"\r" not in ln:
                if L:
                    q = np.frombuffer(ln, np.int8)
                    mn, mx = min(mn, int(q.min())), max(mx, int(q.max()))
            else:
                while i < L:
                    ch = ln[i]
                    if ch == 13:
                        L -= 1
                    else:
                        sc = ch - 256 if ch >= 128 else ch
                        mn, mx = min(mn, sc), max(mx, sc)
                    i += 1
            maxlen, minlen = max(maxlen, L), min(minlen, L)
    return {"a": a, "c": c, "g": g, "t": t, "n": nn, "maxlen": maxlen, "minlen": minlen, "minqs": mn, "maxqs": mx}


def phred(st):
    """the reference's encoding guess from the quality range (src/fastq.c:768-774)"""
    p = 64 if st["maxqs"] > 74 else 0
    return 33 if st["minqs"] < 59 else p
