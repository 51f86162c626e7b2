"""Restatements and seeded inputs for the full-index statistics kernels (K7, csrc/fxg_stats.cu).

Restatements (numpy, vectorised so that they scale to the inputs below):
- composition(data, rows): per-record counts of the bytes < 128 of [boff, boff + blen) other than '\\n', as COMP_ROW
  rows in (seqid, letter) order, and the whole-file totals[128]; the semantics of edgelib.composition.
- fastq_stats(data): the reference's line walk (src/fastq.c:715-752), the semantics of edgelib.fastq_stats.
- phred(st) and encoding_type(minqs, maxqs), restated from src/fastq.c:758-764 and 797-878.

Inputs, each aimed at a branch of K7 that small inputs never reach:
- many_records: more than 2 * BATCH records, with long records at the batch edges, so that one 8 KiB sub-tile holds
  records of two composition batches.
- tile_sweep: record starts and ends at every offset -17..+17 around 8 KiB sub-tile edges, lines of every byte value,
  empty records and one record of more than 64 MiB.
- quality_classes: FASTQ files whose min or max quality sits on each side of every threshold of the phred guess and of
  the encoding classes, and files with quality bytes >= 0x80.
- step_sweep: FASTQ lines of every length 0..1100 and two long ones, at all 16 alignments, ending on lane and step
  edges of fq_line's 512-byte walk.
- many_reads: more reads than 40 times the warps of the stats launch, with the extremes on single reads that are not
  the last read of their warp.
- INNER_CR: quality lines with a '\\r' before their last byte, where the reference's walk stops early."""
import gzip
import struct
import zlib

import numpy as np

# constants of csrc/fxg_stats.cu (test_full_stats_cpu.py checks them against the source)
CT_SUB = 8192                     # bytes per warp of comp_hist_kernel
CT_WARPS = 2                      # warps per CTA of comp_hist_kernel
BATCH = 1 << 21                   # records per composition pass
LANE = 16                         # bytes per lane and step of fq_line
STEP = 32 * LANE                  # 512: bytes per warp step of fq_line
STATS_CTAS_PER_SM = 8             # fastq_stats_kernel: sm_count * 8 CTAs ...
STATS_THREADS = 256               # ... of 256 threads
NOMINAL_SMS = 132                 # an H100 SXM


def stats_warps(sm_count=NOMINAL_SMS):
    """warps of one fastq_stats_kernel launch (8,448 on an H100 SXM)"""
    return sm_count * STATS_CTAS_PER_SM * STATS_THREADS // 32


COMP_ROW = np.dtype([("seqid", "<i8"), ("abc", "<i8"), ("num", "<i8")])      # _cabi.COMP_ROW


# ---------------------------------------------------------------------------------------------
# restatements
# ---------------------------------------------------------------------------------------------
def _span_hist(a, b0, b1):
    """[len(b0), 128] counts of the records [b0[k], b1[k]) (disjoint, ascending) of a, '\\n' and bytes >= 128 dropped"""
    m = len(b0)
    lo, hi = int(b0[0]), int(b1[-1])
    if m == 1:
        h = np.zeros(256, np.int64)
        for p in range(lo, hi, 1 << 24):
            h += np.bincount(a[p:min(p + (1 << 24), hi)], minlength=256)
        h[10] = 0
        return h[None, :128]
    seg = a[lo:hi]
    starts = np.bincount(b0 - lo, minlength=hi - lo + 1)
    inside = np.cumsum(starts - np.bincount(b1 - lo, minlength=hi - lo + 1))[:-1] > 0
    rid = np.cumsum(starts)[:-1] - 1
    keep = inside & (seg != 10) & (seg < 128)
    return np.bincount(rid[keep] * 128 + seg[keep], minlength=m * 128).reshape(m, 128)


def composition(data, rows, chunk_rows=1 << 18, chunk_bytes=1 << 23):
    """full-index composition -> (COMP_ROW array in (seqid, letter) order, seqid 1-based; totals int64[128]).
    Works on groups of at most chunk_rows records and chunk_bytes bytes (a longer record on its own)."""
    a = np.frombuffer(data, np.uint8)
    n = len(rows)
    total = np.zeros(128, np.int64)
    if n == 0:
        return np.zeros(0, COMP_ROW), total
    b0 = np.minimum(rows["boff"].astype(np.int64), a.size)
    b1 = np.maximum(np.minimum(b0 + rows["blen"].astype(np.int64), a.size), b0)
    out = []
    i = 0
    while i < n:
        j = min(n, i + chunk_rows, max(i + 1, int(np.searchsorted(b1, b0[i] + chunk_bytes, "right"))))
        h = _span_hist(a, b0[i:j], b1[i:j])
        total += h.sum(axis=0)
        r, c = np.nonzero(h)
        part = np.zeros(r.size, COMP_ROW)
        part["seqid"], part["abc"], part["num"] = r + i + 1, c, h[r, c]
        out.append(part)
        i = j
    return np.concatenate(out), total


def comp_table(rows, total):
    """the `comp` table of a full index: the per-record rows, then 128 seqid-0 rows of the totals"""
    tot = np.zeros(128, COMP_ROW)
    tot["abc"], tot["num"] = np.arange(128), total
    return np.concatenate([np.asarray(rows, COMP_ROW), tot])


def comp_digest(table):
    """sha256 of a `comp` table (COMP_ROW array, or a list of [seqid, abc, num]) as little-endian int64 triplets"""
    import hashlib
    if isinstance(table, np.ndarray):
        t = np.stack([table["seqid"], table["abc"], table["num"]], axis=1)
    else:
        t = np.asarray(table, np.int64).reshape(-1, 3)
    return hashlib.sha256(np.ascontiguousarray(t, "<i8").tobytes()).hexdigest()


def fasta_getters(total):
    """Fasta.composition / gc_content / gc_skew / type from the totals, with the reference's float32 arithmetic
    (src/fasta.c:1060-1154); a getter the reference raises for maps to None"""
    h = np.asarray(total, np.int64)
    a, c, g, t = (int(h[ord(x)] + h[ord(x.lower())]) for x in "ACGT")
    out = {"composition": {chr(i): int(h[i]) for i in range(32, 127) if h[i] > 0}}
    out["gc_content"] = float(np.float32(g + c) / np.float32(a + c + g + t) * np.float32(100)) if a + c + g + t > 0 else None
    out["gc_skew"] = float(np.float32(g - c) / np.float32(g + c)) if c + g > 0 else None
    alpha = {chr(i) for i in range(33, 127) if h[i] > 0}
    if alpha <= set("ACGTNacgtn") or alpha <= set("abcdghkmnrstvwyABCDGHKMNRSTVWY*-"):
        out["type"] = "DNA"
    elif alpha <= set("ACGUNacgun") or alpha <= set("abcdghkmnrsuvwyABCDGHKMNRSUVWY*-"):
        out["type"] = "RNA"
    elif alpha <= set("acdefghiklmnpqrstvwyACDEFGHIKLMNPQRSTVWY*-"):
        out["type"] = "protein"
    else:
        out["type"] = "unknown"
    return out


def _ranges_mask(n, lo, hi):
    """bool[n]: positions inside any of the disjoint ranges [lo[k], hi[k])"""
    d = np.bincount(lo, minlength=n + 1) - np.bincount(hi, minlength=n + 1)
    return np.cumsum(d)[:-1] > 0


def lines(data):
    """(starts, ends) of the lines of data, the reference's way: a last line without '\\n' counts, nothing after a
    final '\\n' does"""
    a = np.frombuffer(data, np.uint8)
    nl = np.flatnonzero(a == 10)
    starts = np.concatenate([[0], nl + 1]).astype(np.int64)
    ends = np.concatenate([nl, [a.size]]).astype(np.int64)
    if starts[-1] == a.size:
        starts, ends = starts[:-1], ends[:-1]
    return starts, ends


def fastq_stats(data):
    """the reference's statistics walk over every line of the file (src/fastq.c:715-752): of each line 2 (mod 4) the
    A / C / G / T counts and every other byte but '\\r' as n; of each line 4 (mod 4) the quality range as signed chars
    and the length, where a '\\r' met at index i < l shortens l by one and is skipped (so the walk stops early after
    one).  -> dict like Engine.fastq_stats, phred included"""
    a = np.frombuffer(data, np.uint8)
    n = a.size
    starts, ends = lines(data)
    k = np.arange(starts.size)
    st = {"a": 0, "c": 0, "g": 0, "t": 0, "n": 0, "maxlen": 0, "minlen": 10000000000, "minqs": 104, "maxqs": 33}
    sq = k % 4 == 1
    if sq.any():
        bc = np.bincount(a[_ranges_mask(n, starts[sq], ends[sq])], minlength=256)
        st["a"], st["c"], st["g"], st["t"] = (int(bc[ord(x)]) for x in "ACGT")
        st["n"] = int(bc.sum() - bc[[65, 67, 71, 84, 13]].sum())
    ql = k % 4 == 3
    if ql.any():
        qs, qe = starts[ql], ends[ql]
        L = qe - qs
        idx = np.flatnonzero(_ranges_mask(n, qs, qe))
        qid = np.searchsorted(qs, idx, "right") - 1
        cr = a == 13
        crc = np.concatenate([[0], np.cumsum(cr)])                     # '\r' before each position
        visited = (idx - qs[qid]) + (crc[idx] - crc[qs[qid]]) < L[qid]
        is_cr = cr[idx]
        ln = L - np.bincount(qid[visited & is_cr], minlength=qs.size)
        st["maxlen"], st["minlen"] = max(0, int(ln.max())), min(10000000000, int(ln.min()))
        q = a[idx[visited & ~is_cr]].view(np.int8)
        if q.size:
            st["minqs"], st["maxqs"] = min(104, int(q.min())), max(33, int(q.max()))
    st["phred"] = phred(st)
    return st


def phred(st):
    """the reference's guess from the quality range (src/fastq.c:758-764)"""
    p = 64 if st["maxqs"] > 74 else 0
    return 33 if st["minqs"] < 59 else p


def encoding_type(minqs, maxqs):
    """the reference's list of possible quality encodings (src/fastq.c:797-878)"""
    if minqs < 33 or maxqs > 126:
        return ["Unknown"]
    out = []
    for name, lo, hi in (("Sanger Phred+33", 33, 73), ("Illumina 1.8+ Phred+33", 33, 74), ("Solexa Solexa+64", 59, 104),
                         ("Illumina 1.3+ Phred+64", 64, 104), ("Illumina 1.5+ Phred+64", 66, 104),
                         ("PacBio HiFi Phred+33", 33, 126)):
        if minqs >= lo and maxqs <= hi:
            out.append(name)
    return out


def fastq_answers(data):
    """what Fastq(full_index=True) must give for data: the `base` / `meta` rows and the getters"""
    st = fastq_stats(data)
    g, c, a, t = st["g"], st["c"], st["a"], st["t"]
    return {"base": [[st["a"], st["c"], st["g"], st["t"], st["n"]]],
            "meta": [[st["maxlen"], st["minlen"], st["minqs"], st["maxqs"], st["phred"]]],
            "composition": {k.upper(): st[k] for k in "acgtn"},
            "gc_content": float(np.float32(g + c) / np.float32(a + c + g + t) * np.float32(100)) if a + c + g + t else None,
            "maxlen": st["maxlen"], "minlen": st["minlen"], "maxqual": st["maxqs"], "minqual": st["minqs"],
            "phred": st["phred"], "encoding_type": encoding_type(st["minqs"], st["maxqs"])}


# ---------------------------------------------------------------------------------------------
# FASTA inputs
# ---------------------------------------------------------------------------------------------
ALPHABETS = (b"ACGT", b"acgtn", b"ACGTN", b"ACGU", b"RYKMSWBDHVN", b"ACDEFGHIKLMNPQRSTVWY", b"*-acgt", b"ACGTacgt.~ 0",
             b"\x00\x01\x7f\t")
MANY_RECORDS = 2 * BATCH + 3
LONG_AT = (BATCH - 1, BATCH, 2 * BATCH - 1, 2 * BATCH)
LONG_LEN = 3 * CT_SUB + 777       # several sub-tiles each


def many_records(n=MANY_RECORDS, long_at=LONG_AT, seed=11):
    """n FASTA records named by a 7-digit hex id, of 0..12 sequence bytes in lines of 1..5 (LONG_LEN bytes in lines
    of 61 at the indices long_at), each from 1..3 letters of one alphabet of ALPHABETS, one record in five CRLF"""
    rng = np.random.default_rng(seed)
    L = rng.integers(0, 13, n)
    W = rng.integers(1, 6, n)
    long_at = [i for i in long_at if i < n]
    L[long_at], W[long_at] = LONG_LEN, 61
    crlf = rng.random(n) < 0.2
    e = 1 + crlf.astype(np.int64)
    nlines = (L + W - 1) // W
    hdr = 9 + e                                                            # '>' + 7 hex digits + ' ' ... + eol
    size = hdr + L + nlines * e
    start = np.concatenate([[0], np.cumsum(size)])
    out = np.zeros(int(start[-1]), np.uint8)
    s = start[:-1]
    out[s] = ord(">")
    ids = np.arange(n)
    hexd = np.frombuffer(b"0123456789abcdef", np.uint8)
    for d in range(7):
        out[s + 1 + d] = hexd[(ids >> (4 * (6 - d))) & 15]
    out[s + 8] = ord("x")
    out[(s + 9)[crlf]] = 13
    out[s + hdr - 1] = 10
    # sequence bytes: byte j of record r at s + hdr + j + (j // W) * e; letters from 1..3 picks of the alphabet
    alpha = rng.integers(0, len(ALPHABETS), n)
    alpha[long_at] = 0
    width = rng.integers(1, 4, n)
    pick = rng.integers(0, 1 << 30, (n, 3))
    tot = int(L.sum())
    rr = np.repeat(ids, L)
    j = np.arange(tot) - np.repeat(np.cumsum(L) - L, L)
    table = np.zeros((len(ALPHABETS), 32), np.uint8)
    lens = np.array([len(x) for x in ALPHABETS])
    for k, x in enumerate(ALPHABETS):
        table[k, :len(x)] = np.frombuffer(x, np.uint8)
    which = pick[rr, rng.integers(0, 3, tot) % width[rr]] % lens[alpha[rr]]
    out[s[rr] + hdr[rr] + j + (j // W[rr]) * e[rr]] = table[alpha[rr], which]
    # line ends: line k of record r ends at s + hdr + min((k + 1) W, L) + k e
    lr = np.repeat(ids, nlines)
    k = np.arange(int(nlines.sum())) - np.repeat(np.cumsum(nlines) - nlines, nlines)
    pos = s[lr] + hdr[lr] + np.minimum((k + 1) * W[lr], L[lr]) + k * e[lr]
    out[pos[crlf[lr]]] = 13
    out[pos + e[lr] - 1] = 10
    return out.tobytes()


def _line_bytes(rng, n, ascii_only=False):
    """n bytes of every value but '\\n' (only 0..127 if ascii_only), in a random order"""
    hi = 127 if ascii_only else 255
    b = rng.integers(0, hi, n, dtype=np.uint8)
    b[b >= 10] += 1
    return b


class _FaBuilder:
    def __init__(self, rng, ascii_only):
        self.rng, self.ascii_only = rng, ascii_only
        self.out = bytearray()
        self.k = 0

    def header(self, eol=b"\n"):
        self.k += 1
        self.out += b">r%d" % self.k + eol
        return len(self.out)

    def body(self, nbytes):
        """nbytes of sequence lines of 0..120 bytes + '\\n' ('>' never first; no bytes: a blank line)"""
        while nbytes > 0:
            w = min(nbytes, int(self.rng.integers(1, 122)))
            b = _line_bytes(self.rng, w - 1, self.ascii_only)
            if w > 1 and b[0] == ord(">"):
                b[0] = ord("A")
            self.out += b.tobytes() + b"\n"
            nbytes -= w

    def record_to(self, end, eol=b"\n"):
        """one record that ends exactly at `end`"""
        self.header(eol)
        assert end >= len(self.out), (end, len(self.out))
        self.body(end - len(self.out))


SWEEP = tuple(range(-17, 18))
SWEEP_EDGE0 = 4                  # first sub-tile edge used


def sweep_sites():
    """(sub-tile edge index, offset, kind): every offset with kinds 'end' (a record ends there), 'start' (a record's
    first sequence byte is there) and 'empty' (an empty record's), each at an even and an odd sub-tile edge"""
    out = []
    k = SWEEP_EDGE0
    for d in SWEEP:
        for kind in ("end", "start", "empty"):
            out += [(k, d, kind), (k + 1, d, kind)]
            k += 2
    return out


def tile_sweep(big=(64 << 20) + 4099, ascii_only=False, seed=5):
    """FASTA with record starts / ends at sweep_sites(), then a record of `big` bytes (none if 0) and a short last
    one.  -> bytes"""
    rng = np.random.default_rng(seed)
    b = _FaBuilder(rng, ascii_only)
    b.record_to(200)
    for k, d, kind in sweep_sites():
        at = k * CT_SUB + d
        if kind == "end":
            b.record_to(at)
            b.header()
        elif kind == "start":
            b.record_to(at - len(b">r%d\n" % (b.k + 2)))
            b.header()
        else:
            b.record_to(at - len(b">r%d\r\n" % (b.k + 2)))
            b.header(b"\r\n")
            b.header()                                  # the record just opened is empty
        b.body(int(rng.integers(300, 3000)))
    if big:
        b.header()
        at = len(b.out)
        body = _line_bytes(rng, big, ascii_only)
        ends = np.cumsum(rng.integers(1, 4000, big // 1000 + 16))
        ends = ends[ends < big - 1]
        body[ends] = 10
        nxt = ends + 1
        body[nxt[body[nxt] == ord(">")]] = ord("C")
        if body[0] == ord(">"):
            body[0] = ord("C")
        body[-1] = 10
        b.out += body.tobytes()
        assert len(b.out) - at == big
    b.header()
    b.body(50)
    return bytes(b.out)


# ---------------------------------------------------------------------------------------------
# FASTQ inputs
# ---------------------------------------------------------------------------------------------
SEQ_ALPHA = np.frombuffer(b"ACGTACGTACGTNacgtn.RY", np.uint8)


def _read(rng, name, L, qlo, qhi, eol, q=None):
    seq = SEQ_ALPHA[rng.integers(0, SEQ_ALPHA.size, L)].tobytes()
    if q is None:
        q = rng.integers(qlo, qhi + 1, L).astype(np.uint8).tobytes()
    return name + eol + seq + eol + b"+" + eol + q + eol


QUALITY_PAIRS = tuple((lo, hi) for lo in (32, 33, 58, 59, 63, 64, 65, 66) for hi in (73, 74, 75, 104, 105, 126, 127)
                      if lo < hi)
QUALITY_EXTRA = {
    "high_bytes": (0x80, 0xFF),        # quality bytes 0x80..0xFF among ordinary ones: a negative minimum
    "high_byte_ff": (0xFF, 0xFF),      # 0xFF alone: -1
    "above_104": (105, 120),           # nothing below 105: minqs stays at its start value 104
    "below_33": (20, 32),              # nothing above 32: maxqs stays at its start value 33
    "controls": (1, 127),              # 0x01 and 0x7F, and '\r' anywhere in the quality lines
}

# quality lines with a '\r' before their last byte, where the reference's walk stops early (each '\r' it meets shortens
# the line by one): the visited bytes and the length differ from "every byte but '\r'"
INNER_CR = {
    "inner": b"@a\nACGT\n+\nI\r!~\n@b\nACGT\n+\nIIII\n",                  # '~' (126) never visited: maxqual 73
    "doubled": b"@a\nACG\n+\n#\r\r\n@b\nACGT\n+\nIIII\n",                  # length 2, not 1
    "only_cr": b"@a\nAC\n+\n\r\r\r\n@b\nACGT\n+\n5555\n",
    "before_crlf": b"@a\r\nACGT\r\n+\r\nJ\r!\r\n@b\r\nACG\r\n+\r\n\x7f\rJ\r\n",
    "long": b"@a\nACGT\n+\n" + b"5" * 700 + b"\r" * 300 + b"!" * 50 + b"\n@b\nA\n+\nF\n",    # stops at 875 of 1050
    "last": b"@a\nAC\n+\n55\n@b\nACGT\n+\nIII\rJ\r~",                      # no final newline
}


def quality_classes(eol=b"\n", seed=21):
    """name -> one FASTQ per QUALITY_PAIRS (lo, hi): qualities strictly inside (lo, hi) but for one read holding lo
    as its last quality byte and one holding hi as its first; and the QUALITY_EXTRA files"""
    out = {}
    for name, (lo, hi) in [("q%d_%d" % p, p) for p in QUALITY_PAIRS] + sorted(QUALITY_EXTRA.items()):
        rng = np.random.default_rng([seed, lo, hi])
        parts = []
        n = 60
        ia, ib = int(rng.integers(5, n)), int(rng.integers(5, n))
        ib = ib if ib != ia else (ia + 7) % n
        for i in range(n):
            L = int(rng.integers(1, 140))
            if name.startswith("q"):
                q = rng.integers(lo + 1, hi, L).astype(np.uint8)
            elif name == "high_bytes":
                q = rng.integers(40, 70, L).astype(np.uint8)
                if i % 3 == 0:
                    q[rng.integers(0, L, max(1, L // 4))] = rng.integers(0x81, 0xFF, max(1, L // 4))
            elif name == "high_byte_ff":
                q = rng.integers(40, 70, L).astype(np.uint8)
            else:
                q = rng.integers(lo + 1, hi, L).astype(np.uint8)
                q[q == 10] = 50                                   # no '\n' inside a quality line; '\r' stays
            if i == ia:
                q[-1] = lo
            if i == ib:
                q[0] = hi
            parts.append(_read(rng, b"@%s_%d" % (name.encode(), i), L, 0, 0, eol, q.tobytes()))
        out[name] = b"".join(parts)
    return out


STEP_LENGTHS = tuple(range(0, 1101)) + (10 ** 5, 1 << 20)
STEP_ENDS = ("nl", "nonl", "tail1", "tail2", "tail3")


def step_sweep(eol=b"\n", end="nl", seed=31):
    """FASTQ with one read of every length of STEP_LENGTHS (shuffled), names padded so that the sequence lines start
    at every residue mod 16, qualities 40..70 with the minimum 35 and the maximum 73 as the last byte of the quality
    lines of the 1100- and the 2^20-byte read.  end: 'nl' / 'nonl' -- the last quality line ends exactly at an fq_line
    step edge, with and without a final newline; 'tailN' -- a partial record of N lines after the last read."""
    rng = np.random.default_rng(seed)
    lens = list(STEP_LENGTHS)
    rng.shuffle(lens)
    out = bytearray()
    e = len(eol)
    for i, L in enumerate(lens):
        name = b"@s%d" % i
        pad = (i - (len(out) + len(name) + e)) % 16                 # sequence line start = i (mod 16)
        name += b"_" * pad
        q = rng.integers(40, 71, L).astype(np.uint8)
        if L == 1100:
            q[-1] = 35
        if L == 1 << 20:
            q[-1] = 73
        out += _read(rng, name, L, 0, 0, eol, q.tobytes())
    if end in ("nl", "nonl"):
        # a last read whose quality line ends on a step edge: q0 + e... chosen so that (n - (qstart & ~15)) % 512 == 0
        fit = [(pad, L) for pad in range(2) for L in range(600, 1200)
               if (L + (e if end == "nl" else 0) + ((len(out) + 5 + pad + e + L + e + 1 + e) & 15)) % STEP == 0]
        pad, L = fit[0]
        name = b"@last" + b"_" * pad
        q = rng.integers(40, 71, L).astype(np.uint8).tobytes()
        rec = _read(rng, name, L, 0, 0, eol, q)
        out += rec if end == "nl" else rec[:-e]
    else:
        k = int(end[-1])
        tail = [b"@tail x" + eol, b"ACGTNNacgt" + eol, b"+" + eol][:k]
        out += b"".join(tail)
    return bytes(out)


MANY_READS = 40 * stats_warps() + 1234


def many_reads_marks(n=MANY_READS):
    """indices of the reads with the minimum quality, the maximum, the shortest and the longest read.  Each is followed
    by at least 12,000 reads, so on any launch of up to 12,000 warps the warp that handles it has a later read (on the
    8,448 warps of an H100 SXM it sits in the round before the last)"""
    base = n - 2 * stats_warps() + 600
    return {"minq": base, "maxq": base + 1111, "short": base + 2222, "long": base + 3333}


def many_reads(n=MANY_READS, eol=b"\n", seed=41):
    """n reads of 20..200 bytes, qualities 40..70, except: one read holds quality 34, one 72, one is 3 bytes long and
    one 400 (many_reads_marks)"""
    rng = np.random.default_rng(seed)
    m = many_reads_marks(n)
    L = rng.integers(20, 201, n)
    L[m["short"]], L[m["long"]] = 3, 400
    e = len(eol)
    names = [b"@m%d" % i for i in range(n)]
    nlen = np.array([len(x) for x in names])
    size = nlen + e + L + e + 1 + e + L + e
    start = np.concatenate([[0], np.cumsum(size)])
    out = np.zeros(int(start[-1]), np.uint8)
    blob = np.frombuffer(b"".join(names), np.uint8)
    noff = np.concatenate([[0], np.cumsum(nlen)])
    rid = np.repeat(np.arange(n), nlen)
    out[start[:-1][rid] + np.arange(blob.size) - noff[:-1][rid]] = blob
    s0 = start[:-1] + nlen + e                                      # sequence line starts
    q0 = s0 + L + e + 1 + e                                         # quality line starts
    rr = np.repeat(np.arange(n), L)
    j = np.arange(int(L.sum())) - np.repeat(np.cumsum(L) - L, L)
    out[s0[rr] + j] = SEQ_ALPHA[rng.integers(0, SEQ_ALPHA.size, j.size)]
    qv = rng.integers(40, 71, j.size).astype(np.uint8)
    out[q0[rr] + j] = qv
    out[q0[m["minq"]] + L[m["minq"]] // 2] = 34
    out[q0[m["maxq"]] + L[m["maxq"]] - 1] = 72
    out[s0 + L + e] = ord("+")
    for p in (s0 - e, s0 + L, q0 - e, q0 + L):                     # the four line ends of each read
        if e == 2:
            out[p] = 13
        out[p + e - 1] = 10
    return out.tobytes()


# ---------------------------------------------------------------------------------------------
# compressed forms
# ---------------------------------------------------------------------------------------------
def bgzf(data, level=1, block=0xff00):
    """BGZF (SAM spec 4.1): gzip members with a 'BC' extra field, then the empty EOF member"""
    out = []
    for a in list(range(0, len(data), block)) + [None]:
        chunk = b"" if a is None else data[a:a + block]
        co = zlib.compressobj(level, zlib.DEFLATED, -15)
        comp = co.compress(chunk) + co.flush()
        out.append(b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", len(comp) + 25)
                   + comp + struct.pack("<II", zlib.crc32(chunk), len(chunk)))
    return b"".join(out)


def plain_gzip(data, level=1):
    return gzip.compress(data, compresslevel=level, mtime=0)
