"""Seeded inputs and restatements for the batched gather (K3/K4/K5, csrc/fxg_extract.cu).

Inputs, each aimed at a part of extract_bulk_kernel, reads_kernel or the offset prefix that small calls never reach:
- mixed_fasta: one file of named record kinds (uniform lines at many widths, LF and CRLF, a 100 kB single line, norm = 0
  and odd-line records, soft-masked records, uniform records whose bytes fail the layout check, and a last record
  without a newline), each with the (norm, uniform) the scan must give it.
- lane_queries: queries tagged by kind, laid out so that for one batch width some batches are all fast, some have no
  fast lane, some only lane 0, only the last lane or every other lane fast, every kind sits at every lane position,
  and every resident warp serves at least two batches.
- large_queries: 2^21, 2^21 + 1 and 2 * 2^21 + 2048 + 7 queries, past one and two chunks of ps_scan_sums.
- reads_fastq: FASTQ files of 60k reads of 1..600 bytes and a few of 20k or more.

Restatements:
- bulk_fast / pull_ok: the `fast` condition and item count `np` of extract_bulk_kernel, and the pull condition of
  serve_query_warp, so that every query is labelled with the path it takes (path_of).
- expected: the oracle's bytes and A/C/G/T counts, with the zeros the kernel defines where the oracle cannot index.
- expect_reads: a vectorised numpy fetch of read sequences and qualities."""
import numpy as np

from oracle import fxo

# constants of csrc/fxg_extract.cu (test_gather_scale_cpu.py checks them against the source)
XWARPS = 8                        # warps per CTA of extract_bulk_kernel
BK_NS = 4                         # ring slots per warp
BK_WORDS = 64                     # aligned 16-byte output words per item
BK_SLOT = 1280                    # bytes per ring slot
XSTAGE = 512 + 32                 # staging bytes per warp
PS_ITEMS = 2048                   # queries per block of the offset prefix
PS_SCAN_THREADS = 1024            # threads of the single ps_scan_sums block: block sums per chunk
SMEM_PER_SM = 228 * 1024          # shared memory of one H100 SM
MAX_SMS = 144                     # the full GH100 die; an H100 SXM has 132
UPPER, REVERSE, COMPLEMENT, RAW, WHOLE = 1, 2, 4, 8, 16
RC = REVERSE | COMPLEMENT


def bk_smem():
    """dynamic shared memory of one extract_bulk_kernel CTA (BK_SMEM)"""
    off_bar = XWARPS * BK_NS * BK_SLOT
    off_g0 = off_bar + XWARPS * BK_NS * 8
    off_qc = (off_g0 + XWARPS * BK_NS * 4 + 15) & ~15
    off_lut = off_qc + XWARPS * 32 * 32
    off_stage = off_lut + 3 * 256
    return off_stage + XWARPS * XSTAGE


def max_resident_warps(sms=MAX_SMS):
    """an upper bound of the warps one extract_bulk_kernel launch can have: shared memory caps CTAs per SM"""
    return sms * (SMEM_PER_SM // bk_smem()) * XWARPS


MIN_BATCHES = 2 * max_resident_warps()        # batches a set needs so that every warp serves at least two


def min_warp_batches(nq, bq, sms, ctas_per_sm):
    """the fewest batches any warp serves in the launch fxg_extract_dev makes for nq queries of width bq on sms SMs
    with ctas_per_sm CTAs each: warp g of W serves batches g, g + W, ..."""
    blocks = min(-(-nq // (XWARPS * bq)), sms * ctas_per_sm)
    return -(-nq // bq) // (blocks * XWARPS)


# ---- the mixed FASTA -----------------------------------------------------------------------------------------------
ACGTN = np.frombuffer(b"ACGTNacgtn", np.uint8)
IUPAC = np.frombuffer(b"RYKMSWBDHVU", np.uint8)
WIDTHS = (15, 16, 17, 60, 61, 80, 1000, 4096)


def _soft(rng, n):
    """soft-masked sequence: runs of upper ACGT, lower acgt, N runs of 10..5000, and runs with rare IUPAC codes"""
    out, tot = [], 0
    while tot < n:
        k = rng.integers(0, 5)
        if k == 0:
            run = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, rng.integers(3, 400))]
        elif k == 1:
            run = np.frombuffer(b"acgt", np.uint8)[rng.integers(0, 4, rng.integers(3, 400))]
        elif k == 2:
            run = np.full(int(rng.integers(10, 5001 if rng.random() < 0.2 else 200)), ord("N" if rng.random() < 0.8 else "n"),
                          np.uint8)
        else:                                               # IUPAC codes among the bases, in the run's case
            m = int(rng.integers(50, 600))
            run = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, m)]
            hit = rng.random(m) < 1 / 10
            run[hit] = IUPAC[rng.integers(0, IUPAC.size, int(hit.sum()))]
            if k == 4:
                run = run | 0x20
        out.append(run.astype(np.uint8))
        tot += run.size
    return np.concatenate(out)[:n]


def _wrap(seq, width, eol, last_newline=True):
    body = eol.join(bytes(seq[i:i + width]) for i in range(0, len(seq), width))
    return body + eol if last_newline else body


def mixed_fasta(seed=0):
    """-> (data, kinds): one FASTA file; kinds[i] describes record i: name, kind, norm and uniform (what the scan must
    give it), width, eol, and for a record that fails the layout check `bad`, the kept rank whose source byte is bad (for
    'bad_crlf', the last rank before the break whose '\\r' is a letter)."""
    rng = np.random.default_rng(seed)
    recs, kinds = [], []

    def add(name, kind, body, eol, norm, uniform, width, bad=None):
        recs.append(b">" + name.encode() + b" " + kind.encode() + eol + body)
        kinds.append(dict(name=name, kind=kind, norm=norm, uniform=uniform, width=width, eol=eol, bad=bad))

    for w in WIDTHS:
        for eol in (b"\n", b"\r\n"):
            n = max(5000, 3 * w + w // 3) + int(rng.integers(0, 500))
            add("u%d%s" % (w, "cr" if len(eol) == 2 else ""), "uniform", _wrap(ACGTN[rng.integers(0, 10, n)], w, eol), eol,
                1, True, w)
    add("oneline", "oneline", _wrap(_soft(rng, 100_003), 200_000, b"\n"), b"\n", 1, True, 100_003)
    for i, (w, eol) in enumerate(((60, b"\n"), (80, b"\n"), (70, b"\r\n"))):
        add("soft%d" % i, "soft", _wrap(_soft(rng, 60_000 + 7 * i), w, eol), eol, 1, True, w)
    # an odd line inside: one line of another length (norm = 1, not uniform); two of them (norm = 0)
    # (the scan counts every line as long as the first, the last one included, so the last line is a full one)
    for name, odd, norm in (("odd", (45,), 1), ("norm0", (37, 73), 0)):
        widths = [60] * 40 + sum(([w] + [60] * 10 for w in odd), []) + [60] * 40
        seq = ACGTN[rng.integers(0, 10, sum(widths))]
        ends = np.cumsum(widths)
        add(name, name, b"".join(bytes(seq[b - w:b]) + b"\n" for w, b in zip(widths, ends)), b"\n", norm, False, 60)
    # uniform by their line lengths, but one byte contradicts the layout the bulk path assumes
    for name, w, eol, byte in (("bad_hi", 60, b"\n", 0xC7), ("bad_digit", 61, b"\r\n", ord("7")), ("bad_star", 80, b"\n", ord("*"))):
        n = 6600 + int(rng.integers(0, 300))
        seq = ACGTN[rng.integers(0, 10, n)].copy()
        bad = 3200 + int(rng.integers(0, w))
        seq[bad] = byte
        add(name, name, _wrap(seq, w, eol), eol, 1, True, w, bad)
    seq = ACGTN[rng.integers(0, 10, 6600)]
    k = 53                                                  # line k: 61 letters + '\n', as long as 60 letters + "\r\n"
    lines = [bytes(seq[i:i + 60]) + b"\r\n" for i in range(0, 6600, 60)]
    lines[k] = lines[k][:60] + b"G\n"
    add("bad_crlf", "bad_crlf", b"".join(lines), b"\r\n", 1, True, 60, 60 * k + 59)
    add("last", "last", _wrap(_soft(rng, 7777), 70, b"\n", last_newline=False), b"\n", 1, True, 70)
    return b"".join(recs), kinds


def record_lines(data, row):
    """lengths of the sequence lines of one record (end of line included), from the bytes; the unterminated last line
    of a file counts its virtual newline, as the scan does (blen already runs one past the end of the file there)"""
    a = np.frombuffer(data, np.uint8)
    b0 = int(row["boff"])
    blen = int(row["blen"])
    nl = np.flatnonzero(a[b0:min(b0 + blen, a.size)] == 10) + 1
    ends = np.concatenate([nl, [blen]]) if (nl.size == 0 or nl[-1] != blen) else nl
    return np.diff(np.concatenate([[0], ends]))


def uniform_of(data, row):
    """the scan's uniform bit (pad[0] & 1): every line but the last as long as the first, the last no longer"""
    ln = record_lines(data, row)
    return bool((ln[:-1] == ln[0]).all() and ln[-1] <= ln[0])


# ---- restated predicates --------------------------------------------------------------------------------------------
def _row_fields(rows, rid):
    ok = (rid >= 0) & (rid < len(rows))
    r = rows[np.where(ok, rid, 0)]
    return ok, r


def bulk_fast(rows, uniform, rid, s, e, flags, out_off, capacity):
    """extract_bulk_kernel's `fast` and `np` of every query; `uniform` is the rows' pad[0] & 1 and out_off the packed
    offsets (the output buffer is 256-byte aligned, so a query's first output byte sits at out_off & 15)"""
    ok, r = _row_fields(rows, rid)
    uni = np.asarray(uniform, bool)[np.where(ok, rid, 0)]
    out_len = np.maximum(e - s, 0)
    bpl = r["llen"] - r["elen"].astype(np.int64)
    fast = (ok & (out_len >= 16) & (out_len < (1 << 30)) & (r["norm"] != 0) & uni & (bpl >= 16) & (bpl < (1 << 30)) &
            (s >= 0) & (s < (1 << 32)) & (e <= r["slen"]) & (r["boff"] >= 0) & (r["boff"] + r["blen"] + 32 <= capacity) &
            ((flags & RAW) == 0))
    a = np.asarray(out_off[:len(rid)]) & 15
    tot = a + out_len
    nfull = ((tot + 15) >> 4) - (a != 0) - ((tot & 15) != 0)
    npi = np.where(fast, (np.maximum(nfull, 0) + BK_WORDS - 1) // BK_WORDS, 0)
    return fast, npi


def pull_ok(rows, uniform, rid, s, e, flags, fsize, capacity):
    """serve_query_warp's condition for pull_one (the uniform-line path of a handed-back query)"""
    ok, r = _row_fields(rows, rid)
    uni = np.asarray(uniform, bool)[np.where(ok, rid, 0)]
    ok = ok & (r["boff"] >= 0) & (r["blen"] >= 0) & (r["boff"] <= fsize) & (s >= 0)
    out_len = np.maximum(e - s, 0)
    bpl = r["llen"] - r["elen"].astype(np.int64)
    return (ok & (out_len > 0) & (r["norm"] != 0) & uni & (bpl >= 16) & (bpl < (1 << 30)) & (out_len < (1 << 30)) &
            (e <= r["slen"]) & (r["boff"] + r["blen"] + 32 <= capacity) & ((flags & RAW) == 0))


def path_of(kind, fast, pull, record_kind):
    """the path a query takes: the bulk ring, or handed back to pull_one or the strip path.  A bad query is handed back;
    pull_one's own check passes bytes >= 0x80 (record 'bad_hi') and refuses the others."""
    if fast:
        if not kind.startswith("bad"):
            return "bulk"
        return "bulk>pull" if record_kind == "bad_hi" else "bulk>strip"
    return "pull" if pull else "strip"


def zero_defined(rows, rid, s):
    """queries whose output the kernel defines as zero bytes with zero counts and the oracle cannot index"""
    return (rid < 0) | (rid >= len(rows)) | (s < 0)


def formula_rows(kinds):
    """rows on which WHOLE indexes with the slice formula and that differs from the whole-record strip (DESIGN.md
    section 4): the scan calls 'bad_crlf' uniform, but its one CRLF line ends in a letter + '\\n'"""
    return np.array([k["kind"] == "bad_crlf" for k in kinds])


def expected(data, rows, rid, s, e, flags, formula=None):
    """-> (bytes, offsets, acgt) the kernel must return: the oracle's, zeros where zero_defined, and the oracle without
    WHOLE on the rows of `formula` (a bool per row)"""
    if formula is not None:
        ok = (rid >= 0) & (rid < len(rows))
        flags = np.where(ok & formula[np.where(ok, rid, 0)], flags & ~WHOLE, flags).astype(np.int32)
    z = zero_defined(rows, rid, s)
    rs, ss, es = np.where(z, 0, rid), np.where(z, 0, s), np.where(z, np.maximum(e - s, 0), e)
    out, off, acgt = fxo.subseq_batch(data, rows, rs, ss, es, flags, want_acgt=True)
    if z.any():
        zi = np.flatnonzero(z)
        lens = off[zi + 1] - off[zi]
        idx = np.repeat(off[zi], lens) + (np.arange(int(lens.sum())) - np.repeat(np.cumsum(lens) - lens, lens))
        out[idx] = 0
        acgt[zi] = 0
    return out, off, acgt


# ---- lane queries ---------------------------------------------------------------------------------------------------
FAST_KINDS = ("multi", "one", "np0",
              "bad_first+", "bad_first-", "bad_last+", "bad_last-", "bad_item0+", "bad_item0-", "bad_itemN+", "bad_itemN-",
              "bad_break+", "bad_break-", "bad_edge+", "bad_edge-")
SLOW_KINDS = ("short", "empty", "neg", "whole", "beyond", "s_neg", "row_neg", "row_n", "norm0", "odd", "narrow")
ZERO_LEN = ("empty", "neg")
NEEDS_A = ("np0", "bad_first+", "bad_first-")              # need a ragged first word: a != 0
PATTERNS = ("all", "none", "lane0", "last", "even", "odd", "random")


def _len_range(kind, a):
    if kind == "multi":
        return 1040, 4000
    if kind == "one":
        return 32, 1000
    if kind == "np0":
        return 16, 31 - a
    if kind.startswith("bad_itemN"):
        return 2200, 3000
    if kind.startswith("bad"):
        return 60, 900
    if kind == "short":
        return 1, 15
    if kind in ZERO_LEN:
        return 0, 0
    return 1, 600


def _place_bad(kind, rng, a, n, R):
    """the output index j of the bad rank R (bad_break / bad_edge: of R, the last rank before the bad break) for a
    query of length n whose first output byte has alignment a -> start s"""
    rev = kind.endswith("-")
    w_beg, w_end, t = (1 if a else 0), (a + n) >> 4, (a + n) & 15
    base = kind[:-1]
    if base == "bad_first":
        j = int(rng.integers(0, 16 - a))
    elif base == "bad_last":
        j = int(rng.integers(n - t, n))
    elif base in ("bad_item0", "bad_itemN"):
        lo = w_beg + (BK_WORDS if base == "bad_itemN" else 0)
        w = int(rng.integers(lo, min(lo + BK_WORDS, w_end)))
        j = 16 * w - a + int(rng.integers(0, 16))
    elif base == "bad_break":                               # R and R + 1 in one full word
        w = int(rng.integers(w_beg, w_end))
        j = 16 * w - a + (int(rng.integers(1, 16)) if rev else int(rng.integers(0, 15)))
    else:                                                   # bad_edge: R and R + 1 in two adjacent full words
        w = int(rng.integers(w_beg, w_end - 1))
        j = 16 * (w + 1) - a if rev else 16 * w - a + 15
    return R + j - n + 1 if rev else R - j


def _pattern_kinds(bq):
    """-> list of (pattern, [kind per lane]) batches covering every kind at every lane and every batch shape"""
    nf, ns = len(FAST_KINDS), len(SLOW_KINDS)
    F = lambda i: FAST_KINDS[i % nf]                        # noqa: E731
    S = lambda i: SLOW_KINDS[i % ns]                        # noqa: E731
    out = [("none", [S(p + r) for p in range(bq)]) for r in range(ns)]       # the first lane of all: 'short'
    out += [("all", [F(p + r) for p in range(bq)]) for r in range(nf)]
    for r in range(max(nf, ns)):
        out.append(("lane0", [F(r)] + [S(p + r) for p in range(1, bq)]))
        out.append(("last", [S(p + r) for p in range(bq - 1)] + [F(r)]))
    for r in range(nf):
        out.append(("even", [F(p + r) if p % 2 == 0 else S(p + r) for p in range(bq)]))
        out.append(("odd", [S(p + r) if p % 2 == 0 else F(p + r) for p in range(bq)]))
    return out


def lane_queries(data, kinds, rows, bq, seed=0):
    """queries for batch width bq -> dict of arrays rid, s, e, flags, and the list kind / pattern per query.
    The patterned batches come first; random batches follow until every resident warp serves at least two batches
    (MIN_BATCHES), and a last partial batch of bq // 2 queries ends the set."""
    rng = np.random.default_rng(seed * 1000 + bq)
    by_kind = {}
    for i, k in enumerate(kinds):
        by_kind.setdefault(k["kind"], []).append(i)
    fast_recs = by_kind["uniform"] + by_kind["oneline"] + by_kind["soft"] + by_kind["last"]
    fast_recs = [i for i in fast_recs if kinds[i]["width"] >= 16]
    narrow = [i for i in by_kind["uniform"] if kinds[i]["width"] < 16]
    bad_bytes = by_kind["bad_hi"] + by_kind["bad_digit"] + by_kind["bad_star"]
    slen = rows["slen"].astype(np.int64)
    n_rows = len(rows)

    batches = _pattern_kinds(bq)
    slot_kinds = [k for _, ks in batches for k in ks]
    slot_pat = [p for p, ks in batches for _ in ks]
    rid, s, e, fl = [], [], [], []
    off = 0
    nbad = 0
    for i, kind in enumerate(slot_kinds):
        a = off & 15
        assert not (a == 0 and kind in NEEDS_A), (i, kind)
        nxt = next((k for k in slot_kinds[i + 1:] if k not in ZERO_LEN), None)
        need_nz = kind.startswith("bad_last") or nxt in NEEDS_A
        lo, hi = _len_range(kind, a)
        while True:
            n = int(rng.integers(lo, hi + 1))
            if kind in ZERO_LEN or not need_nz or (a + n) & 15:
                break
        f = int(rng.integers(0, 8))
        if kind.startswith("bad"):
            f = (f & ~REVERSE) | (REVERSE if kind.endswith("-") else 0)
            r = by_kind["bad_crlf"][0] if kind[:-1] in ("bad_break", "bad_edge") else bad_bytes[nbad % len(bad_bytes)]
            nbad += 1
            st = _place_bad(kind, rng, a, n, kinds[r]["bad"])
            assert 0 <= st and st + n <= slen[r], (kind, st, n)
        elif kind in ("multi", "one", "np0", "short", "norm0", "odd", "narrow", "whole"):
            pool = {"norm0": by_kind["norm0"], "odd": by_kind["odd"], "narrow": narrow,
                    "whole": by_kind["norm0"] + by_kind["odd"]}.get(kind, fast_recs)
            pool = [x for x in pool if slen[x] >= n]
            r = pool[int(rng.integers(0, len(pool)))]
            st = int(rng.integers(0, slen[r] - n + 1))
            if kind == "whole":
                f |= WHOLE
        elif kind == "empty":
            r = fast_recs[int(rng.integers(0, len(fast_recs)))]
            st = int(rng.integers(0, slen[r] + 1))
        elif kind == "neg":
            r = fast_recs[int(rng.integers(0, len(fast_recs)))]
            st = int(rng.integers(60, slen[r]))
            n = -int(rng.integers(1, 60))
        elif kind == "beyond":
            r = fast_recs[int(rng.integers(0, len(fast_recs)))]
            st = int(slen[r]) - int(rng.integers(0, n))
        elif kind == "s_neg":
            r = fast_recs[int(rng.integers(0, len(fast_recs)))]
            st = -int(rng.integers(1, 100))
        else:                                               # row_neg, row_n
            r = -1 if kind == "row_neg" else n_rows
            st = int(rng.integers(0, 100))
        rid.append(r); s.append(st); e.append(st + n); fl.append(f)
        off += max(n, 0)
    q = dict(rid=np.array(rid, np.int64), s=np.array(s, np.int64), e=np.array(e, np.int64), flags=np.array(fl, np.int32))
    # random batches: the set's bulk, so that every warp serves a second batch
    nb = max(len(batches), MIN_BATCHES)
    nr = (nb - len(batches)) * bq + bq // 2
    r = random_queries(rows, nr, rng, short=0.45, mid=0.5, long=0.01, neg=0.02, whole=0.05)
    for k in q:
        q[k] = np.concatenate([q[k], r[k]])
    q["kind"] = slot_kinds + ["random"] * nr
    q["pattern"] = slot_pat + ["random"] * nr
    return q


def random_queries(rows, n, rng, short=0.9, mid=0.065, long=0.005, neg=0.03, whole=0.0):
    """n queries on rows (every row id valid): lengths 0..40 with probability `short`, 41..600 `mid`, 1024..3000 `long`,
    e < s `neg`, and the rest 0 (s == e); start uniform so that e <= slen; flags all 8 combinations of UPPER, REVERSE,
    COMPLEMENT, and WHOLE with probability `whole`"""
    slen = rows["slen"].astype(np.int64)
    rid = rng.integers(0, len(rows), n)
    u = rng.random(n)
    c = np.cumsum([short, mid, long, neg])
    ln = np.where(u < c[0], rng.integers(0, 41, n),
                  np.where(u < c[1], rng.integers(41, 601, n),
                           np.where(u < c[2], rng.integers(1024, 3001, n),
                                    np.where(u < c[3], -rng.integers(1, 50, n), 0))))
    ln = np.minimum(ln, slen[rid])
    lo = np.maximum(-ln, 0)
    s = lo + (rng.random(n) * (slen[rid] - np.maximum(ln, 0) - lo + 1)).astype(np.int64)
    flags = rng.integers(0, 8, n) | np.where(rng.random(n) < whole, WHOLE, 0)
    return dict(rid=rid.astype(np.int64), s=s, e=s + ln, flags=flags.astype(np.int32))


LARGE_SIZES = (1 << 21, (1 << 21) + 1, 2 * (1 << 21) + 2048 + 7)


def large_queries(rows, nq, seed=0):
    return random_queries(rows, nq, np.random.default_rng(seed + nq))


def prefix_chunks(nq):
    """chunks of block sums that ps_scan_sums walks for nq queries"""
    return -(-(-(-nq // PS_ITEMS)) // PS_SCAN_THREADS)


# ---- reads ----------------------------------------------------------------------------------------------------------
def reads_fastq(eol=b"\n", n=60_000, seed=0, trailing=True):
    """-> FASTQ bytes: 70 % of reads of 1..40 bases, most others of 41..600, and 40 reads of 20,000..30,000"""
    rng = np.random.default_rng(seed + len(eol))
    u = rng.random(n)
    lens = np.where(u < 0.7, rng.integers(1, 41, n), rng.integers(41, 601, n))
    lens[rng.choice(n - 1, 40, replace=False)] = rng.integers(20_000, 30_001, 40)
    lens[-1] = 777
    seq = np.frombuffer(b"ACGTNacgtnRYKM", np.uint8)[rng.integers(0, 14, int(lens.sum()))]
    qual = rng.integers(33, 127, int(lens.sum())).astype(np.uint8)
    off = np.concatenate([[0], np.cumsum(lens)])
    parts = []
    for i in range(n):
        a, b = off[i], off[i + 1]
        parts.append(b"@r%d x" % i + eol + seq[a:b].tobytes() + eol + b"+" + eol + qual[a:b].tobytes() + eol)
    data = b"".join(parts)
    return data if trailing else data[:-len(eol)]


def expect_reads(data, rows, ids, flags):
    """-> (seq, qual, off) of reads `ids`: rlen bytes at soff and at qoff (0 past the end of the data); the sequence
    complemented through fxo.complement_lut() under COMPLEMENT and reversed under REVERSE, qualities only reversed"""
    a = np.frombuffer(data, np.uint8)
    r = rows[ids]
    lens = r["rlen"].astype(np.int64)
    off = np.zeros(ids.size + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    k = np.arange(int(off[-1])) - np.repeat(off[:-1], lens)
    if flags & REVERSE:
        k = np.repeat(lens, lens) - 1 - k
    out = []
    for base in (r["soff"], r["qoff"]):
        p = np.repeat(base.astype(np.int64), lens) + k
        b = np.where(p < a.size, a[np.minimum(p, a.size - 1)], 0).astype(np.uint8)
        out.append(b)
    seq, qual = out
    if flags & COMPLEMENT:
        seq = fxo.complement_lut()[seq]
    if flags & UPPER:
        seq = np.where((seq >= 97) & (seq <= 122), seq - 32, seq).astype(np.uint8)
    return seq, qual, off
