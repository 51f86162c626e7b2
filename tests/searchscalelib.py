"""Seeded inputs, restated work items and a vectorised reference for pattern search at scale (K8, csrc/fxg_search.cu).

Inputs, each aimed at a loop of the search kernels that small calls never reach:
- fasta_a: ~30 MB of interleaved record kinds with at least 3 * MAX_FASTA_WARPS + 97 work items for m = 16, so that
  every warp of search_kernel / search_approx_kernel takes its grid-stride step (it += nw) at least twice, with runs of
  zero-item records where the second pass starts on 132 and on 144 SMs.
- first_b: 4 long uniform records and at least 6,912 slices, so that the first-hit pass steps w += nw at least twice,
  and planted first hits at items 31, 32, 33, 63 and 64 of their query, so that its b0 += 32 step runs.
- fastq_c: ~50 MB of tiles of 32 reads with at least 3 * MAX_READS_WARPS + 97 items, so that every warp of
  search_reads_kernel runs a range of at least 3 items, crossing tiles, reusing a loaded tile and starting inside a long
  read.
- slices_d: 2^21 + 1 one-item slices of fasta_a's uniform records: the item and hit prefixes take a second chunk.

Restatements (test_search_scale_cpu.py checks the constants against the source): fasta_items (search_items_kernel),
reads_items (tile_items / search_reads_plan_kernel) and the grids of search_grid and search_reads_grid.

Reference: every hit of a set of haystacks laid end to end (the oracle's bytes), found with numpy or bytes.find over
the whole buffer and kept where the match lies inside one haystack; slice_hits answers slices of whole records from
the records' own hits, which holds where a slice's haystack is whole[s:e] (uniform records)."""
import numpy as np
from numpy.lib.stride_tricks import sliding_window_view

from oracle import fxo
import gatherlib

# constants of csrc/fxg_search.cu
SW = 8                                  # warps per CTA of search_kernel
SPIECE = 4096                           # start positions per piece (FXG_SEARCH_PIECE)
SMAXPAT = 1024                          # FXG_SEARCH_MAX_PATTERN
RW = 4                                  # warps per CTA of search_reads_kernel
RWIN = 8192                             # staging window per reads warp
RCH = RWIN // 16
SHB = (SPIECE + SMAXPAT - 1 + 512 + 32 + 15) & ~15
SPB = SMAXPAT + 16
FASTA_SMEM = 2 * SPB + SW * SHB                         # static shared memory of one search_kernel CTA
READS_SMEM = 2 * SPB + RW * (RWIN + 16) + RW * RCH      # ... of one search_reads_kernel CTA
FASTA_CTAS_PER_SM = 4                                   # search_grid: at most sm_count * 4 CTAs
SMEM_PER_SM = gatherlib.SMEM_PER_SM
SMEM_RESERVED_PER_CTA = 1024
READS_CTAS_PER_SM = SMEM_PER_SM // (READS_SMEM + SMEM_RESERVED_PER_CTA)     # shared memory bounds the occupancy
MAX_SMS = gatherlib.MAX_SMS
MAX_FASTA_WARPS = MAX_SMS * FASTA_CTAS_PER_SM * SW
MAX_READS_WARPS = MAX_SMS * READS_CTAS_PER_SM * RW
PS_CHUNK = 1 << 21                                      # entries per chunk of ps_scan_sums (gatherlib)
M_RARE = 16


def fasta_warps(n_items, sms):
    """warps of a search_kernel launch over n_items on sms SMs (search_grid)"""
    return max(min(-(-n_items // SW), sms * FASTA_CTAS_PER_SM), 1) * SW


def reads_warps(n_items, sms, ctas_per_sm):
    """warps of a search_reads_kernel launch (search_reads_grid) with ctas_per_sm resident CTAs per SM"""
    return max(min(-(-n_items // RW), sms * ctas_per_sm), 1) * RW


def reads_per_warp(n_items, sms, ctas_per_sm):
    """items in each warp's contiguous range"""
    return -(-n_items // reads_warps(n_items, sms, ctas_per_sm))


# ---- restated work items ------------------------------------------------------------------------------------------
def fasta_items(rows, uniform, rid, s, e, m):
    """search_items_kernel: the work items of each query (row rid, [s, e)); uniform is the rows' pad[0] & 1.  A query on
    a norm = 1 row with uniform lines has one item per SPIECE start positions, any other query with e - s >= m one."""
    rid = np.asarray(rid, np.int64)
    ok = (rid >= 0) & (rid < len(rows))
    r = rows[np.where(ok, rid, 0)]
    split = ok & (r["norm"] != 0) & np.asarray(uniform, bool)[np.where(ok, rid, 0)]
    ln = np.asarray(e, np.int64) - np.asarray(s, np.int64)
    return np.where(ln >= m, np.where(split, (ln - m + SPIECE) // SPIECE, 1), 0), split


def hit_items(item_off, split, q, start):
    """the work item of each hit (query q, start): the query's first item, plus the piece for a split query"""
    return item_off[q] + np.where(split[q], start // SPIECE, 0)


def reads_items(rlen, m):
    """tile_items / search_reads_plan_kernel on reads of lengths rlen: a tile is 32 reads; each run of short reads
    (rlen <= SPIECE) between the tile's long reads is one item, each long read one item per SPIECE start positions.
    -> dict: tile (items per tile), read_item (each read's first item: its run's, or its first piece's), and per item:
    lane0 and lanes (the reads it covers, as tile lanes), piece (-1 for a run of short reads)."""
    rlen = np.asarray(rlen, np.int64)
    n = rlen.size
    nt = -(-n // 32)
    L = np.zeros(nt * 32, np.int64)
    L[:n] = rlen
    valid = np.arange(nt * 32) < n
    lng = L > SPIECE
    brk = lng | ~valid
    lane = np.arange(nt * 32) % 32
    prev_brk = np.concatenate([[True], brk[:-1]])
    start = valid & ~lng & ((lane == 0) | prev_brk)
    cnt = np.where(lng, (L - m + SPIECE) // SPIECE, start.astype(np.int64))
    excl = np.cumsum(cnt) - cnt
    read_item = (excl - (valid & ~lng & ~start))[:n]
    # per item: a run's lanes end at the next long read, invalid lane or tile start
    ends = np.concatenate([np.flatnonzero(brk | (lane == 0)), [nt * 32]])
    run_at = np.flatnonzero(start)
    nxt = ends[np.searchsorted(ends, run_at, side="right")]
    lg = np.flatnonzero(lng)
    pieces = cnt[lg]
    n_items = int(cnt.sum())
    lane0 = np.zeros(n_items, np.int64)
    lanes = np.zeros(n_items, np.int64)
    piece = np.full(n_items, -1, np.int64)
    lane0[excl[run_at]] = run_at % 32
    lanes[excl[run_at]] = nxt - run_at
    pi = np.repeat(excl[lg], pieces) + (np.arange(int(pieces.sum())) - np.repeat(np.cumsum(pieces) - pieces, pieces))
    lane0[pi] = np.repeat(lg % 32, pieces)
    lanes[pi] = 1
    piece[pi] = pi - np.repeat(excl[lg], pieces)
    return dict(tile=cnt.reshape(nt, 32).sum(axis=1), read_item=read_item, lane0=lane0, lanes=lanes, piece=piece)


def read_hit_items(read_item, rlen, q, start):
    """the work item of each hit (read q, start)"""
    return read_item[q] + np.where(rlen[q] > SPIECE, start // SPIECE, 0)


# ---- the reference ------------------------------------------------------------------------------------------------
def revcomp(pat):
    return bytes(fxo.complement_lut()[np.frombuffer(pat, np.uint8)][::-1])


def fasta_haystacks(data, rows, rid, s, e):
    """the oracle's haystacks of FASTA queries laid end to end -> (buf uint8, off[nq + 1])"""
    rid = np.asarray(rid, np.int64)
    out, off, _ = fxo.subseq_batch(data, rows, rid, s, e, np.zeros(rid.size, np.int32))
    return out, off


def read_haystacks(data, rows):
    """the raw rlen bytes at soff of every read (Read.seq), laid end to end -> (buf, off)"""
    a = np.frombuffer(data, np.uint8)
    lens = rows["rlen"].astype(np.int64)
    off = np.zeros(lens.size + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    src = np.repeat(rows["soff"].astype(np.int64) - off[:-1], lens) + np.arange(int(off[-1]))
    return a[src], off


def _positions(buf, pat):
    """every start of pat in buf, overlapping ones included"""
    m = len(pat)
    if buf.size < m:
        return np.zeros(0, np.int64)
    if m <= 8:
        p = np.frombuffer(pat, np.uint8)
        n = buf.size - m + 1
        ok = buf[:n] == p[0]
        for j in range(1, m):
            ok &= buf[j:j + n] == p[j]
        return np.flatnonzero(ok)
    hay = buf.tobytes()
    out, k = [], hay.find(pat)
    while k >= 0:
        out.append(k)
        k = hay.find(pat, k + 1)
    return np.array(out, np.int64)


def _counts(buf, pat, k, chunk=1 << 20):
    """(starts, mismatches) of every window of buf within k substitutions of pat"""
    m = len(pat)
    p = np.frombuffer(pat, np.uint8)
    pos, cnt = [], []
    for c in range(0, max(buf.size - m + 1, 0), chunk):
        w = sliding_window_view(buf[c:c + chunk + m - 1], m)
        d = np.zeros(w.shape[0], np.int64)
        for j in range(m):
            d += w[:, j] != p[j]
        i = np.flatnonzero(d <= k)
        pos.append(i + c)
        cnt.append(d[i])
    if not pos:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(pos), np.concatenate(cnt)


def _assemble(off, m, per_strand):
    """per_strand: [(minus, global starts, mismatches)] -> (query, start, minus, mismatches) of the matches that lie
    inside one haystack, sorted by (query, start, minus)"""
    pos = np.concatenate([p for _, p, _ in per_strand])
    minus = np.concatenate([np.full(p.size, mi, np.int64) for mi, p, _ in per_strand])
    mm = np.concatenate([c for _, _, c in per_strand])
    q = np.searchsorted(off, pos, side="right") - 1
    ok = pos + m <= off[q + 1]
    o = np.argsort(pos[ok] * 2 + minus[ok], kind="stable")
    q, pos, minus, mm = q[ok][o], pos[ok][o], minus[ok][o], mm[ok][o]
    return q, pos - off[q], minus, mm


def exact_hits(buf, off, pat, strands=3):
    """(query, start, minus) of every occurrence of pat (plus) and of its reverse complement (minus) inside the
    haystacks buf[off[q]:off[q + 1]], in (query, start, minus) order"""
    per = []
    for minus, p in ((0, pat), (1, revcomp(pat))):
        if (strands >> minus) & 1:
            x = _positions(buf, p)
            per.append((minus, x, np.zeros(x.size, np.int64)))
    return _assemble(off, len(pat), per)[:3]


def approx_hits(buf, off, pat, k, strands=3):
    """(query, start, minus, mismatches) of every start within k substitutions, in (query, start, minus) order"""
    per = []
    for minus, p in ((0, pat), (1, revcomp(pat))):
        if (strands >> minus) & 1:
            per.append((minus,) + _counts(buf, p, k))
    return _assemble(off, len(pat), per)


def only(hits, k=None, strands=3):
    """the hits of a strand setting (and within k mismatches) out of a both-strand (and larger k) answer"""
    keep = ((strands >> hits[2]) & 1) != 0
    if k is not None:
        keep &= hits[3] <= k
    return tuple(h[keep] for h in hits)


def slice_hits(whole, rid, s, e, m):
    """hits of slices (rid, s, e) from the hits `whole` of the whole records (query = row id): the record's hits with
    s <= start <= e - m, start made relative to s.  Right where a slice's haystack is whole[s:e]."""
    big = np.int64(1) << 40
    key = whole[0] * big + whole[1]
    rid, s, e = (np.asarray(x, np.int64) for x in (rid, s, e))
    lo = np.searchsorted(key, rid * big + s, side="left")
    hi = np.searchsorted(key, rid * big + e - m, side="right")
    n = np.maximum(hi - lo, 0)
    q = np.repeat(np.arange(rid.size), n)
    idx = np.repeat(lo, n) + (np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n))
    return (q, whole[1][idx] - s[q]) + tuple(h[idx] for h in whole[2:])


def first_hits(hits):
    """the first hit of each (query, strand) of (query, start, minus) in order: what first=True answers"""
    q, st, mi = hits[:3]
    key = q * 2 + mi
    o = np.lexsort((st, key))
    keep = np.ones(o.size, bool)
    keep[1:] = key[o][1:] != key[o][:-1]
    f = o[keep]
    o2 = np.lexsort((mi[f], st[f], q[f]))
    return q[f][o2], st[f][o2], mi[f][o2]


# ---- inputs -------------------------------------------------------------------------------------------------------
ACGT = np.frombuffer(b"ACGT", np.uint8)


def patterns(seed=0):
    """rare: a 16-mer; dense: GAATTC and T; long: SMAXPAT bytes"""
    rng = np.random.default_rng(seed + 555)
    return dict(rare=ACGT[rng.integers(0, 4, M_RARE)].tobytes(), gaattc=b"GAATTC", t=b"T",
                long=ACGT[rng.integers(0, 4, SMAXPAT)].tobytes())


def variant(pat, d, rng):
    """pat with d substituted bases"""
    v = np.frombuffer(pat, np.uint8).copy()
    for j in rng.choice(len(pat), d, replace=False):
        v[j] = ACGT[(int(np.flatnonzero(ACGT == v[j])[0]) + int(rng.integers(1, 4))) % 4]
    return v.tobytes()


def wrap(seq, w, eol):
    """seq in lines of w bases, each ended by eol"""
    n, le = seq.size, len(eol)
    if n == 0:
        return b""
    nl = -(-n // w)
    out = np.empty(n + nl * le, np.uint8)
    k = np.arange(n)
    out[k + (k // w) * le] = seq
    ends = np.minimum((np.arange(nl) + 1) * w, n) + np.arange(nl) * le
    for j in range(le):
        out[ends + j] = eol[j]
    return out.tobytes()


def _long_len(rng, pieces, m=M_RARE):
    """a length with `pieces` items at pattern length m that is also long (> SPIECE) for FASTQ"""
    return int(rng.integers(max((pieces - 1) * SPIECE + m, SPIECE + 1), pieces * SPIECE + m))


class _Planter:
    """plants patterns into per-record base arrays, never two within SMAXPAT + 64 of each other"""

    def __init__(self, seqs, rng):
        self.seqs, self.rng, self.used, self.out = seqs, rng, {}, []

    def put(self, rid, pos, pat, minus, d, where):
        p = variant(pat, d, self.rng) if d else pat
        p = revcomp(p) if minus else p
        if pos < 0 or pos + len(p) > self.seqs[rid].size:
            return False
        if any(abs(pos - u) < SMAXPAT + 64 for u in self.used.get(rid, [])):
            return False
        self.seqs[rid][pos:pos + len(p)] = np.frombuffer(p, np.uint8)
        self.used.setdefault(rid, []).append(pos)
        self.out.append(dict(rid=rid, pos=pos, minus=int(minus), d=d, m=len(p), where=where))
        return True


def _items16(kind, n):
    if kind == "norm0":
        return 1
    return (n - M_RARE + SPIECE) // SPIECE if n >= M_RARE else 0


def fasta_a(seed=0):
    """-> (data, kinds, planted, zero_runs).  kinds[i] of record i: kind ('lf', 'crlf' uniform lines, 'norm0' a blank
    line in the middle and longer than 3 windows, 'short' 1 .. m - 1 bases, 'empty'), norm, uniform, width, eol, n
    (bases), items (for m = 16).  planted: the rare 16-mer (d = 0) and variants of it with d = 1, 2 substitutions,
    where = 'boundary' (start in [k * SPIECE - m + 1, k * SPIECE]), 'random' or 'last' (the last items), and the long
    pattern once across a piece boundary late in the file.  zero_runs: (first record, count, item offset for m = 16) of
    the runs of zero-item records: at the start, at items fasta_warps(., 132) and fasta_warps(., 144), at the end."""
    rng = np.random.default_rng(seed + 1)
    pats = patterns(seed)
    body = (["lf1"] * 9400 + ["crlf1"] * 1600 + ["lf"] * 170 + ["crlf"] * 30 + ["norm0"] * 60 + ["short"] * 300 +
            ["empty"] * 150)
    body = [body[i] for i in rng.permutation(len(body))]
    recs = []                                           # (kind, n, width, eol)

    def rec(kind, pieces=None):
        if kind in ("lf1", "crlf1", "lf", "crlf"):
            crlf = kind.startswith("crlf")
            w = int(rng.choice([60, 70])) if crlf else int(rng.choice([60, 61, 80]))
            if pieces is None:
                pieces = 1 if kind.endswith("1") else int(rng.integers(2, 41))
            n = int(rng.integers(M_RARE, 2001)) if pieces == 1 and kind.endswith("1") else _long_len(rng, pieces)
            return ("crlf" if crlf else "lf", n, w, b"\r\n" if crlf else b"\n")
        if kind == "norm0":
            return ("norm0", int(rng.integers(3 * SPIECE + 100, 16001)), 60, b"\n")
        if kind == "short":
            return ("short", int(rng.integers(1, M_RARE)), 60, b"\n")
        return ("empty", 0, 60, b"\n")

    zero_runs = []

    def zero_run(k, items):
        zero_runs.append((len(recs), k, items))
        for j in range(k):
            recs.append(rec("short" if j % 2 == 0 else "empty"))

    zero_run(5, 0)
    targets = [fasta_warps(1 << 30, 132), fasta_warps(1 << 30, 144)]
    items = 0
    for kind in body:
        r = rec(kind)
        n = _items16(r[0], r[1])
        if targets and items + n > targets[0]:
            gap = targets[0] - items
            if gap:
                recs.append(rec("lf", pieces=gap))
            zero_run(4, targets[0])
            items = targets.pop(0)
        recs.append(r)
        items += n
    zero_run(5, items)

    total = sum(r[1] for r in recs)
    bases = ACGT[rng.integers(0, 4, total, dtype=np.uint8)]
    starts = np.concatenate([[0], np.cumsum([r[1] for r in recs])])
    seqs = [bases[starts[i]:starts[i + 1]] for i in range(len(recs))]
    pl = _Planter(seqs, rng)
    multi = [i for i, r in enumerate(recs) if r[0] in ("lf", "crlf") and _items16(r[0], r[1]) >= 2]
    with_items = [i for i, r in enumerate(recs) if _items16(r[0], r[1]) >= 1]
    i = multi[-1]
    assert pl.put(i, (_items16("lf", recs[i][1]) - 1) * SPIECE - 300, pats["long"], False, 0, "long")
    while sum(p["where"] == "boundary" for p in pl.out) < 50:
        i = multi[int(rng.integers(0, len(multi)))]
        k = int(rng.integers(1, _items16("lf", recs[i][1])))
        pl.put(i, k * SPIECE - int(rng.integers(0, M_RARE)), pats["rare"], rng.random() < 0.5, 0, "boundary")
    for d, want in ((0, 90), (1, 30), (2, 30)):
        while sum(p["where"] == "random" and p["d"] == d for p in pl.out) < want:
            i = with_items[int(rng.integers(0, len(with_items)))]
            pl.put(i, int(rng.integers(0, recs[i][1] - M_RARE + 1)), pats["rare"], rng.random() < 0.5, d, "random")
    for j, i in enumerate(with_items[-6:]):             # the last items of the file
        pl.put(i, recs[i][1] - M_RARE - 7 * j, pats["rare"], j % 2 == 1, 0, "last")

    parts, kinds = [], []
    for i, (kind, n, w, eol) in enumerate(recs):
        s = seqs[i]
        if kind == "norm0":
            cut = 60 * int(rng.integers(10, 100))
            b = wrap(s[:cut], 60, eol) + eol + wrap(s[cut:], 60, eol)
        else:
            b = wrap(s, w, eol)
        parts.append(b">a%d %s" % (i, kind.encode()) + eol + b)
        kinds.append(dict(kind=kind, n=n, width=w, eol=eol, norm=0 if kind == "norm0" else 1,
                          uniform=kind != "norm0", items=_items16(kind, n)))
    return b"".join(parts), kinds, pl.out, zero_runs


FIRST_ITEMS = (31, 32, 33, 63, 64)
B_PIECES = ((70, 60, b"\n", "before"), (68, 61, b"\n", "after"), (52, 80, b"\n", "before"), (41, 70, b"\r\n", "after"))
B_NQ = 7200


def first_b(seed=0):
    """-> (data, pattern, q, plants).  4 uniform records of 41 .. 70 pieces, each with one copy of a 20-mer (plus) at
    P and its reverse complement 5000 bases after it; 'before' records have one more reverse complement 3 pieces + 123
    bases before P.  q: B_NQ queries (rid, s, e, kind), shuffled: 'planted' slices whose first plus hit is at item
    q['item'] (one of FIRST_ITEMS), at offset q['at'] in that item (SPIECE - 1 on some: the match runs into the next
    piece), 'whole' records, 'short' slices (most around a copy) and 'zero' slices (e - s < m: no items)."""
    rng = np.random.default_rng(seed + 2)
    pat = ACGT[rng.integers(0, 4, 20)].tobytes()
    m = len(pat)
    seqs, plants, parts = [], [], []
    for r, (pieces, w, eol, side) in enumerate(B_PIECES):
        n = _long_len(rng, pieces, m)
        s = ACGT[rng.integers(0, 4, n, dtype=np.uint8)]
        P = n - SPIECE - 1500 - int(rng.integers(0, 1000))
        cp = {"plus": P, "after": P + 5000}
        if side == "before":
            cp["before"] = P - 3 * SPIECE - 123
        for name, pos in cp.items():
            s[pos:pos + m] = np.frombuffer(pat if name == "plus" else revcomp(pat), np.uint8)
        seqs.append(s)
        plants.append(dict(cp, side=side, n=n))
        parts.append(b">b%d" % r + eol + wrap(s, w, eol))
    data = b"".join(parts)
    rid, st, en, kind, item, at = [], [], [], [], [], []

    def add(r, a, b, k, it=-1, o=-1):
        rid.append(r); st.append(a); en.append(b); kind.append(k); item.append(it); at.append(o)

    for rep in range(3):
        for r, pc in enumerate(plants):
            P, n = pc["plus"], pc["n"]
            for k in FIRST_ITEMS:
                for o in (0, int(rng.integers(1, SPIECE - 1)), SPIECE - 1):
                    a = P - k * SPIECE - o
                    if a < 0:
                        continue
                    b = n if rep != 1 else int(rng.integers(P + m, pc["after"] + m))   # the 'after' copy cut off
                    add(r, a, b, "planted", k, o)
        for r, pc in enumerate(plants):
            add(r, 0, pc["n"], "whole")
    while len(rid) < B_NQ * 3 // 5:
        r = int(rng.integers(0, 4))
        ln = int(rng.integers(m, 6000))
        c = [v for kk, v in plants[r].items() if kk in ("plus", "after", "before")]
        c = c[int(rng.integers(0, len(c)))]
        a = c + m - ln + int(rng.integers(0, ln - m + 1)) if rng.random() < 0.6 else int(rng.integers(0, plants[r]["n"]))
        a = min(max(a, 0), plants[r]["n"] - ln)
        add(r, a, a + ln, "short")
    while len(rid) < B_NQ:
        r = int(rng.integers(0, 4))
        a = int(rng.integers(0, plants[r]["n"] - m))
        add(r, a, a + int(rng.integers(0, m)), "zero")
    o = rng.permutation(len(rid))
    q = dict(rid=np.array(rid, np.int64)[o], s=np.array(st, np.int64)[o], e=np.array(en, np.int64)[o],
             kind=np.array(kind)[o], item=np.array(item, np.int64)[o], at=np.array(at, np.int64)[o])
    return data, pat, q, plants


C_TILES = (("short", 8000), ("long1", 200), ("longs", 80), ("piece", 20))
C_CRLF_TILES = 300


def _tile_lengths(rng, kind):
    """read lengths of one tile, and its item count for m = 16 stated by kind"""
    u = rng.random(32)
    L = np.where(u < 0.7, rng.integers(20, 51, 32), rng.integers(51, 121, 32))
    if kind in ("short", "crlf"):
        L[rng.random(32) < 0.03] = rng.integers(1, M_RARE)
        L[rng.random(32) < 0.02] = 0
        return L, 1
    if kind in ("long1", "last"):
        p = 8 if kind == "last" else int(rng.integers(5, 13))
        L[30 if kind == "last" else int(rng.integers(8, 24))] = _long_len(rng, p)   # 'last': the file ends in a 1-read run
        return L, p + 2
    if kind == "longs":
        n = int(rng.integers(2, 6))
        j = int(rng.integers(0, 33 - n))
        ps = rng.integers(1, 4, n)
        L[j:j + n] = [_long_len(rng, int(p)) for p in ps]
        return L, int(ps.sum()) + (j > 0) + (j + n < 32)
    L[[5, 6, 20, 21]] = [SPIECE, SPIECE + 1, SPIECE + 1, SPIECE]     # PIECE is short, PIECE + 1 long
    return L, 5


def fastq_c(seed=0):
    """-> (data, tiles, planted).  tiles[t]: kind ('short', 'long1' one long read of 5 .. 12 pieces in the middle,
    'longs' 2 .. 5 adjacent long reads, 'piece' reads of SPIECE and SPIECE + 1, 'crlf' short reads in a CRLF stretch,
    'last' the last tile: a long read of 8 pieces at lane 30, holding the long pattern across a piece boundary, and
    one short read after it), eol and items (for m = 16).
    planted: as fasta_a's, by read."""
    rng = np.random.default_rng(seed + 3)
    pats = patterns(seed)
    kinds = sum(([k] * n for k, n in C_TILES), [])
    kinds = [kinds[i] for i in rng.permutation(len(kinds))]
    kinds = ["short"] + kinds[:4000] + ["crlf"] * C_CRLF_TILES + kinds[4000:] + ["last"]
    lens, tiles = [], []
    for k in kinds:
        L, it = _tile_lengths(rng, k)
        lens.append(L)
        tiles.append(dict(kind=k, eol=b"\r\n" if k == "crlf" else b"\n", items=it))
    rlen = np.concatenate(lens).astype(np.int64)
    bases = ACGT[rng.integers(0, 4, int(rlen.sum()), dtype=np.uint8)]
    off = np.concatenate([[0], np.cumsum(rlen)])
    seqs = [bases[off[i]:off[i + 1]] for i in range(rlen.size)]
    pl = _Planter(seqs, rng)
    long_ids = np.flatnonzero(rlen > SPIECE)
    multi = long_ids[(rlen[long_ids] - M_RARE + SPIECE) // SPIECE >= 2]
    fits = np.flatnonzero(rlen >= M_RARE)
    i = int(long_ids[-1])
    assert pl.put(i, 5 * SPIECE - 400, pats["long"], True, 0, "long")
    while sum(p["where"] == "boundary" for p in pl.out) < 40:
        i = int(multi[int(rng.integers(0, multi.size))])
        k = int(rng.integers(1, (rlen[i] - M_RARE + SPIECE) // SPIECE))
        pl.put(i, k * SPIECE - int(rng.integers(0, M_RARE)), pats["rare"], rng.random() < 0.5, 0, "boundary")
    for d, want in ((0, 70), (1, 25), (2, 25)):
        while sum(p["where"] == "random" and p["d"] == d for p in pl.out) < want:
            i = int(fits[int(rng.integers(0, fits.size))])
            pl.put(i, int(rng.integers(0, rlen[i] - M_RARE + 1)), pats["rare"], rng.random() < 0.5, d, "random")
    for j, i in enumerate(fits[-8:]):
        pl.put(int(i), int(rlen[i]) - M_RARE, pats["rare"], j % 2 == 0, 0, "last")
    parts = []
    qual = b"I" * int(rlen.max())
    for i in range(rlen.size):
        eol = tiles[i // 32]["eol"]
        parts.append(b"@c%d" % i + eol + seqs[i].tobytes() + eol + b"+" + eol + qual[:rlen[i]] + eol)
    return b"".join(parts), tiles, pl.out


D_NQ = PS_CHUNK + 1


def slices_d(rows, uniform, planted, seed=0):
    """D_NQ slices of 64 .. 400 bases of fasta_a's uniform records of at least 400 bases: a third placed over a planted
    exact copy of the rare 16-mer, a tenth over a planted variant, the rest anywhere -> (rid, s, e)"""
    rng = np.random.default_rng(seed + 4)
    slen = rows["slen"].astype(np.int64)
    ok = np.asarray(uniform, bool) & (rows["norm"] != 0) & (slen >= 400)
    elig = np.flatnonzero(ok)
    n = D_NQ
    ln = rng.integers(64, 401, n)
    rid = elig[np.searchsorted(np.cumsum(slen[elig]), rng.random(n) * slen[elig].sum(), side="right")]
    s = (rng.random(n) * (slen[rid] - ln + 1)).astype(np.int64)
    pl = [p for p in planted if p["m"] == M_RARE and ok[p["rid"]]]
    for frac, exact in ((1 / 3, True), (1 / 10, False)):
        pool = [p for p in pl if (p["d"] == 0) == exact]
        pr = np.array([p["rid"] for p in pool])
        pp = np.array([p["pos"] for p in pool])
        sel = np.flatnonzero(rng.random(n) < frac)
        c = rng.integers(0, len(pool), sel.size)
        rid[sel] = pr[c]
        a = pp[c] + M_RARE - ln[sel] + (rng.random(sel.size) * (ln[sel] - M_RARE + 1)).astype(np.int64)
        s[sel] = np.clip(a, 0, slen[pr[c]] - ln[sel])
    return rid.astype(np.int64), s, s + ln
