"""CPU companion of test_gather_scale_gpu.py: the constants of gatherlib are the ones in csrc/fxg_extract.cu, the large
sets cross the chunk edges of the offset prefix, every forced batch width gives every resident warp a second batch, and
every record kind, lane kind, batch shape and bad-byte position is what it claims to be, checked against the oracle."""
import os
import re

import numpy as np
import pytest

import gatherlib as G
from oracle import fxo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "pyfastx_b200", "csrc", "fxg_extract.cu")
WIDTHS = (1, 3, 8, 31, 32)


@pytest.fixture(scope="module")
def mixed():
    data, kinds = G.mixed_fasta()
    rows = fxo.fasta_scan(data)[0]
    uni = np.array([G.uniform_of(data, r) for r in rows])
    return data, kinds, rows, uni


def test_constants_match_the_source():
    with open(SRC) as fh:
        src = fh.read()

    def const(name):
        return re.search(r"constexpr (?:int|size_t) %s = ([^;]+);" % name, src).group(1)

    assert int(const("XTHREADS")) // 32 == G.XWARPS and const("XWARPS") == "XTHREADS / 32"
    assert const("XSTAGE") == "512 + 32" and 512 + 32 == G.XSTAGE
    assert int(re.search(r"#define FXG_BK_NS (\d+)", src).group(1)) == G.BK_NS
    assert int(const("BK_WORDS")) == G.BK_WORDS and int(const("BK_SLOT")) == G.BK_SLOT
    assert int(const("PS_ITEMS")) == G.PS_ITEMS
    assert "ps_scan_sums<<<1, %d, 0, ctx->stream>>>" % G.PS_SCAN_THREADS in src
    # BK_SMEM, term by term as gatherlib.bk_smem restates it
    assert const("BK_OFF_BAR") == "(size_t)XWARPS * BK_NS * BK_SLOT"
    assert const("BK_OFF_G0") == "BK_OFF_BAR + (size_t)XWARPS * BK_NS * 8"
    assert const("BK_OFF_QC") == "(BK_OFF_G0 + (size_t)XWARPS * BK_NS * 4 + 15) & ~(size_t)15"
    assert const("BK_OFF_LUT") == "BK_OFF_QC + (size_t)XWARPS * 32 * 32"
    assert const("BK_OFF_STAGE") == "BK_OFF_LUT + 3 * 256"
    assert const("BK_SMEM") == "BK_OFF_STAGE + (size_t)XWARPS * XSTAGE"
    assert G.bk_smem() == 54656 and G.SMEM_PER_SM // G.bk_smem() == 4
    # the default batch width, the forced one, and the grid cap at the resident CTAs
    assert "int bq = nq >= resident_warps * 32 ? 32 : (nq >= resident_warps * 16 ? 16 : 8);" in src
    assert 'getenv("FXG_BK_BQ")' in src and "if (v >= 1 && v <= 32) bq = v;" in src
    assert "const int64_t maxb = (int64_t)ctx->sm_count * ctas_per_sm[v];" in src
    # reads_kernel: a warp per read, at most 8 CTAs of XTHREADS per SM
    assert "const int64_t maxb = (int64_t)ctx->sm_count * 8;" in src


def test_large_sets_cross_the_prefix_chunks():
    chunk = G.PS_ITEMS * G.PS_SCAN_THREADS
    assert chunk == 1 << 21
    a, b, c = G.LARGE_SIZES
    assert G.prefix_chunks(a) == 1 and -(-a // G.PS_ITEMS) == G.PS_SCAN_THREADS        # exactly one full chunk
    assert G.prefix_chunks(b) == 2 and -(-b // G.PS_ITEMS) == G.PS_SCAN_THREADS + 1    # a second chunk of one block
    nb = -(-c // G.PS_ITEMS)
    assert G.prefix_chunks(c) == 3 and 0 < nb % G.PS_SCAN_THREADS < G.PS_SCAN_THREADS  # the third chunk partial
    assert G.prefix_chunks(2000000) == 1                                               # the largest call before


def test_every_warp_serves_two_batches(mixed):
    data, kinds, rows, _ = mixed
    ctas = G.SMEM_PER_SM // G.bk_smem()
    for bq in WIDTHS:
        nq = G.lane_queries(data, kinds, rows, bq)["rid"].size
        assert (nq - bq // 2) // bq >= G.MIN_BATCHES
        for sms in range(1, G.MAX_SMS + 1):
            for c in range(1, ctas + 1):
                assert G.min_warp_batches(nq, bq, sms, c) >= 2, (bq, sms, c)
    # with FXG_BK_BQ unset, the width-32 set and the large sets run at width 32 (nq >= resident warps * 32) ...
    n32 = G.lane_queries(data, kinds, rows, 32)["rid"].size
    assert min(n32, *G.LARGE_SIZES) >= G.max_resident_warps() * 32
    for nq in (n32,) + G.LARGE_SIZES:
        for sms in range(1, G.MAX_SMS + 1):
            assert G.min_warp_batches(nq, 32, sms, ctas) >= 2
    # ... and reads_kernel (a warp per read, 8 CTAs per SM) loops past one read per warp at 50k ids
    assert 50_000 > 2 * G.MAX_SMS * 8 * G.XWARPS


def test_record_kinds(mixed):
    data, kinds, rows, uni = mixed
    assert len(rows) == len(kinds)
    names = fxo.fasta_names(data, rows)
    a = np.frombuffer(data, np.uint8)
    for r, k, u, name in zip(rows, kinds, uni, names):
        assert name.decode() == k["name"]
        assert (int(r["norm"]), bool(u)) == (k["norm"], k["uniform"]), k["name"]
        assert int(r["elen"]) == len(k["eol"]), k["name"]
        if k["uniform"]:
            assert int(r["llen"]) == min(k["width"], int(r["slen"])) + len(k["eol"]), k["name"]
        if k["bad"] is not None:
            bpl = int(r["llen"]) - int(r["elen"])
            R = k["bad"]
            p = int(r["boff"]) + R + int(r["elen"]) * (R // bpl)               # the slice formula's source byte
            if k["kind"] == "bad_crlf":
                assert R % bpl == bpl - 1 and a[p] not in (10, 13, 32) and a[p + 1] == ord("G") and a[p + 2] == 10
            else:
                assert a[p] >= 0x80 or a[p] < 0x40
    by = {k["kind"]: [] for k in kinds}
    for r, k in zip(rows, kinds):
        by[k["kind"]].append(r)
    assert sorted({k["width"] for k in kinds if k["kind"] == "uniform"}) == list(G.WIDTHS)
    assert {int(r["llen"] - r["elen"]) for r in by["uniform"]} >= {15, 16, 4096}
    assert len(by["uniform"]) == 16 and sum(int(r["elen"]) == 2 for r in by["uniform"]) == 8
    assert int(by["oneline"][0]["slen"]) == 100_003 and int(by["oneline"][0]["llen"]) == 100_004
    assert not data.endswith(b"\n") and kinds[-1]["kind"] == "last"
    for r in by["soft"]:
        seq = np.frombuffer(fxo.subseq(data, r, 0, int(r["slen"])), np.uint8)
        assert np.isin(seq, G.IUPAC).any() and np.isin(seq, G.IUPAC | 0x20).any()
        assert (seq == ord("N")).sum() > 1000 and (seq >= 97).mean() > 0.2 and (seq < 97).mean() > 0.2


def _bad_word(a, n, j):
    """where output index j of a query (alignment a, length n) falls: the ragged first or last word, or the item of a
    full word"""
    w = (a + j) >> 4
    if a and w == 0:
        return "first"
    if (a + n) & 15 and w == (a + n - 1) >> 4:
        return "last"
    return "item%d" % ((w - (1 if a else 0)) // G.BK_WORDS)


@pytest.mark.parametrize("bq", WIDTHS)
def test_lane_queries(mixed, bq):
    data, kinds, rows, uni = mixed
    q = G.lane_queries(data, kinds, rows, bq)
    rid, s, e, fl = q["rid"], q["s"], q["e"], q["flags"]
    nq = rid.size
    assert nq % bq == bq // 2
    off = np.concatenate([[0], np.cumsum(np.maximum(e - s, 0))])
    fast, npi = G.bulk_fast(rows, uni, rid, s, e, fl, off, 1 << 40)
    pull = G.pull_ok(rows, uni, rid, s, e, fl, len(data), 1 << 40)
    kind = np.array(q["kind"])
    npat = int((kind != "random").sum())
    assert npat % bq == 0
    # each kind is what it says, and sits at every lane position
    for k in G.FAST_KINDS + G.SLOW_KINDS:
        m = kind == k
        assert set(np.flatnonzero(m) % bq) == set(range(bq)), k
        assert fast[m].all() if k in G.FAST_KINDS else not fast[m].any(), k
    assert (npi[kind == "np0"] == 0).all() and (npi[kind == "one"] == 1).all() and (npi[kind == "multi"] >= 2).all()
    assert (npi[np.char.startswith(kind, "bad_itemN")] >= 2).all()
    assert (e[kind == "neg"] < s[kind == "neg"]).all() and (e[kind == "empty"] == s[kind == "empty"]).all()
    slen = rows["slen"][np.clip(rid, 0, len(rows) - 1)]
    assert (e[kind == "beyond"] > slen[kind == "beyond"]).all()
    assert (fl[kind == "whole"] & G.WHOLE).all() and not uni[rid[kind == "whole"]].any()
    assert (rows["llen"] - rows["elen"])[rid[kind == "narrow"]].max() < 16
    zd = G.zero_defined(rows, rid, s)
    assert np.array_equal(zd, np.isin(kind, ["s_neg", "row_neg", "row_n"]))
    assert {-1, len(rows)} <= set(rid[zd].tolist())
    # batch shapes
    pat = np.array(q["pattern"])[:npat].reshape(-1, bq)[:, 0]
    fb = fast[:npat].reshape(-1, bq)
    lanes = np.arange(bq)
    want = {"all": np.ones(bq, bool), "none": np.zeros(bq, bool), "lane0": lanes == 0, "last": lanes == bq - 1,
            "even": lanes % 2 == 0, "odd": lanes % 2 == 1}
    for p, m in want.items():
        assert (fb[pat == p] == m).all() and (pat == p).any(), p
    nb = fast[npat:npat + (nq - npat) // bq * bq].reshape(-1, bq).sum(axis=1)
    assert ((nb > 0) & (nb < bq)).any() if bq > 1 else ((nb == 0).any() and (nb == 1).any())
    # every bad-byte position on both strands, at the word it was placed in
    seen = set()
    for i in np.flatnonzero(np.char.startswith(kind, "bad")):
        k = kinds[rid[i]]
        a, n, rev = int(off[i]) & 15, int(e[i] - s[i]), bool(fl[i] & G.REVERSE)
        j = (int(s[i]) + n - 1 - k["bad"]) if rev else k["bad"] - int(s[i])
        where = _bad_word(a, n, j)
        base = kind[i][:-1]
        if base in ("bad_break", "bad_edge"):
            j2 = j - 1 if rev else j + 1                     # the first rank after the break
            same = (a + j) >> 4 == (a + j2) >> 4
            assert same == (base == "bad_break") and where.startswith("item") and _bad_word(a, n, j2).startswith("item")
            where = base
        assert rev == kind[i].endswith("-")
        seen.add((base, where, rev))
    assert {(b, w) for b, w, _ in seen} == {("bad_first", "first"), ("bad_last", "last"), ("bad_item0", "item0"),
                                             ("bad_itemN", "item1"), ("bad_break", "bad_break"), ("bad_edge", "bad_edge")}
    assert len(seen) == 12
    paths = {G.path_of(kind[i], fast[i], pull[i], kinds[rid[i]]["kind"] if 0 <= rid[i] < len(rows) else None)
             for i in range(npat)}
    assert paths == {"bulk", "bulk>pull", "bulk>strip", "pull", "strip"}


def test_both_complement_paths(mixed):
    """full output words of bulk queries with COMPLEMENT on soft-masked records: at least 30 % all of A C G T N in either
    case (the register complement), at least 30 % not (the 256-entry LUT)"""
    data, kinds, rows, uni = mixed
    q = G.lane_queries(data, kinds, rows, 32)
    soft = np.array([k["kind"] == "soft" for k in kinds])
    m = soft[q["rid"].clip(0, len(rows) - 1)] & (q["rid"] >= 0) & (q["rid"] < len(rows)) & (q["flags"] & G.COMPLEMENT != 0)
    sub = {k: q[k][m] for k in ("rid", "s", "e", "flags")}
    out, off, _ = fxo.subseq_batch(data, rows, sub["rid"], sub["s"], sub["e"], sub["flags"])
    fast, _ = G.bulk_fast(rows, uni, sub["rid"], sub["s"], sub["e"], sub["flags"], off, 1 << 40)
    # the output buffer is 256-byte aligned: word boundaries are those of the packed offsets
    words = out[:out.size // 16 * 16].reshape(-1, 16)
    wq = np.searchsorted(off, np.arange(words.shape[0]) * 16, side="right") - 1
    full = (off[wq] <= np.arange(words.shape[0]) * 16) & (np.arange(1, words.shape[0] + 1) * 16 <= off[wq + 1])
    keep = full & fast[wq]
    comp4 = np.isin(words[keep], G.ACGTN).all(axis=1)
    assert keep.sum() > 20_000
    assert 0.3 <= comp4.mean() <= 0.7, comp4.mean()
    # and the case changes inside a word: words with lower and upper letters, on both paths
    w = words[keep]
    mixed_case = (w >= 97).any(axis=1) & ((w >= 65) & (w <= 90)).any(axis=1)
    assert (mixed_case & comp4).sum() > 1000 and (mixed_case & ~comp4).sum() > 300


def test_oracle_matches_the_slice_formula(mixed):
    """on records with clean uniform lines, the oracle equals a numpy restatement of the slice formula
    src(k) = boff + k + elen * (k // bpl), with UPPER, COMPLEMENT and REVERSE applied after"""
    data, kinds, rows, uni = mixed
    q = G.lane_queries(data, kinds, rows, 8)
    clean = np.array([k["uniform"] and k["bad"] is None for k in kinds])
    ok = (q["rid"] >= 0) & (q["rid"] < len(rows))
    r = q["rid"].clip(0, len(rows) - 1)
    m = ok & clean[r] & (q["s"] >= 0) & (q["e"] <= rows["slen"][r]) & (q["flags"] & G.WHOLE == 0)
    rid, s, e, fl = q["rid"][m], q["s"][m], q["e"][m], q["flags"][m]
    assert rid.size > 50_000 and (e - s).max() >= 1040
    out, off, _ = fxo.subseq_batch(data, rows, rid, s, e, fl)
    lens = np.maximum(e - s, 0)
    k = np.arange(int(lens.sum())) - np.repeat(off[:-1], lens)          # output index within the query
    rev = np.repeat(fl & G.REVERSE != 0, lens)
    rr = rows[rid]
    kk = np.repeat(s, lens) + np.where(rev, np.repeat(lens, lens) - 1 - k, k)
    bpl = np.repeat(rr["llen"] - rr["elen"].astype(np.int64), lens)
    src = np.repeat(rr["boff"], lens) + kk + np.repeat(rr["elen"].astype(np.int64), lens) * (kk // bpl)
    b = np.frombuffer(data, np.uint8)[src]
    up = np.repeat(fl & G.UPPER != 0, lens) & (b >= 97) & (b <= 122)
    b = np.where(up, b - 32, b).astype(np.uint8)
    b = np.where(np.repeat(fl & G.COMPLEMENT != 0, lens), fxo.complement_lut()[b], b)
    assert np.array_equal(out, b)


def test_reads_inputs():
    for eol, trailing in ((b"\n", True), (b"\r\n", False)):
        data = G.reads_fastq(eol, trailing=trailing)
        rows = fxo.fastq_scan(data)[0]
        rl = rows["rlen"]
        short = rl[:-1][rl[:-1] < 20_000]
        assert len(rows) == 60_000 and short.min() == 1 and 590 < short.max() <= 600 and (rl >= 20_000).sum() == 40
        assert rl[-1] == 777
        assert data.endswith(eol) == trailing
        ids = np.concatenate([np.flatnonzero(rl >= 20_000), [len(rows) - 1], np.arange(0, len(rows), 997)])
        for flags in (0, 2, 4, 6):
            seq, qual, off = G.expect_reads(data, rows, ids, flags)
            for j, i in enumerate(ids):
                es, eq = fxo.read_fetch(data, rows[i])
                es = np.frombuffer(es, np.uint8)
                if flags & G.COMPLEMENT:
                    es = fxo.complement_lut()[es]
                if flags & G.REVERSE:
                    es, eq = es[::-1], eq[::-1]
                assert seq[off[j]:off[j + 1]].tobytes() == es.tobytes() and qual[off[j]:off[j + 1]].tobytes() == eq
