"""CPU companion of test_search_scale_gpu.py: the constants of searchscalelib are the ones in csrc/fxg_search.cu, every
set reaches the loop it aims at on any H100 (up to 144 SMs), every record, tile and planted hit is what it claims to be,
checked against the oracle, and the vectorised reference equals searchlib / approxlib."""
import gzip
import os
import re

import numpy as np
import pytest

import approxlib as A
import gatherlib as G
import gen
import goldenlib
import searchlib as S
import searchscalelib as L
from oracle import fxo
from pyfastx_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "pyfastx_b200", "csrc", "fxg_search.cu")
PATS = L.patterns()


@pytest.fixture(scope="module")
def fa_a():
    data, kinds, planted, zero_runs = L.fasta_a()
    rows = fxo.fasta_scan(data)[0]
    uni = np.array([G.uniform_of(data, r) for r in rows])
    n = len(rows)
    buf, off = L.fasta_haystacks(data, rows, np.arange(n), np.zeros(n, np.int64), rows["slen"])
    return data, kinds, planted, zero_runs, rows, uni, buf, off, L.approx_hits(buf, off, PATS["rare"], 2)


@pytest.fixture(scope="module")
def fq_c():
    data, tiles, planted = L.fastq_c()
    rows = fxo.fastq_scan(data)[0]
    buf, off = L.read_haystacks(data, rows)
    return data, tiles, planted, rows, buf, off, L.approx_hits(buf, off, PATS["rare"], 2)


def as_list(hits):
    return list(zip(*(h.tolist() for h in hits)))


def test_constants_match_the_source():
    with open(SRC) as fh:
        src = fh.read()

    def const(name):
        return re.search(r"constexpr int %s = ([^;]+);" % name, src).group(1).strip()

    assert int(const("SW")) == L.SW and int(const("RW")) == L.RW and int(const("RWIN")) == L.RWIN
    assert const("SPIECE") == "FXG_SEARCH_PIECE" and const("SMAXPAT") == "FXG_SEARCH_MAX_PATTERN"
    hdr = open(os.path.join(ROOT, "include", "fxg.h")).read()
    assert int(re.search(r"#define FXG_SEARCH_PIECE\s+(\d+)", hdr).group(1)) == L.SPIECE
    assert int(re.search(r"#define FXG_SEARCH_MAX_PATTERN\s+(\d+)", hdr).group(1)) == L.SMAXPAT
    assert const("SHB") == "(SPIECE + SMAXPAT - 1 + 512 + 32 + 15) & ~15"
    assert const("SPB") == "SMAXPAT + 16" and const("RCH") == "RWIN / 16"
    # static shared memory, as the kernels declare it
    assert "__shared__ __align__(16) uint8_t s_pat[2][SPB];" in src
    assert "__shared__ __align__(16) uint8_t s_hay[SW][SHB];" in src
    assert "__shared__ __align__(16) uint8_t s_win[RW][RWIN + 16];" in src
    assert "__shared__ uint8_t s_map[RW][RCH];" in src
    assert (L.SHB, L.FASTA_SMEM, L.READS_SMEM) == (5664, 47392, 36960)
    # the launch bounds and the grid caps
    assert src.count("__launch_bounds__(SW * 32, 4)") == 2 and src.count("__launch_bounds__(RW * 32)") == 2
    assert "const int64_t maxb = (int64_t)ctx->sm_count * 4;" in src and L.FASTA_CTAS_PER_SM == 4
    assert "const int64_t maxb = (int64_t)ctx->sm_count * per_sm[approx ? 1 : 0];" in src
    assert "int64_t blocks = (warps + SW - 1) / SW;" in src and "int64_t blocks = (n_items + RW - 1) / RW;" in src
    # the loops the sets aim at
    assert "for (int64_t it = gw; it < n_items; it += nw) {" in src
    assert "for (int64_t w = gw; w < 2 * A.nq; w += nw) {" in src
    assert "for (int64_t b0 = i0; b0 < i1; b0 += 32) {" in src
    assert "per = (n_items + nw - 1) / nw;" in src and "while (A.tile_off[t + 1] <= it) ++t;" in src
    assert "if (len >= A.m) n = split_row(r, row_ok) ? (len - A.m + SPIECE) / SPIECE : 1;" in src
    assert "if (lng) return (len - A.m + SPIECE) / SPIECE;" in src
    assert "const bool lng = len > SPIECE;" in src
    # shared memory bounds the reads kernels at 6 CTAs per SM, so at most 3,456 warps; search_kernel at 4,608
    assert L.READS_CTAS_PER_SM == 6 and L.MAX_READS_WARPS == 3456 and L.MAX_FASTA_WARPS == 4608


def test_fasta_items_give_every_warp_three(fa_a):
    data, kinds, planted, zero_runs, rows, uni, buf, off, rare = fa_a
    n = len(rows)
    items, split = L.fasta_items(rows, uni, np.arange(n), np.zeros(n, np.int64), rows["slen"], L.M_RARE)
    assert items.tolist() == [k["items"] for k in kinds]
    tot = int(items.sum())
    assert tot >= 3 * L.MAX_FASTA_WARPS + 97
    for sms in range(1, L.MAX_SMS + 1):
        assert tot // L.fasta_warps(tot, sms) >= 3, sms
    # the other patterns' item counts too
    for p in PATS.values():
        it, _ = L.fasta_items(rows, uni, np.arange(n), np.zeros(n, np.int64), rows["slen"], len(p))
        assert it.sum() >= 2 * L.MAX_FASTA_WARPS + 97 or len(p) == L.SMAXPAT
    # kinds interleaved: every kind with items meets warps on their first and on their third pass, at 132 and 144 SMs
    item_off = np.concatenate([[0], np.cumsum(items)])
    kind = np.array([k["kind"] + ("1" if k["kind"] != "norm0" and k["items"] == 1 else "") for k in kinds])
    for sms in (132, 144):
        nw = L.fasta_warps(tot, sms)
        first = set(kind[(items > 0) & (item_off[:-1] < nw)])
        third = set(kind[(items > 0) & (item_off[:-1] >= 2 * nw) & (item_off[:-1] < 3 * nw)])
        assert first == third == {"lf", "lf1", "crlf", "crlf1", "norm0"}, sms


def test_fasta_record_kinds(fa_a):
    data, kinds, planted, zero_runs, rows, uni, buf, off, rare = fa_a
    assert len(rows) == len(kinds)
    for r, k, u in zip(rows, kinds, uni):
        assert (int(r["norm"]), bool(u), int(r["slen"])) == (k["norm"], k["uniform"], k["n"]), k
        if k["kind"] in ("lf", "crlf") and k["n"] > k["width"]:
            assert (int(r["llen"]), int(r["elen"])) == (k["width"] + len(k["eol"]), len(k["eol"]))
    kind = np.array([k["kind"] for k in kinds])
    slen = rows["slen"]
    assert (slen[kind == "norm0"] > 3 * L.SPIECE).all() and (kind == "norm0").sum() >= 50
    assert slen[kind == "short"].max() < L.M_RARE and (slen[kind == "empty"] == 0).all()
    pieces = np.array([k["items"] for k in kinds])
    for kk in ("lf", "crlf"):
        assert pieces[kind == kk].min() == 1 and pieces[kind == kk].max() == 40, kk
    assert {k["width"] for k in kinds if k["kind"] == "lf"} == {60, 61, 80}


def test_zero_item_runs(fa_a):
    data, kinds, planted, zero_runs, rows, uni, buf, off, rare = fa_a
    n = len(rows)
    items, _ = L.fasta_items(rows, uni, np.arange(n), np.zeros(n, np.int64), rows["slen"], L.M_RARE)
    item_off = np.concatenate([[0], np.cumsum(items)])
    tot = int(item_off[-1])
    want = [0, L.fasta_warps(tot, 132), L.fasta_warps(tot, 144), tot]
    assert [z[2] for z in zero_runs] == want
    for first, cnt, at in zero_runs:
        assert (items[first:first + cnt] == 0).all() and cnt >= 4
        assert item_off[first] == at and item_off[first + cnt] == at
    assert zero_runs[0][0] == 0 and zero_runs[-1][0] + zero_runs[-1][1] == n


def test_planted_fasta_hits(fa_a):
    """every planted copy is a hit of the reference where the plant says; boundary copies start at one of k * SPIECE -
    m + 1 .. k * SPIECE, 'last' copies in the last items, the long pattern late and across a piece boundary"""
    data, kinds, planted, zero_runs, rows, uni, buf, off, rare = fa_a
    n = len(rows)
    items, split = L.fasta_items(rows, uni, np.arange(n), np.zeros(n, np.int64), rows["slen"], L.M_RARE)
    item_off = np.concatenate([[0], np.cumsum(items)])
    tot = int(item_off[-1])
    hits = rare
    got = set(as_list(hits))
    for p in planted:
        if p["m"] == L.M_RARE:
            assert (p["rid"], p["pos"], p["minus"], p["d"]) in got, p
            assert p["where"] != "boundary" or (p["pos"] + L.M_RARE - 1) % L.SPIECE < L.M_RARE
    where = [p["where"] for p in planted]
    assert where.count("boundary") == 50 and where.count("last") >= 3 and where.count("long") == 1
    assert {p["minus"] for p in planted if p["where"] == "boundary"} == {0, 1}
    ex = L.only(hits, 0)
    it = L.hit_items(item_off, split, ex[0], ex[1])
    assert 0.005 * tot <= np.unique(it).size <= 0.02 * tot
    assert it.max() >= tot - 3 and set(ex[2].tolist()) == {0, 1}
    lg = L.exact_hits(buf, off, PATS["long"])
    assert lg[0].size == 1 and lg[1][0] // L.SPIECE != (lg[1][0] + L.SMAXPAT - 1) // L.SPIECE
    assert L.hit_items(item_off, split, lg[0], lg[1])[0] > 0.9 * tot


def test_first_hit_set():
    data, pat, q, plants = L.first_b()
    rows = fxo.fasta_scan(data)[0]
    uni = np.array([G.uniform_of(data, r) for r in rows])
    assert uni.all() and (rows["norm"] == 1).all() and len(rows) == 4
    pieces = (rows["slen"] - len(pat) + L.SPIECE) // L.SPIECE
    assert pieces.tolist() == [p for p, _, _, _ in L.B_PIECES] and 40 <= pieces.min() and pieces.max() <= 70
    nq = q["rid"].size
    assert 2 * nq >= 3 * L.MAX_FASTA_WARPS
    items, split = L.fasta_items(rows, uni, q["rid"], q["s"], q["e"], len(pat))
    assert ((items == 0) == (q["kind"] == "zero")).all()
    # the whole records' hits, then each slice's first hits from them; checked against searchlib on the records
    buf, off = L.fasta_haystacks(data, rows, np.arange(4), np.zeros(4, np.int64), rows["slen"])
    whole = L.exact_hits(buf, off, pat)
    hays = [buf[off[i]:off[i + 1]].tobytes() for i in range(4)]
    assert as_list(whole) == S.expected_hits(hays, pat, 3)
    fq, fs, fm = L.first_hits(L.slice_hits(whole, q["rid"], q["s"], q["e"], len(pat)))
    first = {(a, c): b for a, b, c in zip(fq.tolist(), fs.tolist(), fm.tolist())}
    seen = set()
    for i in np.flatnonzero(q["kind"] == "planted"):
        k, at = int(q["item"][i]), int(q["at"][i])
        assert first[(i, 0)] == k * L.SPIECE + at, i
        side = plants[int(q["rid"][i])]["side"]
        if (i, 1) in first:
            mi = first[(i, 1)] // L.SPIECE
            assert mi != k and (mi < k) == (side == "before")
            seen.add(("before" if mi < k else "after", k))
        else:
            seen.add(("none", k))
        if at == L.SPIECE - 1:
            seen.add(("runs into the next piece", k))
    assert {("before", k) for k in L.FIRST_ITEMS} | {("after", k) for k in L.FIRST_ITEMS} <= seen
    assert {("runs into the next piece", k) for k in L.FIRST_ITEMS} <= seen and ("none", 64) in seen
    # slices with s > 0 shift the piece grid; planted queries on every pass of the first-hit warps
    pl = np.flatnonzero(q["kind"] == "planted")
    assert len({int(s) % L.SPIECE for s in q["s"][pl]}) > 50
    w = 2 * pl
    assert (w < L.fasta_warps(2 * nq, 132)).any() and (w >= 2 * L.MAX_FASTA_WARPS).any()
    # the short slices mostly hold a hit
    sh = np.flatnonzero(q["kind"] == "short")
    assert 0.3 < np.isin(sh, fq).mean() < 0.9
    # the slices are whole[s:e]: the oracle's extraction of a sample
    smp = np.random.default_rng(0).choice(nq, 400, replace=False)
    out, o2 = L.fasta_haystacks(data, rows, q["rid"][smp], q["s"][smp], q["e"][smp])
    for j, i in enumerate(smp):
        assert out[o2[j]:o2[j + 1]].tobytes() == hays[q["rid"][i]][q["s"][i]:q["e"][i]]


def _tile_items_loop(rlen, m):
    """tile_items, lane by lane as the kernel states it: items of each tile"""
    out = []
    for t in range(-(-len(rlen) // 32)):
        L_ = [rlen[t * 32 + j] if t * 32 + j < len(rlen) else None for j in range(32)]
        brk = [x is None or x > L.SPIECE for x in L_]
        n = 0
        for j, x in enumerate(L_):
            if x is None:
                continue
            if x > L.SPIECE:
                n += (x - m + L.SPIECE) // L.SPIECE
            elif j == 0 or brk[j - 1]:
                n += 1
        out.append(n)
    return out


def test_reads_items_restatement():
    rng = np.random.default_rng(5)
    rlen = rng.integers(0, 300, 1000)
    rlen[rng.choice(1000, 60, replace=False)] = rng.integers(L.SPIECE - 2, 5 * L.SPIECE, 60)
    rlen[64:70] = L.SPIECE + 1
    for n in (1000, 999, 993, 961):
        for m in (1, 16, 1024):
            R = L.reads_items(rlen[:n], m)
            assert R["tile"].tolist() == _tile_items_loop(rlen[:n].tolist(), m)
            # each read sits in its item's lanes; a long read's pieces follow each other
            tile = np.arange(n) // 32
            it = R["read_item"]
            assert (R["lane0"][it] <= np.arange(n) % 32).all()
            assert (np.arange(n) % 32 < R["lane0"][it] + R["lanes"][it]).all()
            lg = np.flatnonzero(rlen[:n] > L.SPIECE)
            assert (R["piece"][it[lg]] == 0).all() and (R["piece"][it[rlen[:n] <= L.SPIECE]] == -1).all()
            assert (np.bincount(tile[np.unique(it, return_index=True)[1]], minlength=R["tile"].size) <= R["tile"]).all()


def test_fastq_items_give_every_warp_three(fq_c):
    data, tiles, planted, rows, buf, off, rare = fq_c
    assert len(rows) == 32 * len(tiles) and 40e6 <= len(data) <= 60e6
    for p in PATS.values():
        R = L.reads_items(rows["rlen"], len(p))
        tot = int(R["tile"].sum())
        assert tot >= 3 * L.MAX_READS_WARPS + 97, len(p)
        for drop in (0, 1, 37, 301):
            t = int(L.reads_items(rows["rlen"][:len(rows) - drop], len(p))["tile"].sum())
            for sms in range(1, L.MAX_SMS + 1):
                for c in range(1, L.READS_CTAS_PER_SM + 1):
                    assert L.reads_per_warp(t, sms, c) >= 3, (len(p), drop, sms, c)
    # each truncation changes the item total, so the warps' ranges and the last one's length move on any grid
    totals = {int(L.reads_items(rows["rlen"][:len(rows) - d], L.M_RARE)["tile"].sum()) for d in (0, 1, 37, 301)}
    assert len(totals) == 4


def test_fastq_tile_kinds(fq_c):
    data, tiles, planted, rows, buf, off, rare = fq_c
    R = L.reads_items(rows["rlen"], L.M_RARE)
    assert R["tile"].tolist() == [t["items"] for t in tiles]
    kind = np.array([t["kind"] for t in tiles])
    rl = rows["rlen"].reshape(-1, 32)
    assert set(kind.tolist()) == {"short", "long1", "longs", "piece", "crlf", "last"} and kind[-1] == "last"
    sh = rl[kind == "short"]
    assert sh.max() <= 120 and (sh == 0).any() and ((sh > 0) & (sh < L.M_RARE)).any()
    assert ((rl[kind == "long1"] > L.SPIECE).sum(axis=1) == 1).all()
    nl = (rl[kind == "longs"] > L.SPIECE).sum(axis=1)
    assert nl.min() == 2 and nl.max() == 5
    assert ((rl[kind == "piece"] == L.SPIECE).sum(axis=1) == 2).all()
    assert ((rl[kind == "piece"] == L.SPIECE + 1).sum(axis=1) == 2).all()
    lp = R["tile"][kind == "long1"] - 2
    assert lp.min() == 5 and lp.max() == 12
    # the CRLF stretch: one run of tiles whose lines end in '\r\n', sequences without the '\r'
    cr = np.flatnonzero(kind == "crlf")
    assert cr.size == L.C_CRLF_TILES and np.all(np.diff(cr) == 1)
    a = np.frombuffer(data, np.uint8)
    first = rows[cr[0] * 32]
    assert a[first["soff"] + first["rlen"]] == 13 and a[rows[0]["soff"] + rows[0]["rlen"]] == 10
    for i in np.concatenate([np.arange(cr[0] * 32 - 3, cr[0] * 32 + 40), np.arange(len(rows) - 40, len(rows))]):
        assert buf[off[i]:off[i + 1]].tobytes() == fxo.read_fetch(data, rows[i])[0]
    assert not np.isin(buf, [10, 13]).any()


def test_planted_fastq_hits(fq_c):
    data, tiles, planted, rows, buf, off, rare = fq_c
    hits = rare
    got = set(as_list(hits))
    for p in planted:
        if p["m"] == L.M_RARE:
            assert (p["rid"], p["pos"], p["minus"], p["d"]) in got, p
    R = L.reads_items(rows["rlen"], L.M_RARE)
    tot = int(R["tile"].sum())
    ex = L.only(hits, 0)
    it = L.read_hit_items(R["read_item"], rows["rlen"], ex[0], ex[1])
    assert 0.005 * tot <= np.unique(it).size <= 0.02 * tot and it.max() >= tot - 3
    bd = [p for p in planted if p["where"] == "boundary"]
    assert len(bd) == 40 and all((p["pos"] + L.M_RARE - 1) % L.SPIECE < L.M_RARE for p in bd)
    lg = L.exact_hits(buf, off, PATS["long"])
    assert lg[0].size == 1 and lg[0][0] // 32 == len(tiles) - 1 and rows["rlen"][lg[0][0]] > L.SPIECE
    assert lg[1][0] // L.SPIECE != (lg[1][0] + L.SMAXPAT - 1) // L.SPIECE and lg[2][0] == 1


def test_slices_d(fa_a):
    data, kinds, planted, zero_runs, rows, uni, buf, off, rare = fa_a
    rid, s, e = L.slices_d(rows, uni, planted)
    nq = rid.size
    assert nq == L.D_NQ == (1 << 21) + 1 and G.prefix_chunks(nq) == 2
    items, _ = L.fasta_items(rows, uni, rid, s, e, L.M_RARE)
    assert (items == 1).all()                                  # item and hit prefixes: 2^21 + 1 entries each
    assert ((e - s >= 64) & (e - s <= 400)).all() and uni[rid].all()
    whole = rare
    ex = L.slice_hits(L.only(whole, 0), rid, s, e, L.M_RARE)
    assert 0.2 < np.unique(ex[0]).size / nq < 0.4
    # whole[s:e] is what the oracle extracts, on a sample
    smp = np.random.default_rng(1).choice(nq, 20_000, replace=False)
    out, o2 = L.fasta_haystacks(data, rows, rid[smp], s[smp], e[smp])
    src = np.repeat(off[rid[smp]] + s[smp] - o2[:-1], e[smp] - s[smp]) + np.arange(int(o2[-1]))
    assert np.array_equal(out, buf[src])
    # slice_hits on the sample equals searchlib / approxlib on the sample's haystacks
    hays = [out[o2[j]:o2[j + 1]].tobytes() for j in range(smp.size)]
    sub = L.slice_hits(whole, rid[smp], s[smp], e[smp], L.M_RARE)
    assert as_list(L.only(sub, 0)[:3]) == S.expected_hits(hays, PATS["rare"], 3)
    assert as_list(L.only(sub, 1)) == A.expected_hits(hays, PATS["rare"], 1, 3)


def _check_reference(buf, off, pats, ks=(1, 2), approx_upto=16):
    hays = [buf[off[i]:off[i + 1]].tobytes() for i in range(off.size - 1)]
    for p in pats:
        for strands in (1, 2, 3):
            assert as_list(L.exact_hits(buf, off, p, strands)) == S.expected_hits(hays, p, strands), (p[:20], strands)
        if len(p) > approx_upto:
            continue
        both = L.approx_hits(buf, off, p, max(ks))
        counts = A.strand_counts(hays, p)
        for k in ks:
            if k < len(p):
                for strands in (1, 2, 3):
                    assert as_list(L.only(both, k, strands)) == A.expected_from_counts(counts, k, strands), (p[:20], k)


def test_reference_on_samples(fa_a, fq_c):
    """the vectorised reference equals searchlib / approxlib on a seeded sample of each set"""
    rng = np.random.default_rng(2)
    data, kinds, planted, zero_runs, rows, uni, _, _, _ = fa_a
    i = np.sort(rng.choice(len(rows), 150, replace=False))
    i = np.concatenate([i, [p["rid"] for p in planted[:40]], np.arange(len(rows) - 8, len(rows))])
    buf, off = L.fasta_haystacks(data, rows, i, np.zeros(i.size, np.int64), rows["slen"][i])
    _check_reference(buf, off, list(PATS.values()))
    data, tiles, planted, rows, buf, off, rare = fq_c
    sel = rows[np.sort(np.concatenate([rng.choice(len(rows), 1000, replace=False), [p["rid"] for p in planted]]))]
    buf, off = L.read_haystacks(data, sel)
    _check_reference(buf, off, [PATS["rare"], PATS["gaattc"], PATS["t"]])
    hays = [fxo.read_fetch(data, r)[0] for r in sel]
    assert b"".join(hays) == buf.tobytes()


def test_reference_on_existing_inputs():
    """... and on the inputs of the existing search tests: the golden file, synth files, irregular layouts"""
    data = gzip.open(os.path.join(goldenlib.GOLD, "data", "test.fa.gz")).read()
    rows = fxo.fasta_scan(data)[0][:40]
    buf, off = L.fasta_haystacks(data, rows, np.arange(40), np.zeros(40, np.int64), rows["slen"])
    _check_reference(buf, off, [b"GCTTCAATACA", b"GAATTC", b"A", b"ACGTN"])
    for seed in (1, 2):
        data = gen.random_fasta(seed)
        rows = fxo.fasta_scan(data)[0]
        n = len(rows)
        buf, off = L.fasta_haystacks(data, rows, np.arange(n), np.zeros(n, np.int64), rows["slen"])
        _check_reference(buf, off, [b"ACG", b"acgt", b"N", bytes(buf[100:117])])
    data = synth.synth_fastq(3000, seed=20240602)
    buf, off = L.read_haystacks(data, fxo.fastq_scan(data)[0])
    _check_reference(buf, off, [b"GAATTC", b"T", bytes(buf[500:530])])
    data = gen.random_fastq(3, crlf=True)
    buf, off = L.read_haystacks(data, fxo.fastq_scan(data)[0])
    _check_reference(buf, off, [b"AC", bytes(buf[50:60])], ks=(1,))
